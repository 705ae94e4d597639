/* C module adapters: the bodies a reference maintainer puts behind each module's
 * process() / process_cl() / tiling_callback() (src/iop/iop_api.h:265-266, 292-293, 121-122).
 *
 * The reference prefixes a module's plain symbols with dt_iop_<op>__ through asm labels
 * (src/common/module_api.h:139-154); the same names are exported here so the adapters can be
 * exercised from tests exactly as lib_ansel would call them.  Everything else of each module
 * (params, commit_params, GUI, introspection) stays the reference's own C.
 *
 * Return conventions (SURVEY.md 3.3): process() 0 = success; process_cl() TRUE = success.
 */
#include "dt_surface.h"
#include <math.h>
#include <string.h>

#define ADAPT(op)                                                                                         \
  int dt_iop_##op##__process(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe,                \
                             const dt_dev_pixelpipe_iop_t *piece, const void *const i, void *const o)     \
  {                                                                                                       \
    b200_piece_t p;                                                                                       \
    b200_piece_from_dt(&p, self, pipe, piece);                                                            \
    return b200_##op##_process_host(&p, i, o);                                                            \
  }                                                                                                       \
  int dt_iop_##op##__process_cl(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe,             \
                                const dt_dev_pixelpipe_iop_t *piece, cl_mem dev_in, cl_mem dev_out)       \
  {                                                                                                       \
    b200_piece_t p;                                                                                       \
    b200_piece_from_dt(&p, self, pipe, piece);                                                            \
    return b200_##op##_process_dev(&p, dev_in, dev_out, pipe->stream) == 0 ? TRUE : FALSE;                \
  }                                                                                                       \
  void dt_iop_##op##__tiling_callback(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe,       \
                                      const dt_dev_pixelpipe_iop_t *piece, dt_develop_tiling_t *tiling)   \
  {                                                                                                       \
    b200_piece_t p;                                                                                       \
    b200_piece_from_dt(&p, self, pipe, piece);                                                            \
    b200_##op##_tiling(&p, tiling);                                                                       \
  }

/* demosaic: src/iop/demosaic.c:1043 (process), rcd.c:568 (process_rcd_cl), :1916 (tiling_callback).  FDC's process() reads the user's
 * crossover ISO (markesteijn.c:1137); the adapter carries it next to a copy of the data block. */
int b200_userpref_fdc_xover_iso = 1600; /* plugins/darkroom/demosaic/fdc_xover_iso, data/anselconfig.xml.in:1814 */
static int demosaic_view(b200_demosaic_piece_t *dp, b200_piece_t *p, const dt_dev_pixelpipe_iop_t *piece)
{
  if(!piece->data || piece->data_size < sizeof(b200_demosaic_data_t)) return 1;
  memcpy(&dp->data, piece->data, sizeof(b200_demosaic_data_t));
  dp->fdc_xover_iso = b200_userpref_fdc_xover_iso;
  p->data = dp;
  p->data_size = sizeof(*dp);
  return 0;
}
int dt_iop_demosaic__process(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece, const void *const i,
                             void *const o)
{
  b200_piece_t p;
  b200_demosaic_piece_t dp;
  b200_piece_from_dt(&p, self, pipe, piece);
  if(demosaic_view(&dp, &p, piece)) return 1;
  return b200_demosaic_process_host(&p, i, o);
}
int dt_iop_demosaic__process_cl(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece, cl_mem dev_in,
                                cl_mem dev_out)
{
  b200_piece_t p;
  b200_demosaic_piece_t dp;
  b200_piece_from_dt(&p, self, pipe, piece);
  if(demosaic_view(&dp, &p, piece)) return FALSE;
  return b200_demosaic_process_dev(&p, dev_in, dev_out, pipe->stream) == 0 ? TRUE : FALSE;
}
void dt_iop_demosaic__tiling_callback(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                                      dt_develop_tiling_t *tiling)
{
  b200_piece_t p;
  b200_piece_from_dt(&p, self, pipe, piece);
  b200_demosaic_tiling(&p, tiling);
}
ADAPT(colorin)  /* src/iop/colorin.c:711, :590-681 (process_cl) */
ADAPT(colorout) /* src/iop/colorout.c:373, :288-371 (process_cl) */

ADAPT(denoiseprofile) /* src/iop/denoiseprofile.c:2037 (process), :1880-2035 (process_cl), :1091 (tiling_callback) */
ADAPT(diffuse)        /* src/iop/diffuse.c:1155 (process), :1486 (process_cl), :585 (tiling_callback) */
ADAPT(nlmeans)        /* src/iop/nlmeans.c:458 (process), :150-398 (process_cl), :400 (tiling_callback) */
ADAPT(bilat)          /* src/iop/bilat.c:336 (process), :313-334 (process_cl), :296 (commit: tiling off) */

/* the modules either side of that path (SURVEY.md 8f): sensor data in, display/export integers out */
ADAPT(rawprepare)  /* src/iop/rawprepare.c:467 (process), :636 (process_cl); default_tiling_callback */
ADAPT(temperature) /* src/iop/temperature.c:487 (process), :611 (process_cl) */
ADAPT(highlights)  /* src/iop/highlights.c:680 (process), :464 (process_cl), :575 (tiling_callback) */
ADAPT(exposure)    /* src/iop/exposure.c:503 (process), :473 (process_cl) */
ADAPT(gamma)       /* src/iop/gamma.c:367 (process), :461 (process_cl) */

/* colour calibration reads the work profile next to piece->data (channelmixerrgb.c:1926, :1936-1942); everything of its
 * process() that precedes the switch on data->adaptation -- the GUI's colour-checker fit and illuminant detection, the
 * re-derivation of data->illuminant for DT_ILLUMINANT_CAMERA from the image metadata (:1986-2014) -- stays in the
 * reference and runs before this call. */
static int channelmixer_view(b200_channelmixerrgb_piece_t *cp, b200_piece_t *p, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece)
{
  if(!piece->data || piece->data_size < sizeof(b200_channelmixerrgb_data_t)) return 1;
  memcpy(&cp->data, piece->data, sizeof(b200_channelmixerrgb_data_t));
  const dt_iop_order_iccprofile_info_t *const work = dt_ioppr_get_pipe_work_profile_info(pipe); /* = dt_ioppr_get_pipe_current_profile_info(self, pipe) */
  if(!work) return 1; /* the reference would multiply by uninitialised matrices: refuse */
  memcpy(cp->work_profile.matrix_in, work->matrix_in, sizeof(work->matrix_in));
  memcpy(cp->work_profile.matrix_out, work->matrix_out, sizeof(work->matrix_out));
  p->data = cp;
  p->data_size = sizeof(*cp);
  return 0;
}
int dt_iop_channelmixerrgb__process(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                                    const void *const i, void *const o)
{
  b200_piece_t p;
  b200_channelmixerrgb_piece_t cp;
  b200_piece_from_dt(&p, self, pipe, piece);
  if(channelmixer_view(&cp, &p, pipe, piece)) return 1;
  return b200_channelmixerrgb_process_host(&p, i, o);
}
int dt_iop_channelmixerrgb__process_cl(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                                       cl_mem dev_in, cl_mem dev_out)
{
  b200_piece_t p;
  b200_channelmixerrgb_piece_t cp;
  b200_piece_from_dt(&p, self, pipe, piece);
  if(channelmixer_view(&cp, &p, pipe, piece)) return FALSE;
  return b200_channelmixerrgb_process_dev(&p, dev_in, dev_out, pipe->stream) == 0 ? TRUE : FALSE;
}
void dt_iop_channelmixerrgb__tiling_callback(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe,
                                             const dt_dev_pixelpipe_iop_t *piece, dt_develop_tiling_t *tiling)
{
  b200_piece_t p;
  b200_piece_from_dt(&p, self, pipe, piece);
  b200_channelmixerrgb_tiling(&p, tiling);
}

/* colour balance rgb reads the pipe's current work profile next to piece->data (colorbalancergb.c:590-591) and the gamut LUT behind
 * data->gamut_LUT, which commit_params() builds and the library reads as given.  piece->data_size is the hashed prefix (init_pipe
 * :1365); the runtime pointers follow it in the reference's struct. */
typedef struct cbrgb_ref_data_t
{
  b200_colorbalancergb_data_t prefix;
  const void *work_profile;
  const float *gamut_LUT;
  const float *chroma_LUT;
} cbrgb_ref_data_t;
/* 1: not a colour balance rgb piece; -1: no work profile (process() :592 returns without writing) */
static int colorbalancergb_view(b200_colorbalancergb_piece_t *cp, b200_piece_t *p, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece)
{
  if(!piece->data || piece->data_size < sizeof(b200_colorbalancergb_data_t)) return 1;
  const cbrgb_ref_data_t *d = (const cbrgb_ref_data_t *)piece->data;
  if(!d->gamut_LUT) return 1;
  const dt_iop_order_iccprofile_info_t *const work = dt_ioppr_get_pipe_work_profile_info(pipe); /* = dt_ioppr_get_pipe_current_profile_info(self, pipe) */
  if(!work) return -1;
  memcpy(&cp->data, &d->prefix, sizeof(cp->data));
  memcpy(cp->work_profile.matrix_in, work->matrix_in, sizeof(work->matrix_in));
  memcpy(cp->work_profile.matrix_out, work->matrix_out, sizeof(work->matrix_out));
  memcpy(cp->gamut_LUT, d->gamut_LUT, sizeof(cp->gamut_LUT));
  p->data = cp;
  p->data_size = sizeof(*cp);
  return 0;
}
int dt_iop_colorbalancergb__process(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                                    const void *const i, void *const o)
{
  b200_piece_t p;
  b200_colorbalancergb_piece_t cp;
  b200_piece_from_dt(&p, self, pipe, piece);
  const int v = colorbalancergb_view(&cp, &p, pipe, piece);
  if(v) return v < 0 ? 0 : 1;
  return b200_colorbalancergb_process_host(&p, i, o);
}
int dt_iop_colorbalancergb__process_cl(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                                       cl_mem dev_in, cl_mem dev_out)
{
  b200_piece_t p;
  b200_colorbalancergb_piece_t cp;
  b200_piece_from_dt(&p, self, pipe, piece);
  const int v = colorbalancergb_view(&cp, &p, pipe, piece);
  if(v) return v < 0 ? TRUE : FALSE; /* process_cl :946-948 returns its (non-zero) default error code there: not a failure */
  return b200_colorbalancergb_process_dev(&p, dev_in, dev_out, pipe->stream) == 0 ? TRUE : FALSE;
}
void dt_iop_colorbalancergb__tiling_callback(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe,
                                             const dt_dev_pixelpipe_iop_t *piece, dt_develop_tiling_t *tiling)
{
  b200_piece_t p;
  b200_piece_from_dt(&p, self, pipe, piece);
  b200_colorbalancergb_tiling(&p, tiling);
}

/* finalscale's data block is one dummy int (finalscale.c:46-51); its process() resolves the interpolator from the user
 * preference: dt_interpolation_new(DT_INTERPOLATION_USERPREF) (develop/imageop_math.c:150).  In the reference tree the
 * adapter passes that interpolator's id; standing alone, dt_surface.h keeps the preference in a variable. */
int b200_userpref_interpolator = B200_INTERPOLATION_MITCHELL; /* plugins/lighttable/export/pixel_interpolator, default "mitchell" */
static void finalscale_view(b200_finalscale_data_t *fd, b200_piece_t *p)
{
  fd->dummy = 0;
  fd->interpolator = b200_userpref_interpolator; /* = dt_interpolation_new(DT_INTERPOLATION_USERPREF)->id */
  p->data = fd;
  p->data_size = sizeof(*fd);
}
int dt_iop_finalscale__process(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                               const void *const i, void *const o)
{
  b200_piece_t p;
  b200_finalscale_data_t fd;
  b200_piece_from_dt(&p, self, pipe, piece);
  finalscale_view(&fd, &p);
  return b200_finalscale_process_host(&p, i, o);
}
int dt_iop_finalscale__process_cl(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                                  cl_mem dev_in, cl_mem dev_out)
{
  b200_piece_t p;
  b200_finalscale_data_t fd;
  b200_piece_from_dt(&p, self, pipe, piece);
  finalscale_view(&fd, &p);
  return b200_finalscale_process_dev(&p, dev_in, dev_out, pipe->stream) == 0 ? TRUE : FALSE;
}
void dt_iop_finalscale__tiling_callback(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe,
                                        const dt_dev_pixelpipe_iop_t *piece, dt_develop_tiling_t *tiling)
{
  b200_piece_t p;
  b200_piece_from_dt(&p, self, pipe, piece);
  b200_finalscale_tiling(&p, tiling);
}

ADAPT(flip) /* src/iop/flip.c:388 (process), :403 (process_cl); default_tiling_callback */
/* initialscale resamples like finalscale, with the user's interpolator and the ROIs as they are (iop/initialscale.c:122-129) */
int dt_iop_initialscale__process(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                                 const void *const i, void *const o)
{
  b200_piece_t p;
  b200_finalscale_data_t fd;
  b200_piece_from_dt(&p, self, pipe, piece);
  finalscale_view(&fd, &p);
  return b200_initialscale_process_host(&p, i, o);
}
int dt_iop_initialscale__process_cl(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                                    cl_mem dev_in, cl_mem dev_out)
{
  b200_piece_t p;
  b200_finalscale_data_t fd;
  b200_piece_from_dt(&p, self, pipe, piece);
  finalscale_view(&fd, &p);
  return b200_initialscale_process_dev(&p, dev_in, dev_out, pipe->stream) == 0 ? TRUE : FALSE;
}
void dt_iop_initialscale__tiling_callback(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe,
                                          const dt_dev_pixelpipe_iop_t *piece, dt_develop_tiling_t *tiling)
{
  b200_piece_t p;
  b200_piece_from_dt(&p, self, pipe, piece);
  b200_initialscale_tiling(&p, tiling);
}

/* lens correction's process() resolves its interpolator from the user preference (dt_interpolation_new(DT_INTERPOLATION_USERPREF_WARP),
 * lens.c:716); the adapter carries it next to a copy of the data block.  Which images are monochrome comes with the piece
 * (image_flags). */
int b200_userpref_warp_interpolator = B200_INTERPOLATION_MITCHELL; /* plugins/lighttable/export/pixel_interpolator_warp, default "mitchell" */
static int lens_view(b200_lens_piece_t *lp, b200_piece_t *p, const dt_dev_pixelpipe_iop_t *piece)
{
  if(!piece->data || piece->data_size < sizeof(b200_lens_data_t)) return 1;
  memcpy(&lp->data, piece->data, sizeof(b200_lens_data_t));
  lp->interpolation = b200_userpref_warp_interpolator;
  p->data = lp;
  p->data_size = sizeof(*lp);
  return 0;
}
int dt_iop_lens__process(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece, const void *const i,
                         void *const o)
{
  b200_piece_t p;
  static _Thread_local b200_lens_piece_t lp; /* 45 KB: kept off the caller's stack */
  b200_piece_from_dt(&p, self, pipe, piece);
  if(lens_view(&lp, &p, piece)) return 1;
  return b200_lens_process_host(&p, i, o);
}
int dt_iop_lens__process_cl(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece, cl_mem dev_in,
                            cl_mem dev_out)
{
  b200_piece_t p;
  static _Thread_local b200_lens_piece_t lp;
  b200_piece_from_dt(&p, self, pipe, piece);
  if(lens_view(&lp, &p, piece)) return FALSE;
  return b200_lens_process_dev(&p, dev_in, dev_out, pipe->stream) == 0 ? TRUE : FALSE;
}
void dt_iop_lens__tiling_callback(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                                  dt_develop_tiling_t *tiling)
{
  b200_piece_t p;
  b200_piece_from_dt(&p, self, pipe, piece);
  b200_lens_tiling(&p, tiling); /* reads nothing of the piece */
}

/* dither's process() reads pipe->levels next to piece->data (get_dither_parameters, dither.c:285-314): the adapter copies the
 * data block and adds it */
static int dither_view(b200_dither_data_t *dd, b200_piece_t *p, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece)
{
  const size_t n = offsetof(b200_dither_data_t, levels); /* sizeof(dt_iop_dither_data_t) */
  if(!piece->data || piece->data_size < n) return 1;
  memcpy(dd, piece->data, n);
  dd->levels = pipe->levels;
  p->data = dd;
  p->data_size = sizeof(*dd);
  return 0;
}
int dt_iop_dither__process(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                           const void *const i, void *const o)
{
  b200_piece_t p;
  b200_dither_data_t dd;
  b200_piece_from_dt(&p, self, pipe, piece);
  if(dither_view(&dd, &p, pipe, piece)) return 1;
  return b200_dither_process_host(&p, i, o);
}
int dt_iop_dither__process_cl(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                              cl_mem dev_in, cl_mem dev_out)
{
  b200_piece_t p;
  b200_dither_data_t dd;
  b200_piece_from_dt(&p, self, pipe, piece);
  if(dither_view(&dd, &p, pipe, piece)) return FALSE;
  return b200_dither_process_dev(&p, dev_in, dev_out, pipe->stream) == 0 ? TRUE : FALSE;
}
void dt_iop_dither__tiling_callback(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe, const dt_dev_pixelpipe_iop_t *piece,
                                    dt_develop_tiling_t *tiling)
{
  b200_piece_t p;
  b200_piece_from_dt(&p, self, pipe, piece);
  b200_dither_tiling(&p, tiling); /* reads the two ROIs only */
}

/* filmic reads two pipe-level profiles next to piece->data (filmicrgb.c:2714-2715); the adapter flattens the
 * three into the b200_filmicrgb_piece_t the library takes.  A soft-proof profile (data->softproof_mode != 0,
 * _filmic_get_output_profile :2650-2666) is resolved by the reference's own dt_colorspaces_add_profile() in
 * the maintainer's tree; here the pipe output profile is what is available. */
#include <math.h>
#include <string.h>
static int filmic_view(b200_filmicrgb_piece_t *fp, b200_piece_t *p, const dt_dev_pixelpipe_t *pipe,
                       const dt_dev_pixelpipe_iop_t *piece)
{
  if(!piece->data || piece->data_size < sizeof(b200_filmicrgb_data_t)) return 1;
  memcpy(&fp->data, piece->data, sizeof(b200_filmicrgb_data_t));
  const dt_iop_order_iccprofile_info_t *const work = dt_ioppr_get_pipe_work_profile_info(pipe);
  const dt_iop_order_iccprofile_info_t *const out = dt_ioppr_get_pipe_output_profile_info(pipe);
  if(!work) return 1; /* filmicrgb.c:2716: "no work profile" -> process() fails */
  memcpy(fp->work_profile.matrix_in, work->matrix_in, sizeof(work->matrix_in));
  memcpy(fp->work_profile.matrix_out, work->matrix_out, sizeof(work->matrix_out));
  fp->has_export_profile = out && !isnan(out->matrix_in[0][0]) && !isnan(out->matrix_out[0][0]);
  if(fp->has_export_profile)
  {
    memcpy(fp->export_profile.matrix_in, out->matrix_in, sizeof(out->matrix_in));
    memcpy(fp->export_profile.matrix_out, out->matrix_out, sizeof(out->matrix_out));
  }
  else
    memset(&fp->export_profile, 0, sizeof(fp->export_profile));
  p->data = fp;
  p->data_size = sizeof(*fp);
  return 0;
}
int dt_iop_filmicrgb__process(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe,
                              const dt_dev_pixelpipe_iop_t *piece, const void *const i, void *const o)
{
  b200_piece_t p;
  b200_filmicrgb_piece_t fp;
  b200_piece_from_dt(&p, self, pipe, piece);
  if(filmic_view(&fp, &p, pipe, piece)) return 1;
  return b200_filmicrgb_process_host(&p, i, o);
}
int dt_iop_filmicrgb__process_cl(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe,
                                 const dt_dev_pixelpipe_iop_t *piece, cl_mem dev_in, cl_mem dev_out)
{
  b200_piece_t p;
  b200_filmicrgb_piece_t fp;
  b200_piece_from_dt(&p, self, pipe, piece);
  if(filmic_view(&fp, &p, pipe, piece)) return FALSE;
  return b200_filmicrgb_process_dev(&p, dev_in, dev_out, pipe->stream) == 0 ? TRUE : FALSE;
}
void dt_iop_filmicrgb__tiling_callback(struct dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe,
                                       const dt_dev_pixelpipe_iop_t *piece, dt_develop_tiling_t *tiling)
{
  b200_piece_t p;
  b200_piece_from_dt(&p, self, pipe, piece);
  b200_filmicrgb_tiling(&p, tiling); /* reads roi_in and the data block's reconstruction settings only */
}

/* layout probes so non-C callers (tests, bench.py) can verify their mirror of dt_surface.h */
#include <stddef.h>
size_t b200_dt_surface_probe(int which)
{
  switch(which)
  {
    case 0: return sizeof(dt_iop_buffer_dsc_t);
    case 1: return offsetof(dt_iop_buffer_dsc_t, temperature.coeffs);
    case 2: return offsetof(dt_iop_buffer_dsc_t, processed_maximum);
    case 3: return offsetof(dt_iop_buffer_dsc_t, cst);
    case 4: return sizeof(dt_dev_pixelpipe_iop_t);
    case 5: return offsetof(dt_dev_pixelpipe_iop_t, roi_in);
    case 6: return offsetof(dt_dev_pixelpipe_iop_t, dsc_in);
    case 7: return offsetof(dt_dev_pixelpipe_iop_t, dsc_out);
    case 8: return sizeof(dt_dev_pixelpipe_t);
    case 9: return sizeof(dt_iop_module_t);
    case 10: return sizeof(b200_piece_t);
    case 11: return sizeof(b200_conversion_t);
    case 12: return sizeof(dt_iop_order_iccprofile_info_t);
    case 13: return offsetof(dt_dev_pixelpipe_t, work_profile_info);
    default: return 0;
  }
}
