// b200_demosaic_*: the demosaic module's process()/process_cl()/tiling_callback() bodies.
// Reference: src/iop/demosaic.c:1043-1253 (process), :1916-2013 (tiling_callback).
#include "runtime.h"
#include <math.h>

namespace b200
{
int rcd_demosaic_dev(const float *d_in, float *d_out, int width, int height, uint32_t filters,
                     const float processed_maximum[3], cudaStream_t stream);
int amaze_demosaic_dev(const float *d_in, float *d_out, int width, int height, uint32_t filters, const float processed_maximum[3], cudaStream_t stream);
int vng_demosaic_dev(const float *d_in, float *d_out, int width, int height, int x0, int y0, uint32_t filters, const uint8_t *xtrans36, int lin_slot,
                     const double (*cam_to_rgb)[4], cudaStream_t s);
int dual_demosaic_dev(float *d_rgb, const float *d_raw, int width, int height, int x0, int y0, uint32_t filters, const uint8_t *xtrans36, const float wb[4],
                      float dual_threshold, cudaStream_t s);
int passthrough_demosaic_dev(const float *d_in, float *d_out, int width, int height, int colour, uint32_t filters, int x0, int y0, const uint8_t xtrans[6][6],
                             cudaStream_t s);
int downsample_demosaic_dev(const float *d_in, float *d_out, int width, int height, uint32_t filters, cudaStream_t s);
int demosaic_postfilter_dev(float *d_rgba, int width, int height, int iterations, cudaStream_t s);
int downsample4_demosaic_dev(const float *d_in, float *d_out, int width, int height, uint32_t filters, const double cam_to_rgb[3][4], cudaStream_t s);
int downsample_xtrans_demosaic_dev(const float *d_in, float *d_out, int width, int height, int x0, int y0, const uint8_t xtrans[6][6], cudaStream_t s);
int ppg_demosaic_dev(const float *d_in, float *d_out, int width, int height, uint32_t filters, float median_thrs, cudaStream_t s);
int lmmse_demosaic_dev(const float *d_in, float *d_out, int width, int height, uint32_t filters, int mode, const float processed_maximum[3], cudaStream_t stream);
int markesteijn_demosaic_dev(const float *d_in, float *d_out, int width, int height, int x0, int y0, const uint8_t xtrans[6][6], int passes, cudaStream_t stream);
int fdc_demosaic_dev(const float *d_in, float *d_out, int width, int height, int x0, int y0, const uint8_t xtrans[6][6], int pure, cudaStream_t stream);
int demosaic_green_eq_dev(const float *d_in, float *d_tmp0, float *d_tmp1, double *d_partial, int width, int height, uint32_t dsc_filters, int x, int y,
                          unsigned green_eq, float threshold, const float **d_result, cudaStream_t s);
int demosaic_green_eq_partial_doubles();
int demosaic_color_smoothing_dev(float *d_out, int width, int height, int passes, cudaStream_t s);
}
#define DT_IMAGE_4BAYER (1u << 14) /* common/image.h:139 */
using namespace b200;

#define DEMOSAIC_DUAL 2048 /* iop/demosaic.c:109 */
#define MARKEST3_VNG (DEMOSAIC_DUAL | 1026u) /* DT_IOP_DEMOSAIC_MARKEST3_VNG, iop/demosaic.c:138 */

// methods that, like the reference, leave (part of) the alpha lane as they find it
static bool keeps_alpha(uint32_t m)
{
  return m == B200_DEMOSAIC_PPG || m == 3u || m == 4u || m == 1024u || m == 1025u || m == 1026u || m == B200_DEMOSAIC_FDC || m == MARKEST3_VNG;
}

static int check_piece(const b200_piece_t *piece, const void *in, void *out)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "demosaic: NULL argument");
  if(!piece->data || piece->data_size < sizeof(b200_demosaic_data_t))
    return fail(B200_ERR_ARG, "demosaic: piece->data is not a b200_demosaic_data_t");
  if(piece->roi_in.width <= 0 || piece->roi_in.height <= 0) return fail(B200_ERR_ARG, "demosaic: empty roi_in");
  return B200_OK;
}

extern "C" int b200_demosaic_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = check_piece(piece, d_in, d_out);
  if(rc) return rc;
  rc = bind_device(piece->devid);
  if(rc) return rc;
  const b200_demosaic_data_t *d = (const b200_demosaic_data_t *)piece->data;
  // demosaic.c:1071 -- fold the ROI origin into the CFA phase for the tile-local algorithms
  const uint32_t filters = b200_roi_filters(piece->filters, piece->roi_in.x, piece->roi_in.y);
  // the passthrough methods come first and take any sensor (demosaic.c:1111-1118); colour smoothing still follows (:1249),
  // green equilibration does not apply
  {
    const uint32_t m = d->demosaicing_method;
    const bool mono = m == 3u, colour = m == 4u; // commit_params() :2196-2199 folds the X-Trans ids (1027, 1029) onto these
    if(mono || colour)
    {
      if(piece->roi_out.width != piece->roi_in.width || piece->roi_out.height != piece->roi_in.height)
        return fail(B200_ERR_UNSUPPORTED, "demosaic: passthrough with roi_out != roi_in");
      rc = passthrough_demosaic_dev((const float *)d_in, (float *)d_out, piece->roi_in.width, piece->roi_in.height, colour ? 1 : 0, piece->filters,
                                    piece->roi_in.x, piece->roi_in.y, piece->xtrans, (cudaStream_t)stream);
      if(rc) return rc;
      if(d->color_smoothing)
        rc = demosaic_color_smoothing_dev((float *)d_out, piece->roi_out.width, piece->roi_out.height, (int)d->color_smoothing, (cudaStream_t)stream);
      return rc;
    }
  }
  if(d->demosaicing_method == 7u)
  { // DT_IOP_DEMOSAIC_DOWNSAMPLE, demosaic.c:1101-1108: half-size output (modify_roi_out :940-952), then the guided-Laplacian
    // post-filter when data->color_smoothing asks for iterations of it
    if(piece->roi_out.width != (piece->roi_in.width + 1) / 2 || piece->roi_out.height != (piece->roi_in.height + 1) / 2)
      return fail(B200_ERR_ARG, "demosaic: downsample wants roi_out = (roi_in + 1) / 2, got %dx%d for %dx%d", piece->roi_out.width, piece->roi_out.height,
                  piece->roi_in.width, piece->roi_in.height);
    if(filters == 9u)
      rc = downsample_xtrans_demosaic_dev((const float *)d_in, (float *)d_out, piece->roi_in.width, piece->roi_in.height, piece->roi_in.x, piece->roi_in.y,
                                          piece->xtrans, (cudaStream_t)stream);
    else if(piece->image_flags & DT_IMAGE_4BAYER)
      rc = downsample4_demosaic_dev((const float *)d_in, (float *)d_out, piece->roi_in.width, piece->roi_in.height, filters, d->CAM_to_RGB, (cudaStream_t)stream);
    else
      rc = downsample_demosaic_dev((const float *)d_in, (float *)d_out, piece->roi_in.width, piece->roi_in.height, filters, (cudaStream_t)stream);
    if(rc) return rc;
    return demosaic_postfilter_dev((float *)d_out, piece->roi_out.width, piece->roi_out.height, (int)d->color_smoothing, (cudaStream_t)stream);
  }
  if(filters == 9u)
  { // demosaic.c:1119-1131: Markesteijn with one pass (DT_IOP_DEMOSAIC_MARKESTEIJN = 1025, the default of X-Trans frames, :1085) or three
    // (DT_IOP_DEMOSAIC_MARKESTEIJN_3 = 1026, and MARKEST3_VNG = 3074, which blends in VNG after it, :1243-1247); VNG is what every
    // X-Trans method below them resolves to (DT_IOP_DEMOSAIC_VNG = 1024)
    const uint32_t m = d->demosaicing_method;
    if(m != 1024u && m != 1025u && m != 1026u && m != MARKEST3_VNG && m != B200_DEMOSAIC_FDC)
      return fail(B200_ERR_UNSUPPORTED, "demosaic: X-Trans method %u is not built (VNG, Markesteijn, Markesteijn 3-pass + VNG and FDC are)", m);
    if(m == B200_DEMOSAIC_FDC && piece->data_size < sizeof(b200_demosaic_piece_t))
      return fail(B200_ERR_UNSUPPORTED, "demosaic: FDC is not built for a bare b200_demosaic_data_t: it needs fdc_xover_iso, the user's crossover ISO "
                                        "(pass a b200_demosaic_piece_t)");
    if(piece->roi_out.width != piece->roi_in.width || piece->roi_out.height != piece->roi_in.height)
      return fail(B200_ERR_UNSUPPORTED, "demosaic: roi_out != roi_in (downsampling paths are not built)");
    if(m == B200_DEMOSAIC_FDC)
    { // demosaic.c:1124-1125, then colour smoothing (:1249); markesteijn.c:1137-1139: int iso = exif_iso, pure FDC above the crossover
      const int iso = (int)piece->exif_iso, pure = iso > ((const b200_demosaic_piece_t *)piece->data)->fdc_xover_iso;
      rc = fdc_demosaic_dev((const float *)d_in, (float *)d_out, piece->roi_in.width, piece->roi_in.height, piece->roi_in.x, piece->roi_in.y, piece->xtrans,
                            pure, (cudaStream_t)stream);
      if(rc) return rc;
      if(d->color_smoothing)
        rc = demosaic_color_smoothing_dev((float *)d_out, piece->roi_out.width, piece->roi_out.height, (int)d->color_smoothing, (cudaStream_t)stream);
      return rc;
    }
    if(m == 1025u || m == 1026u || m == MARKEST3_VNG)
    {
      rc = markesteijn_demosaic_dev((const float *)d_in, (float *)d_out, piece->roi_in.width, piece->roi_in.height, piece->roi_in.x, piece->roi_in.y,
                                    piece->xtrans, m == 1025u ? 1 : 3, (cudaStream_t)stream);
      if(rc) return rc;
      if(m == MARKEST3_VNG
         && (rc = dual_demosaic_dev((float *)d_out, (const float *)d_in, piece->roi_in.width, piece->roi_in.height, piece->roi_in.x, piece->roi_in.y, 9u,
                                    &piece->xtrans[0][0], piece->wb_coeffs, d->dual_thrs, (cudaStream_t)stream)))
        return rc;
      if(d->color_smoothing)
        rc = demosaic_color_smoothing_dev((float *)d_out, piece->roi_out.width, piece->roi_out.height, (int)d->color_smoothing, (cudaStream_t)stream);
      return rc;
    }
    rc = vng_demosaic_dev((const float *)d_in, (float *)d_out, piece->roi_in.width, piece->roi_in.height, piece->roi_in.x, piece->roi_in.y, 9u,
                          &piece->xtrans[0][0], SLOT_TMP3, nullptr, (cudaStream_t)stream);
    if(rc) return rc;
    if(d->color_smoothing)
      rc = demosaic_color_smoothing_dev((float *)d_out, piece->roi_out.width, piece->roi_out.height, (int)d->color_smoothing, (cudaStream_t)stream);
    return rc;
  }
  if(d->green_eq > 3) return fail(B200_ERR_ARG, "demosaic: green_eq %u", d->green_eq);
  // roi_out has the size of roi_in with origin 0 for the full demosaicers (demosaic.c:1052-1054)
  if(piece->roi_out.width != piece->roi_in.width || piece->roi_out.height != piece->roi_in.height)
    return fail(B200_ERR_UNSUPPORTED, "demosaic: roi_out %dx%d != roi_in %dx%d (downsampling paths are not built)",
                piece->roi_out.width, piece->roi_out.height, piece->roi_in.width, piece->roi_in.height);

  const uint32_t method = d->demosaicing_method & ~(uint32_t)DEMOSAIC_DUAL;
  const bool dual = (d->demosaicing_method & DEMOSAIC_DUAL) != 0;
  if(method != B200_DEMOSAIC_RCD && method != B200_DEMOSAIC_AMAZE && method != B200_DEMOSAIC_PPG && method != B200_DEMOSAIC_VNG4 && method != B200_DEMOSAIC_LMMSE)
    return fail(B200_ERR_UNSUPPORTED, "demosaic: method %u is not built", d->demosaicing_method);
  if(dual && method != B200_DEMOSAIC_RCD && method != B200_DEMOSAIC_AMAZE)
    return fail(B200_ERR_UNSUPPORTED, "demosaic: dual demosaic is RCD + VNG4 or AMaZE + VNG4 (method %u)", d->demosaicing_method);
  const int width = piece->roi_in.width, height = piece->roi_in.height;
  cudaStream_t s = (cudaStream_t)stream;
  const float *mosaic = (const float *)d_in;
  // a four-colour Bayer sensor (CYGM, RGBE) skips green equilibration and runs VNG whatever the method (demosaic.c:1137, :1173)
  const bool four = (piece->image_flags & DT_IMAGE_4BAYER) != 0;
  if(!four && d->green_eq != 0)
  { // demosaic.c:1137-1170: the equalised mosaic replaces the input of the demosaicer
    const size_t n = (size_t)width * height;
    void *t0 = nullptr, *t1 = nullptr, *pd = nullptr;
    if((rc = scratch(SLOT_TMP0, n * sizeof(float), &t0))) return rc;
    if((rc = scratch(SLOT_TMP1, n * sizeof(float), &t1))) return rc;
    if((rc = scratch(SLOT_SMALL, (size_t)demosaic_green_eq_partial_doubles() * sizeof(double), &pd))) return rc;
    const float threshold = 0.0001f * piece->exif_iso; // :1049
    if((rc = demosaic_green_eq_dev(mosaic, (float *)t0, (float *)t1, (double *)pd, width, height, piece->filters, piece->roi_in.x, piece->roi_in.y,
                                   d->green_eq, threshold, &mosaic, s)))
      return rc;
  }
  if(method == B200_DEMOSAIC_VNG4 || four) // demosaic.c:1172-1183, then data->CAM_to_RGB on a four-colour sensor
    rc = vng_demosaic_dev(mosaic, (float *)d_out, width, height, piece->roi_in.x, piece->roi_in.y, piece->filters, nullptr, SLOT_TMP3,
                          four ? d->CAM_to_RGB : nullptr, s);
  else if(method == B200_DEMOSAIC_PPG)
    rc = ppg_demosaic_dev(mosaic, (float *)d_out, width, height, filters, d->median_thrs, s); // demosaic.c:1218-1226
  else if(method == B200_DEMOSAIC_LMMSE)
    rc = lmmse_demosaic_dev(mosaic, (float *)d_out, width, height, filters, (int)d->lmmse_refine, piece->processed_maximum, s); // demosaic.c:1189-1216
  else if(method == B200_DEMOSAIC_AMAZE)
    rc = amaze_demosaic_dev(mosaic, (float *)d_out, width, height, filters, piece->processed_maximum, s); // demosaic.c:1227
  else
    rc = rcd_demosaic_dev(mosaic, (float *)d_out, width, height, filters, piece->processed_maximum, s);
  if(rc) return rc;
  // demosaic.c:1243-1247: the blend reads the module's own input (not the green-equilibrated copy) and the sensor's filters word; on a
  // four-colour sensor its VNG frame is not converted by CAM_to_RGB, as in the reference
  if(dual && (rc = dual_demosaic_dev((float *)d_out, (const float *)d_in, width, height, piece->roi_in.x, piece->roi_in.y, piece->filters, nullptr,
                                     piece->wb_coeffs, d->dual_thrs, s)))
    return rc;
  if(d->color_smoothing) rc = demosaic_color_smoothing_dev((float *)d_out, piece->roi_out.width, piece->roi_out.height, (int)d->color_smoothing, s); // :1249-1250
  return rc;
}

extern "C" int b200_demosaic_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_piece(piece, in, out);
  if(rc) return rc;
  // The caller's cacheline may hold anything; the reference leaves the alpha of the outer 3 px
  // and (for frames under 16 px) the whole buffer as found.  Start from the caller's bytes only
  // in the too-small case and for PPG (which, like the reference, keeps the alpha of the outer three pixels);
  // otherwise every pixel is overwritten.
  const bool carry_out = piece->roi_in.width < 16 || piece->roi_in.height < 16
                         || keeps_alpha(((const b200_demosaic_data_t *)piece->data)->demosaicing_method);
  return through_device(piece, in, (size_t)piece->roi_in.width * piece->roi_in.height * sizeof(float), out,
                        (size_t)piece->roi_out.width * piece->roi_out.height * 4 * sizeof(float), carry_out, b200_demosaic_process_dev);
}

// tiling_callback(), iop/demosaic.c:1916-2013 (Bayer branches for the methods built here)
extern "C" void b200_demosaic_tiling(const b200_piece_t *piece, b200_tiling_t *tiling)
{
  if(!piece || !tiling || !piece->data) return;
  const b200_demosaic_data_t *d = (const b200_demosaic_data_t *)piece->data;
  const float ioratio = (float)piece->roi_out.width * piece->roi_out.height
                        / ((float)piece->roi_in.width * piece->roi_in.height);
  const float smooth = d->color_smoothing ? ioratio : 0.0f;
  const float greeneq = ((piece->filters != 9u) && (d->green_eq != 0)) ? 0.25f : 0.0f;
  const uint32_t method = d->demosaicing_method & ~DEMOSAIC_DUAL;

  tiling->factor = 1.0f + ioratio;
  tiling->factor += fmaxf(1.0f + greeneq, smooth);
  tiling->factor_cl = tiling->factor;
  tiling->maxbuf = 1.0f;
  tiling->maxbuf_cl = 1.0f;
  tiling->overhead = 0;
  if(method == 7u)
  { // DT_IOP_DEMOSAIC_DOWNSAMPLE, :1928-1936
    tiling->factor = 1.0f + ioratio + (d->color_smoothing ? 7.0f * ioratio : 0.0f);
    tiling->factor_cl = tiling->factor;
    tiling->xalign = 1;
    tiling->yalign = 1;
    tiling->overlap = (piece->filters == 9u) ? 18 : 16;
    return;
  }
  if(method == B200_DEMOSAIC_RCD)
  {
    // the CPU figure counts per-thread tile scratch; the device keeps its tiles in shared memory
    tiling->xalign = 2;
    tiling->yalign = 2;
    tiling->overlap = 10;
    tiling->factor_cl = tiling->factor; // no full-frame temporaries on the device (reference: +3, rcd.c:671-686)
  }
  else if(method == B200_DEMOSAIC_LMMSE)
  { // :1983-1993
    tiling->xalign = 2;
    tiling->yalign = 2;
    tiling->overlap = 10;
  }
  else if(method == B200_DEMOSAIC_AMAZE || method == B200_DEMOSAIC_PPG || method == 3u || method == 4u)
  { // PPG, the passthrough methods, AMaZE :1937-1950
    tiling->xalign = 2;
    tiling->yalign = 2;
    tiling->overlap = 5;
  }
  else if(method == 1025u || method == 1026u || method == 1028u)
  { // Markesteijn (1 and 3 passes) and FDC, :1951-1971: the per-thread tile buffers counted in units of the frame
    const int ndir = method == 1026u ? 8 : 4;
    tiling->factor = 1.0f + ioratio;
    tiling->factor += ndir * 1.0f + ndir * 0.25f + ndir * 0.125f + 1.0f;
    tiling->factor += fmaxf(1.0f + greeneq, smooth);
    tiling->factor_cl = 1.0f + ioratio + fmaxf(1.0f + greeneq, smooth); // the device keeps its tiles in per-CTA scratch, not per frame
    tiling->xalign = 6; // XTRANS_SNAPPER, :116
    tiling->yalign = 6;
    tiling->overlap = method == 1026u ? 18 : 12;
  }
  else
  {
    tiling->xalign = 6;
    tiling->yalign = 6;
    tiling->overlap = 6;
  }
  if(d->demosaicing_method & DEMOSAIC_DUAL)
  {
    tiling->factor += 1.0f;
    tiling->xalign = tiling->xalign > 6 ? tiling->xalign : 6;
    tiling->yalign = tiling->yalign > 6 ? tiling->yalign : 6;
    tiling->overlap = tiling->overlap > 6 ? tiling->overlap : 6;
  }
}
