/* oracle/_ref wrapper: colour balance rgb, built into oracle/_ref/libref_colorbalancergb_{strict,fast}.so by oracle/colorbalancergb.mk.
 * TEST INFRASTRUCTURE ONLY.
 *
 * oracle/colorbalancergb.mk cuts verbatim out of iop/colorbalancergb.c LUT_ELEM, STEPS and DEG_TO_RAD (:70-78), the enums, the params, GUI and data
 * structs (:82-192), opacity_masks / soft_clip / lookup_gamut / process() (:509-927) and Delta_H + commit_params() (:1096-1353).
 * common/colorspaces_inline_conversions.h, math/matrices.h, system/simd.h, math/math.h, pixel/chromatic_adaptation.h (the CAT16 matrices)
 * and pixel/format.h are the reference's, unmodified.
 * The operator-surface types carry the members those lines read; the work profile is the caller's two matrices (or NULL); the GUI's
 * mask settings and the checkerboard preferences are the caller's.  commit_params() runs serially (no OpenMP in this wrapper's
 * calls of it: the LUT march writes entries from several iterations).  __DT_CLONE_TARGETS__ is empty, so the release build is the
 * x86-64-v2 one. */
#include <glib.h>
#include <gtk/gtk.h>
#include <math.h>
#include <float.h>
#include <string.h>
#include <stdlib.h>
#include <stdint.h>
#include <stddef.h>
#include <omp.h>
#include "system/macros.h"
#include "system/openmp.h"
#define __DT_CLONE_TARGETS__
#include "system/simd.h"
#include "math/math.h"
#include "math/matrices.h"
#include "common/colorspaces_inline_conversions.h"
#include "pixel/chromatic_adaptation.h"
#include "pixel/format.h"

#define DT_MODULE_INTROSPECTION(version, params)
#define DT_PIXEL_APPLY_DPI(x) (x)
typedef void dt_iop_params_t;
typedef enum { DT_DEV_PIXELPIPE_NONE = 0, DT_DEV_PIXELPIPE_EXPORT = 1, DT_DEV_PIXELPIPE_FULL = 2 } dt_dev_pixelpipe_type_t;
typedef struct dt_iop_order_iccprofile_info_t { dt_colormatrix_t matrix_in, matrix_out; } dt_iop_order_iccprofile_info_t;
typedef struct dt_develop_t { int gui_attached; } dt_develop_t;
typedef struct dt_iop_module_t { dt_develop_t *dev; void *gui_data; } dt_iop_module_t;
typedef struct dt_dev_pixelpipe_t { dt_dev_pixelpipe_type_t type; struct dt_iop_order_iccprofile_info_t *work; } dt_dev_pixelpipe_t;
typedef struct dt_dev_pixelpipe_iop_t { void *data; dt_iop_roi_t roi_out; } dt_dev_pixelpipe_iop_t;
static inline struct dt_iop_order_iccprofile_info_t *dt_ioppr_get_pipe_current_profile_info(dt_iop_module_t *self, const dt_dev_pixelpipe_t *pipe)
{
  return pipe->work;
}
#define dt_iop_gui_data(self) ((self)->gui_data)
#define dt_alloc_align_float(n) ((float *)aligned_alloc(64, sizeof(float) * (n)))
#define dt_free_align(p) free(p)
/* the darkroom preferences commit_params() copies into the data block (plugins/darkroom/colorbalancergb/...) */
static float ref_conf_float = 0.5f;
static int ref_conf_int = 8, ref_conf_bool = 0;
static float dt_conf_get_float(const char *key) { return ref_conf_float; }
static int dt_conf_get_int(const char *key) { return ref_conf_int; }
static int dt_conf_get_bool(const char *key) { return ref_conf_bool; }

#include "gen_colorbalancergb.c"

static dt_iop_order_iccprofile_info_t *profile(const float *rgb_to_xyz, const float *xyz_to_rgb, dt_iop_order_iccprofile_info_t *w)
{
  if(!rgb_to_xyz) return NULL;
  memset(w, 0, sizeof(*w));
  for(int r = 0; r < 3; r++)
    for(int c = 0; c < 3; c++)
    {
      w->matrix_in[r][c] = rgb_to_xyz[3 * r + c];
      w->matrix_out[r][c] = xyz_to_rgb[3 * r + c];
    }
  return w;
}

/* commit_params() on one params block into *data (the hashed prefix) and lut[360].  rgb_to_xyz / xyz_to_rgb: row-major 3x3 of the work
 * profile, or NULL for no profile.  lut_fill: what the 360 floats hold before the call (init_pipe's allocation is not zeroed).
 * mask_display / mask_type: the GUI state a FULL pipe with a GUI reads. */
void ref_colorbalancergb_commit(const void *params, void *data, float *lut, const float *rgb_to_xyz, const float *xyz_to_rgb, float lut_fill,
                                int mask_display, int mask_type)
{
  dt_iop_colorbalancergb_data_t *d = aligned_alloc(64, 256 * ((sizeof(*d) + 255) / 256));
  memset(d, 0, sizeof(*d));
  d->gamut_LUT = dt_alloc_align_float(LUT_ELEM);
  for(int k = 0; k < LUT_ELEM; k++) d->gamut_LUT[k] = lut_fill;
  dt_iop_colorbalancergb_gui_data_t gui;
  memset(&gui, 0, sizeof(gui));
  gui.mask_display = mask_display;
  gui.mask_type = mask_type;
  dt_develop_t dev = { 1 };
  dt_iop_module_t self = { &dev, mask_display ? &gui : NULL };
  dt_iop_order_iccprofile_info_t w;
  dt_dev_pixelpipe_t pipe = { mask_display ? DT_DEV_PIXELPIPE_FULL : DT_DEV_PIXELPIPE_EXPORT, profile(rgb_to_xyz, xyz_to_rgb, &w) };
  dt_dev_pixelpipe_iop_t piece = { d };
  dt_iop_colorbalancergb_params_t p;
  memcpy(&p, params, sizeof(p));
  const int threads = omp_get_max_threads();
  omp_set_num_threads(1);
  commit_params(&self, (dt_iop_params_t *)&p, &pipe, &piece);
  omp_set_num_threads(threads);
  memcpy(data, d, offsetof(dt_iop_colorbalancergb_data_t, work_profile));
  memcpy(lut, d->gamut_LUT, sizeof(float) * LUT_ELEM);
  free(d->gamut_LUT);
  free(d);
}

/* process() over npixels RGBA floats with the data prefix and the LUT the caller gives (the mask display needs width for the checker) */
int ref_colorbalancergb(const float *in, float *out, int width, int height, const void *data, const float *lut, const float *rgb_to_xyz,
                        const float *xyz_to_rgb)
{
  dt_iop_colorbalancergb_data_t *d = aligned_alloc(64, 256 * ((sizeof(*d) + 255) / 256));
  memset(d, 0, sizeof(*d));
  memcpy(d, data, offsetof(dt_iop_colorbalancergb_data_t, work_profile));
  d->gamut_LUT = dt_alloc_align_float(LUT_ELEM);
  memcpy(d->gamut_LUT, lut, sizeof(float) * LUT_ELEM);
  dt_develop_t dev = { 0 };
  dt_iop_module_t self = { &dev, NULL };
  dt_iop_order_iccprofile_info_t w;
  dt_dev_pixelpipe_t pipe = { DT_DEV_PIXELPIPE_EXPORT, profile(rgb_to_xyz, xyz_to_rgb, &w) };
  dt_dev_pixelpipe_iop_t piece = { d, { 0, 0, width, height, 1.0 } };
  const int rc = process(&self, &pipe, &piece, in, out);
  free(d->gamut_LUT);
  free(d);
  return rc;
}

size_t ref_colorbalancergb_layout(int which)
{
  switch(which)
  {
    case 0: return offsetof(dt_iop_colorbalancergb_data_t, work_profile);
    case 1: return offsetof(dt_iop_colorbalancergb_data_t, midtones_Y);
    case 2: return offsetof(dt_iop_colorbalancergb_data_t, chroma);
    case 3: return offsetof(dt_iop_colorbalancergb_data_t, saturation);
    case 4: return offsetof(dt_iop_colorbalancergb_data_t, brilliance);
    case 5: return offsetof(dt_iop_colorbalancergb_data_t, hue_angle);
    case 6: return offsetof(dt_iop_colorbalancergb_data_t, white_fulcrum);
    case 7: return offsetof(dt_iop_colorbalancergb_data_t, checker_color_1);
    case 8: return offsetof(dt_iop_colorbalancergb_data_t, saturation_formula);
    case 9: return offsetof(dt_iop_colorbalancergb_data_t, checker_size);
    case 10: return offsetof(dt_iop_colorbalancergb_data_t, mask_display);
    case 11: return offsetof(dt_iop_colorbalancergb_data_t, lut_inited);
    case 12: return sizeof(dt_iop_colorbalancergb_params_t);
    default: return sizeof(dt_iop_colorbalancergb_data_t);
  }
}
