/* oracle/_ref wrapper: lens correction, built into oracle/_ref/libref_lens_{strict,fast}.so by oracle/lens.mk.  TEST INFRASTRUCTURE ONLY.
 *
 * oracle/lens.mk cuts verbatim out of iop/lens.c the correction enums (:121-167), dt_iop_lensfun_data_t (:392-409), get_modifier
 * (:620-653) and process() (:680-923), and out of pixel/interpolation.c / .h the interpolators, their table, the tap and border helpers,
 * dt_interpolation_compute_sample and dt_interpolation_new.  LensSerious's src/lensserious.c is compiled unmodified beside this file.
 * The operator-surface types carry the members those lines read; dt_conf answers the warp interpolator the caller names.
 * __DT_CLONE_TARGETS__ is empty, so the release build is the x86-64-v2 one. */
#include <glib.h>
#include <math.h>
#include <float.h>
#include <string.h>
#include <stdlib.h>
#include <stdint.h>
#include <assert.h>
#include <sys/types.h>
#include "system/macros.h"
#include "system/openmp.h"
#define __DT_CLONE_TARGETS__
#include "system/simd.h"
#include "math/math.h"
#include "pixel/format.h"
#include "lensserious.h"

#define DT_DEV_PIXELPIPE_DISPLAY_MASK 1 /* develop/develop.h:123 */
#define DT_MODULE_INTROSPECTION(version, params)
#define dt_pthread_mutex_lock(m) ((void)0)
#define dt_pthread_mutex_unlock(m) ((void)0)
#define dt_plugin_threadsafe_mutex() NULL
#define dt_print(...) ((void)0)
#ifndef MIN
#define MIN(a, b) (((a) < (b)) ? (a) : (b))
#define MAX(a, b) (((a) > (b)) ? (a) : (b))
#endif
#define DT_IMAGE_MONOCHROME (1 << 15)       /* common/image.h:141 */
#define DT_IMAGE_MONOCHROME_BAYER (1 << 19) /* common/image.h:150 */

typedef struct dt_image_t { uint32_t flags; } dt_image_t;
typedef struct dt_develop_t { dt_image_t image_storage; } dt_develop_t;
typedef struct dt_iop_module_t { dt_develop_t *dev; } dt_iop_module_t;
typedef struct dt_dev_pixelpipe_t { int mask_display; } dt_dev_pixelpipe_t;
typedef struct dt_dev_pixelpipe_iop_t
{
  void *data;
  dt_iop_roi_t buf_in, roi_in, roi_out;
  dt_iop_buffer_dsc_t dsc_in;
} dt_dev_pixelpipe_iop_t;
/* common/image.c:183-186 */
static gboolean dt_image_is_monochrome(const dt_image_t *img) { return (img->flags & (DT_IMAGE_MONOCHROME | DT_IMAGE_MONOCHROME_BAYER)) ? TRUE : FALSE; }
/* common/imagebuf.c dt_iop_image_copy: a copy of nfloats */
static inline void dt_iop_image_copy_by_size(float *const out, const float *const in, const size_t width, const size_t height, const size_t ch)
{
  memcpy(out, in, sizeof(float) * width * height * ch);
}
/* caches/pixelpipe_cache_alloc.h:141-153: one buffer of n floats per OpenMP thread */
static float *dt_pixelpipe_cache_alloc_perthread_float(const size_t n, size_t *padded)
{
  *padded = (n + 15) & ~(size_t)15;
  return aligned_alloc(64, sizeof(float) * *padded * omp_get_max_threads());
}
#define dt_get_perthread(buf, padsize) ((buf) + ((padsize) * dt_get_thread_num()))
#define dt_pixelpipe_cache_free_align(p) free(p)

static const char *ref_warp_interpolator = "mitchell";
static const char *dt_conf_get_string_const(const char *key) { return ref_warp_interpolator; }

#include "gen_lens_interpolation.c"
#include "gen_lens.c"

/* process() on roi_in -> roi_out RGBA; interpolator: "bilinear", "bicubic" or "mitchell" */
int ref_lens(const float *in, float *out, const void *data, const char *interpolator, int monochrome, int mask_display, int in_x, int in_y, int in_w,
             int in_h, double in_scale, int out_x, int out_y, int out_w, int out_h, int buf_in_w, int buf_in_h)
{
  ref_warp_interpolator = interpolator;
  dt_develop_t dev = { { monochrome ? DT_IMAGE_MONOCHROME : 0u } };
  dt_iop_module_t self = { &dev };
  dt_dev_pixelpipe_t pipe = { mask_display };
  dt_dev_pixelpipe_iop_t piece;
  memset(&piece, 0, sizeof(piece));
  piece.data = (void *)data;
  piece.buf_in = (dt_iop_roi_t){ 0, 0, buf_in_w, buf_in_h, 1.0 };
  piece.roi_in = (dt_iop_roi_t){ in_x, in_y, in_w, in_h, in_scale };
  piece.roi_out = (dt_iop_roi_t){ out_x, out_y, out_w, out_h, in_scale };
  piece.dsc_in.channels = 4;
  return process(&self, &pipe, &piece, in, out);
}

/* get_modifier(.., used_lf_mask, FALSE, ..) + ls_eval_from_modifier, as process() resolves its plan */
int ref_lens_plan(const void *data, int w, int h, int monochrome, int *modflags, ls_eval_t *eval)
{
  ls_modifier_t mod;
  const int mask = monochrome ? DT_LENS_MODIFY_ALL & ~DT_LENS_MODIFY_TCA : DT_LENS_MODIFY_ALL;
  get_modifier(modflags, w, h, (const dt_iop_lensfun_data_t *)data, mask, FALSE, &mod);
  ls_eval_from_modifier(&mod, eval);
  return 0;
}

size_t ref_lens_sizeof(int which)
{
  switch(which)
  {
    case 0: return sizeof(dt_iop_lensfun_data_t);
    case 1: return sizeof(ls_lens_t);
    case 2: return offsetof(dt_iop_lensfun_data_t, ls_lens);
    case 3: return offsetof(dt_iop_lensfun_data_t, ls_have);
    case 4: return offsetof(ls_lens_t, n_tca);
    case 5: return offsetof(ls_lens_t, n_vig);
    case 6: return offsetof(ls_lens_t, n_real_focal);
    default: return sizeof(ls_eval_t);
  }
}
