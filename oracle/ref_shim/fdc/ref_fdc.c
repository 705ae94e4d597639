/* oracle/_ref wrapper: frequency-domain chroma (FDC) for X-Trans sensors, built into oracle/_ref/libref_fdc_{strict,fast}.so by
 * oracle/fdc.mk.  TEST INFRASTRUCTURE ONLY.
 *
 * oracle/fdc.mk cuts verbatim out of iop/demosaic/markesteijn.c SQR (:25-26), hexmap (:29-40) and xtrans_fdc_interpolate (:525-1639),
 * and out of develop/imageop_math.h FCxtrans (:175-219).  Around those lines this file supplies:
 *   - the operator-surface types with the one member the lines read (self->dev->image_storage.exif_iso, a float as in
 *     common/image.h:342) and dt_conf_get_int, which answers the crossover ISO the caller names;
 *   - glib's ABS (gmacros.h), which is what the module's translation unit resolves ABS to;
 *   - the per-thread scratch allocator.  It fills every byte of every thread's buffer with a pattern the caller chooses, so that
 *     what the reference reads from bytes it never wrote this tile is a function of that pattern, not of the heap.
 * The lines run with FTZ|DAZ set, as the pipe's threads do (darktable.c:877, common/dtpthread.c:54).  __DT_CLONE_TARGETS__ is empty,
 * so the release build is the x86-64-v2 one. */
#include <glib.h>
#include <math.h>
#include <float.h>
#include <string.h>
#include <stdlib.h>
#include <stdint.h>
#include <assert.h>
#include <complex.h>
#include <xmmintrin.h>
#include "system/macros.h"
#include "system/openmp.h"
#define __DT_CLONE_TARGETS__
#include "system/simd.h"
#include "math/math.h"
#include "pixel/format.h"
#include "gen_fdc_imageop_math.c"

#ifndef ABS
#define ABS(a) (((a) < 0) ? -(a) : (a)) /* glib/gmacros.h */
#endif

typedef struct dt_image_t { float exif_iso; } dt_image_t;
typedef struct dt_develop_t { dt_image_t image_storage; } dt_develop_t;
typedef struct dt_iop_module_t { dt_develop_t *dev; } dt_iop_module_t;

static int ref_xover_iso = 1600;
static int dt_conf_get_int(const char *key) { (void)key; return ref_xover_iso; }

static int ref_fill = 0;
static void *dt_pixelpipe_cache_alloc_perthread(const size_t n, const size_t objsize, size_t *padded)
{
  *padded = (n * objsize + 63) & ~(size_t)63;
  void *p = aligned_alloc(64, *padded * omp_get_max_threads());
  if(p) memset(p, ref_fill, *padded * omp_get_max_threads());
  return p;
}
#undef dt_get_perthread
#define dt_get_perthread(buf, padsize) ((buf) + ((padsize) * dt_get_thread_num()))
#define dt_pixelpipe_cache_free_align(p) free(p)

#include "gen_fdc.c"

/* in: the X-Trans mosaic of the region (width x height floats), (x, y): its origin on the sensor, iso: the image's exif_iso,
 * xover_iso: the preference plugins/darkroom/demosaic/fdc_xover_iso, fill: the byte every scratch byte starts as, nthreads: OpenMP
 * threads over the rows of tiles.  out: 4 floats per pixel, lane 3 untouched. */
void ref_fdc(float *out, const float *in, int width, int height, int x, int y, const uint8_t xtrans[36], float iso, int xover_iso, int fill,
             int nthreads)
{
  const dt_iop_roi_t roi_in = { x, y, width, height, 1.0 }, roi_out = { 0, 0, width, height, 1.0 };
  dt_develop_t dev = { { iso } };
  dt_iop_module_t self = { &dev };
  ref_xover_iso = xover_iso;
  ref_fill = fill;
  const unsigned csr = _mm_getcsr();
  const int threads = omp_get_max_threads();
  omp_set_num_threads(nthreads);
  _mm_setcsr(csr | 0x8040u);
  xtrans_fdc_interpolate(&self, out, in, &roi_out, &roi_in, (const uint8_t(*)[6])xtrans);
  _mm_setcsr(csr);
  omp_set_num_threads(threads);
}

/* the reference's coefficient tables (markesteijn.c:548-1071) as the compiler laid them out: Minv[3][8], modarr[6][6][8], harr[4][13][13]
 * complex floats, re/im interleaved */
void ref_fdc_tables(float *minv, float *mod, float *harr_out)
{
#include "gen_fdc_tables.c"
  memcpy(minv, Minv, sizeof(Minv));
  memcpy(mod, modarr, sizeof(modarr));
  memcpy(harr_out, harr, sizeof(harr));
}
