// Internal runtime of libb200iop.so: error reporting, device binding, per-thread device scratch.
// Stands where the reference's OpenCL runtime does (src/common/opencl.c: dt_opencl_*), sized for
// one process driving 1..8 B200s.  Nothing here is visible through include/b200iop.h.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <functional>
#include "../../include/b200iop.h"

namespace b200
{
// thread-local last-error text (b200_last_error)
void set_error(const char *fmt, ...);
int fail(int code, const char *fmt, ...);

#define B200_CUDA_TRY(expr)                                                                       \
  do                                                                                              \
  {                                                                                               \
    cudaError_t _e = (expr);                                                                      \
    if(_e != cudaSuccess)                                                                         \
      return ::b200::fail(B200_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr,             \
                          cudaGetErrorString(_e));                                                \
  } while(0)

// Select the device a piece asks for (pipe->devid analogue); < 0 keeps the current device.
int bind_device(int devid);
int sm_count();

// Grow-only device scratch owned by the calling thread on the current device.  `slot` names an
// independent buffer (modules needing several temporaries use several slots).  Freed by
// b200_shutdown() or thread exit.  This is the shim's own device scratch, the counterpart of
// dt_opencl_alloc_device_buffer(); host-side tiling accounting never sees it (SURVEY 8b).
int scratch(int slot, size_t bytes, void **ptr);
enum
{
  SLOT_IN = 0,
  SLOT_OUT = 1,
  SLOT_TMP0 = 2,
  SLOT_TMP1 = 3,
  SLOT_TMP2 = 4,
  SLOT_TMP3 = 5,
  SLOT_SMALL = 6,
  SLOT_COUNT = 12
};

// Host <-> device transfer for the process() (host pointer) entry points.  Pinned or registered
// host memory goes straight over PCIe; pageable memory is staged through two pinned buffers so
// the copy into staging overlaps the DMA.
int copy_h2d(void *dst, const void *src, size_t bytes, cudaStream_t stream);
int copy_d2h(void *dst, const void *src, size_t bytes, cudaStream_t stream);

// per-thread non-blocking stream used by the *_process_host entry points
int host_stream(cudaStream_t *s);

// The body of every b200_<op>_process_host(), run after the module has checked its arguments: bind the device, upload
// `in_bytes` of `in` (and, with carry_out, the caller's `out` too, for modules that leave part of their output as they find
// it), run the module's _dev entry on the thread's host stream, download `out_bytes` into `out` and synchronise.  `out` is
// not written unless the _dev entry succeeded.
typedef int (*dev_fn)(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream);
int through_device(const b200_piece_t *piece, const void *in, size_t in_bytes, void *out, size_t out_bytes, bool carry_out, dev_fn fn);
// the same for an entry point without a piece: `run` gets the device buffers and the stream
int through_device(int devid, const void *in, size_t in_bytes, void *out, size_t out_bytes, bool carry_out,
                   const std::function<int(const void *d_in, void *d_out, void *stream)> &run);

// default_tiling_callback(), develop/tiling.c:1423-1463, for the modules that declare no tiling callback: factor 1 + the
// roi_out / roi_in area ratio, no overhead; `overlap` 4 for IOP_FLAGS_TILING_FULL_ROI, else 0; `raw` (placed before
// demosaic) aligns tiles on the mosaic's pattern, 2 px on Bayer sensors and 3 on X-Trans.
void default_tiling(const b200_piece_t *piece, b200_tiling_t *t, unsigned overlap, bool raw);

// Launch timing of the headline kernels (b200_kernel_timing, b200_kernel_timing_read): when enabled, a pair of CUDA
// events brackets the launch on the stream it goes to.  One `if` per launch when disabled.
enum
{
  TIMED_NLM = 0,
  TIMED_RCD = 1,
  TIMED_COUNT = 2
};
bool timing_enabled();
void timing_mark(int which, bool end, cudaStream_t stream);
struct timed_launch
{ // brackets the statement(s) between construction and destruction
  int which;
  cudaStream_t stream;
  bool on;
  timed_launch(int w, cudaStream_t s) : which(w), stream(s), on(timing_enabled())
  {
    if(on) timing_mark(which, false, stream);
  }
  ~timed_launch()
  {
    if(on) timing_mark(which, true, stream);
  }
};

// Device copy of three tone curves (3 * B200_LUT_SAMPLES floats), cached per device by `identity` and `side`
// (0 = decoding / source, 1 = encoding / target); identity 0 = upload every time.  color.cu.
int device_curves(const float *const host[3], uint64_t identity, int side, cudaStream_t stream, const float **out);
} // namespace b200
