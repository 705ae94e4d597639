// libb200iop.so runtime: errors, device binding, per-thread scratch, host<->device staging, the host entries' round trip, the
// default tiling callback.
// Counterpart of the reference's OpenCL runtime (src/common/opencl.c) for CUDA on H100.
#include "runtime.h"
#include <vector>
#include <string.h>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>

namespace b200
{
static thread_local char tls_error[512] = "";
static std::atomic<int> g_ndev{ -1 }; // -1 = not initialised
static std::atomic<bool> g_alive{ false };
static int g_sm_count[16];

void set_error(const char *fmt, ...)
{
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(tls_error, sizeof(tls_error), fmt, ap);
  va_end(ap);
}

int fail(int code, const char *fmt, ...)
{
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(tls_error, sizeof(tls_error), fmt, ap);
  va_end(ap);
  return code;
}

static int ensure_init()
{
  if(g_ndev.load() >= 0) return g_ndev.load() > 0 ? B200_OK : fail(B200_ERR_NODEVICE, "no CUDA device");
  return b200_init(0);
}

int bind_device(int devid)
{
  int rc = ensure_init();
  if(rc) return rc;
  if(devid < 0) return B200_OK;
  if(devid >= g_ndev.load()) return fail(B200_ERR_ARG, "devid %d out of range (%d devices bound)", devid, g_ndev.load());
  B200_CUDA_TRY(cudaSetDevice(devid));
  return B200_OK;
}

int sm_count()
{
  int dev = 0;
  if(cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return 132;
  return g_sm_count[dev] > 0 ? g_sm_count[dev] : 132;
}

// ---- per-thread state -------------------------------------------------------------------
struct thread_state_t
{
  void *buf[16][SLOT_COUNT];
  size_t cap[16][SLOT_COUNT];
  cudaStream_t stream[16];
  void *pinned[2];
  size_t pinned_cap;
  cudaEvent_t pinned_ev[2];
  bool pinned_ev_ok;

  thread_state_t()
  {
    memset(buf, 0, sizeof(buf));
    memset(cap, 0, sizeof(cap));
    memset(stream, 0, sizeof(stream));
    pinned[0] = pinned[1] = nullptr;
    pinned_cap = 0;
    pinned_ev_ok = false;
  }
  void release()
  {
    if(!g_alive.load()) return; // the CUDA context may already be gone at process exit
    int cur = 0;
    cudaGetDevice(&cur);
    for(int d = 0; d < 16; d++)
    {
      bool any = stream[d] != nullptr;
      for(int s = 0; s < SLOT_COUNT; s++) any |= buf[d][s] != nullptr;
      if(!any) continue;
      cudaSetDevice(d);
      for(int s = 0; s < SLOT_COUNT; s++)
        if(buf[d][s])
        {
          cudaFree(buf[d][s]);
          buf[d][s] = nullptr;
          cap[d][s] = 0;
        }
      if(stream[d])
      {
        cudaStreamDestroy(stream[d]);
        stream[d] = nullptr;
      }
    }
    cudaSetDevice(cur);
    for(int k = 0; k < 2; k++)
      if(pinned[k])
      {
        cudaFreeHost(pinned[k]);
        pinned[k] = nullptr;
      }
    if(pinned_ev_ok)
    {
      cudaEventDestroy(pinned_ev[0]);
      cudaEventDestroy(pinned_ev[1]);
      pinned_ev_ok = false;
    }
    pinned_cap = 0;
  }
  ~thread_state_t() { release(); }
};
static thread_local thread_state_t tls;

int scratch(int slot, size_t bytes, void **ptr)
{
  if(slot < 0 || slot >= SLOT_COUNT) return fail(B200_ERR_ARG, "bad scratch slot %d", slot);
  int dev = 0;
  B200_CUDA_TRY(cudaGetDevice(&dev));
  if(dev >= 16) return fail(B200_ERR_ARG, "device ordinal %d too large", dev);
  if(tls.cap[dev][slot] < bytes)
  {
    if(tls.buf[dev][slot]) cudaFree(tls.buf[dev][slot]);
    tls.buf[dev][slot] = nullptr;
    tls.cap[dev][slot] = 0;
    const size_t want = (bytes + (size_t(1) << 20) - 1) & ~((size_t(1) << 20) - 1);
    cudaError_t e = cudaMalloc(&tls.buf[dev][slot], want);
    if(e != cudaSuccess)
    {
      tls.buf[dev][slot] = nullptr;
      return fail(B200_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
    }
    tls.cap[dev][slot] = want;
  }
  *ptr = tls.buf[dev][slot];
  return B200_OK;
}

int host_stream(cudaStream_t *s)
{
  int dev = 0;
  B200_CUDA_TRY(cudaGetDevice(&dev));
  if(!tls.stream[dev]) B200_CUDA_TRY(cudaStreamCreateWithFlags(&tls.stream[dev], cudaStreamNonBlocking));
  *s = tls.stream[dev];
  return B200_OK;
}

static bool host_is_pinned(const void *p)
{
  cudaPointerAttributes a;
  if(cudaPointerGetAttributes(&a, p) != cudaSuccess)
  {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost;
}

static const size_t STAGE_BYTES = size_t(32) << 20;

static int ensure_staging()
{
  if(tls.pinned_cap) return B200_OK;
  for(int k = 0; k < 2; k++) B200_CUDA_TRY(cudaMallocHost(&tls.pinned[k], STAGE_BYTES));
  for(int k = 0; k < 2; k++) B200_CUDA_TRY(cudaEventCreateWithFlags(&tls.pinned_ev[k], cudaEventDisableTiming));
  tls.pinned_ev_ok = true;
  tls.pinned_cap = STAGE_BYTES;
  return B200_OK;
}

int copy_h2d(void *dst, const void *src, size_t bytes, cudaStream_t stream)
{
  if(!bytes) return B200_OK;
  if(host_is_pinned(src))
  {
    B200_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));
    return B200_OK;
  }
  int rc = ensure_staging();
  if(rc) return rc;
  size_t off = 0;
  int k = 0;
  bool used[2] = { false, false };
  while(off < bytes)
  {
    const size_t n = bytes - off < STAGE_BYTES ? bytes - off : STAGE_BYTES;
    if(used[k]) B200_CUDA_TRY(cudaEventSynchronize(tls.pinned_ev[k]));
    memcpy(tls.pinned[k], (const char *)src + off, n);
    B200_CUDA_TRY(cudaMemcpyAsync((char *)dst + off, tls.pinned[k], n, cudaMemcpyHostToDevice, stream));
    B200_CUDA_TRY(cudaEventRecord(tls.pinned_ev[k], stream));
    used[k] = true;
    off += n;
    k ^= 1;
  }
  // the staging buffers are reused by the next call: drain before returning
  B200_CUDA_TRY(cudaStreamSynchronize(stream));
  return B200_OK;
}

int copy_d2h(void *dst, const void *src, size_t bytes, cudaStream_t stream)
{
  if(!bytes) return B200_OK;
  if(host_is_pinned(dst))
  {
    B200_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, stream));
    return B200_OK;
  }
  int rc = ensure_staging();
  if(rc) return rc;
  size_t off = 0, done = 0;
  int k = 0;
  size_t pend_off[2] = { 0, 0 }, pend_n[2] = { 0, 0 };
  bool used[2] = { false, false };
  while(off < bytes || used[0] || used[1])
  {
    if(used[k])
    {
      B200_CUDA_TRY(cudaEventSynchronize(tls.pinned_ev[k]));
      memcpy((char *)dst + pend_off[k], tls.pinned[k], pend_n[k]);
      done += pend_n[k];
      used[k] = false;
    }
    if(off < bytes)
    {
      const size_t n = bytes - off < STAGE_BYTES ? bytes - off : STAGE_BYTES;
      B200_CUDA_TRY(cudaMemcpyAsync(tls.pinned[k], (const char *)src + off, n, cudaMemcpyDeviceToHost, stream));
      B200_CUDA_TRY(cudaEventRecord(tls.pinned_ev[k], stream));
      pend_off[k] = off;
      pend_n[k] = n;
      used[k] = true;
      off += n;
    }
    k ^= 1;
  }
  (void)done;
  return B200_OK;
}

int through_device(int devid, const void *in, size_t in_bytes, void *out, size_t out_bytes, bool carry_out,
                   const std::function<int(const void *d_in, void *d_out, void *stream)> &run)
{
  int rc = bind_device(devid);
  if(rc) return rc;
  void *d_in = nullptr, *d_out = nullptr;
  cudaStream_t s;
  if((rc = host_stream(&s))) return rc;
  if((rc = scratch(SLOT_IN, in_bytes, &d_in))) return rc;
  if((rc = scratch(SLOT_OUT, out_bytes, &d_out))) return rc;
  if((rc = copy_h2d(d_in, in, in_bytes, s))) return rc;
  if(carry_out && (rc = copy_h2d(d_out, out, out_bytes, s))) return rc;
  if((rc = run(d_in, d_out, (void *)s))) return rc;
  if((rc = copy_d2h(out, d_out, out_bytes, s))) return rc;
  B200_CUDA_TRY(cudaStreamSynchronize(s));
  return B200_OK;
}

int through_device(const b200_piece_t *piece, const void *in, size_t in_bytes, void *out, size_t out_bytes, bool carry_out, dev_fn fn)
{
  return through_device(piece->devid, in, in_bytes, out, out_bytes, carry_out,
                        [=](const void *d_in, void *d_out, void *stream) { return fn(piece, d_in, d_out, stream); });
}

void default_tiling(const b200_piece_t *piece, b200_tiling_t *t, unsigned overlap, bool raw)
{
  if(!piece || !t) return;
  const float ioratio = ((float)piece->roi_out.width * (float)piece->roi_out.height) / ((float)piece->roi_in.width * (float)piece->roi_in.height);
  t->factor = 1.0f + ioratio;
  t->factor_cl = t->factor;
  t->maxbuf = 1.0f;
  t->maxbuf_cl = 1.0f;
  t->overhead = 0;
  t->overlap = overlap;
  t->xalign = 1;
  t->yalign = 1;
  if(!raw || !piece->filters) return;
  t->xalign = t->yalign = (piece->filters == 9u) ? 3 : 2;
}
// ---- launch timing of the headline kernels ----------------------------------------------------------------
namespace
{
std::atomic<bool> g_timing(false);
std::mutex g_timing_mu;
struct timed_pair
{
  cudaEvent_t e0, e1;
};
std::vector<timed_pair> g_timed[TIMED_COUNT];
const char *const g_timed_names[TIMED_COUNT] = { "nlm_kernel", "rcd_tiles_kernel" } /* nlm_kernel: whichever non-local-means kernel the launcher picked (nlm_pipe_kernel for the bench frame) */;
} // namespace
bool timing_enabled() { return g_timing.load(std::memory_order_relaxed); }
void timing_mark(int which, bool end, cudaStream_t stream)
{
  std::lock_guard<std::mutex> lock(g_timing_mu);
  if(which < 0 || which >= TIMED_COUNT) return;
  if(!end)
  {
    timed_pair p = { nullptr, nullptr };
    if(cudaEventCreate(&p.e0) != cudaSuccess || cudaEventCreate(&p.e1) != cudaSuccess) return;
    cudaEventRecord(p.e0, stream);
    g_timed[which].push_back(p);
  }
  else if(!g_timed[which].empty())
    cudaEventRecord(g_timed[which].back().e1, stream);
}
} // namespace b200

// ---- exported C ABI ---------------------------------------------------------------------
using namespace b200;

extern "C" int b200_kernel_timing(int enable)
{
  std::lock_guard<std::mutex> lock(g_timing_mu);
  for(auto &v : g_timed)
  {
    for(auto &p : v)
    {
      cudaEventDestroy(p.e0);
      cudaEventDestroy(p.e1);
    }
    v.clear();
  }
  g_timing.store(enable != 0);
  return B200_OK;
}

extern "C" int b200_kernel_timing_read(const char *kernel, double *sum_ms, int *count)
{
  if(!kernel || !sum_ms || !count) return fail(B200_ERR_ARG, "kernel_timing_read: null argument");
  std::lock_guard<std::mutex> lock(g_timing_mu);
  for(int k = 0; k < TIMED_COUNT; k++)
    if(!strcmp(kernel, g_timed_names[k]))
    {
      double sum = 0.0;
      int n = 0;
      for(auto &p : g_timed[k])
      {
        float ms = 0.0f;
        if(cudaEventSynchronize(p.e1) != cudaSuccess || cudaEventElapsedTime(&ms, p.e0, p.e1) != cudaSuccess)
        {
          cudaGetLastError();
          continue;
        }
        sum += ms;
        n++;
      }
      *sum_ms = sum;
      *count = n;
      return B200_OK;
    }
  return fail(B200_ERR_ARG, "kernel_timing_read: no timed kernel named %s", kernel);
}

extern "C" int b200_abi_version(void) { return B200_ABI_VERSION; }

extern "C" const char *b200_last_error(void) { return tls_error; }

extern "C" int b200_init(int ndev)
{
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  if(g_ndev.load() > 0) return B200_OK;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if(e != cudaSuccess || n <= 0)
  {
    cudaGetLastError();
    g_ndev.store(0);
    return fail(B200_ERR_NODEVICE, "no CUDA device (%s); libb200iop has no CPU path",
                e == cudaSuccess ? "count 0" : cudaGetErrorString(e));
  }
  if(ndev > 0 && ndev < n) n = ndev;
  if(n > 16) n = 16;
  for(int d = 0; d < n; d++)
  {
    cudaDeviceProp prop;
    if(cudaGetDeviceProperties(&prop, d) != cudaSuccess) return fail(B200_ERR_CUDA, "cudaGetDeviceProperties(%d) failed", d);
    if(prop.major != 9 || prop.minor != 0)
    {
      g_ndev.store(0);
      return fail(B200_ERR_NODEVICE, "device %d (%s) is sm_%d%d; this library is built for sm_90a only", d,
                  prop.name, prop.major, prop.minor);
    }
    g_sm_count[d] = prop.multiProcessorCount;
  }
  g_ndev.store(n);
  g_alive.store(true);
  return B200_OK;
}

extern "C" void b200_shutdown(void)
{
  tls.release();
  g_alive.store(false);
  g_ndev.store(-1);
}

extern "C" int b200_device_count(void) { return g_ndev.load() > 0 ? g_ndev.load() : 0; }

// ---- integer CFA phase (bit-exact by construction) ----------------------------------------
// ColorFilterArray::shiftDcrawFilter, external/rawspeed/src/librawspeed/metadata/ColorFilterArray.cpp:143-170,
// reached through dt_dev_get_roi_filters (develop/imageop.c:139-142) and
// dt_rawspeed_crop_dcraw_filters (imageio/imageio_rawspeed.cc:146-151: 0 and 9 pass through).
extern "C" uint32_t b200_roi_filters(uint32_t filters, int roi_x, int roi_y)
{
  if(!filters || filters == 9u) return filters;
  // dt_rawspeed_crop_dcraw_filters takes uint32_t crops; the int conversion inside rawspeed
  // sees the same bit pattern, so negative ROI origins behave as they do upstream.
  int x = (int)(uint32_t)roi_x, y = (int)(uint32_t)roi_y;
  if((x < 0 ? -x : x) & 1)
  {
    // odd horizontal shift: swap the two 2-bit colours inside every nibble
    const uint32_t lo = filters & 0x33333333u, hi = filters & 0xCCCCCCCCu;
    filters = (lo << 2) | (hi >> 2);
  }
  if(y == 0) return filters;
  // vertical shift: rotate by 4 bits per row (rawspeed computes y *= 4 in int)
  const int yy = (int)((unsigned)y * 4u);
  const int s = yy >= 0 ? yy % 32 : (int)(32 - ((-(long long)yy) % 32));
  if(s != 0 && s != 32) filters = (filters >> s) | (filters << (32 - s));
  return filters;
}

extern "C" int b200_fc(int row, int col, uint32_t filters)
{
  return (int)((filters >> (((((unsigned)row << 1) & 14u) + ((unsigned)col & 1u)) << 1)) & 3u);
}

// ---- device memory for resident chains (dt_opencl_alloc_device / copy_* analogues) ---------
extern "C" int b200_dev_alloc(void **ptr, size_t bytes)
{
  if(!ptr) return fail(B200_ERR_ARG, "dev_alloc: NULL");
  int rc = bind_device(-1);
  if(rc) return rc;
  cudaError_t e = cudaMalloc(ptr, bytes ? bytes : 1);
  if(e != cudaSuccess)
  {
    *ptr = nullptr;
    return fail(B200_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
  }
  return B200_OK;
}
extern "C" void b200_dev_free(void *ptr)
{
  if(ptr && g_alive.load()) cudaFree(ptr);
}
extern "C" int b200_copy_host_to_device(void *d_dst, const void *h_src, size_t bytes, void *stream)
{
  if(!d_dst || !h_src) return fail(B200_ERR_ARG, "copy_host_to_device: NULL");
  return copy_h2d(d_dst, h_src, bytes, (cudaStream_t)stream);
}
extern "C" int b200_copy_device_to_host(void *h_dst, const void *d_src, size_t bytes, void *stream)
{
  if(!h_dst || !d_src) return fail(B200_ERR_ARG, "copy_device_to_host: NULL");
  return copy_d2h(h_dst, d_src, bytes, (cudaStream_t)stream);
}
extern "C" int b200_ipc_export(void *d_ptr, unsigned char handle[B200_IPC_HANDLE_BYTES])
{
  static_assert(sizeof(cudaIpcMemHandle_t) == B200_IPC_HANDLE_BYTES, "IPC handle size");
  if(!d_ptr || !handle) return fail(B200_ERR_ARG, "ipc_export: NULL");
  cudaIpcMemHandle_t h;
  B200_CUDA_TRY(cudaIpcGetMemHandle(&h, d_ptr));
  memcpy(handle, &h, sizeof(h));
  return B200_OK;
}
extern "C" int b200_ipc_import(const unsigned char handle[B200_IPC_HANDLE_BYTES], void **d_ptr)
{
  if(!d_ptr || !handle) return fail(B200_ERR_ARG, "ipc_import: NULL");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  B200_CUDA_TRY(cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return B200_OK;
}
extern "C" int b200_ipc_release(void *d_ptr)
{
  if(d_ptr) B200_CUDA_TRY(cudaIpcCloseMemHandle(d_ptr));
  return B200_OK;
}
extern "C" int b200_stream_create(void **stream)
{
  if(!stream) return fail(B200_ERR_ARG, "stream_create: NULL");
  cudaStream_t s;
  B200_CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  *stream = (void *)s;
  return B200_OK;
}
extern "C" void b200_stream_destroy(void *stream)
{
  if(stream) cudaStreamDestroy((cudaStream_t)stream);
}
extern "C" int b200_event_create(void **event)
{
  if(!event) return fail(B200_ERR_ARG, "event_create: NULL");
  cudaEvent_t e;
  B200_CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  *event = (void *)e;
  return B200_OK;
}
extern "C" void b200_event_destroy(void *event)
{
  if(event) cudaEventDestroy((cudaEvent_t)event);
}
extern "C" int b200_event_record(void *event, void *stream)
{
  B200_CUDA_TRY(cudaEventRecord((cudaEvent_t)event, (cudaStream_t)stream));
  return B200_OK;
}
extern "C" int b200_stream_wait_event(void *stream, void *event)
{
  B200_CUDA_TRY(cudaStreamWaitEvent((cudaStream_t)stream, (cudaEvent_t)event, 0));
  return B200_OK;
}
extern "C" int b200_stream_synchronize(void *stream)
{
  B200_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
  return B200_OK;
}
