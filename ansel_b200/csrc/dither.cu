// dither (src/iop/dither.c): Floyd-Steinberg error diffusion of the display-referred RGBA frame down to the output's levels,
// process() :497-511 -> process_floyd_steinberg :331-454, bit for bit against the reference's lines under C float semantics.
//
// The diffusion is serial along rows and down the frame: pixel (j, i) adds, in this order, the errors of (j-1, i-1) * 1/16,
// (j-1, i) * 5/16, (j-1, i+1) * 3/16 and (j, i-1) * 7/16 to clipnan(in) and then quantises.  Row j can therefore take pixel i
// once row j-1 has finished i+1: a wavefront with rows skewed by two pixels.  dither_fs_kernel runs one row per thread and
// 32 consecutive rows per warp (= per block), lane l two pixels behind lane l-1; the row above hands its errors down with
// __shfl_up_sync, so the warp needs no barrier.  Lane 0 takes the errors of the previous block's last row from a global row
// buffer that block publishes in chunks of D pixels behind a release/acquire progress counter.  Blocks draw their row block
// from a ticket counter, so a block only ever waits on one that started before it and is resident: the forward-progress
// argument of decoupled look-back.  Every wait is bounded; past the bound the kernel raises a fault flag the host reports.
#ifndef B200_KERNELS_ON_CPU // tests/emul/emul_dither.cpp compiles the step, the parameters and the hand-off rules with g++
#include "runtime.h"
#include <cuda/atomic>
#endif
#include <math.h>

namespace b200
{
namespace
{
// what the host derives from the data block and the pipe (get_dither_parameters :257-323): f = levels - 1, rf = 1.0 / f as
// a double quotient stored as a float
struct dither_q_t
{
  float f, rf;
  int gray;
};

// which diffused errors reach a pixel (the first column, the last column and row 0 drop some)
enum
{
  DT_UL = 1,
  DT_U = 2,
  DT_UR = 4,
  DT_L = 8
};

__host__ __device__ __forceinline__ float dither_clipnan(const float x)
{ // clipnan :237-245
  return (x > 0.0f) ? ((x < 1.0f) ? x : 1.0f) : (isnan(x) ? 0.5f : 0.0f);
}
// _quantize :175-182 is rf * ceilf((val * f) - 0.5) with a double 0.5: ceilf((float)((double)x - 0.5)) == ceilf(x - 0.5f) for
// every float x (tests/test_cpu_dither.py walks all 2^32 of them), so the float subtraction gives the same bits
__host__ __device__ __forceinline__ float dither_quantize(const float v, const dither_q_t &q) { return q.rf * ceilf(v * q.f - 0.5f); }

__host__ __device__ __forceinline__ float dither_add(const float v, const float e, const float w, const bool on) { return on ? v + e * w : v; }

// One pixel: clipnan(in), the errors of the upper-left, upper, upper-right and left neighbours in the reference's order
// (PROCESS_PIXEL_* :380-405 and the final row :436-449), then nearest_color :191-218.  Returns the output; *err = old - new.
__host__ __device__ __forceinline__ float4 dither_pixel(const float4 in, const float4 ul, const float4 u, const float4 ur, const float4 l,
                                                        const int terms, const dither_q_t &q, float4 *err)
{
  float v[4] = { dither_clipnan(in.x), dither_clipnan(in.y), dither_clipnan(in.z), dither_clipnan(in.w) };
  const float a[4] = { ul.x, ul.y, ul.z, ul.w }, b[4] = { u.x, u.y, u.z, u.w }, c[4] = { ur.x, ur.y, ur.z, ur.w }, d[4] = { l.x, l.y, l.z, l.w };
#pragma unroll
  for(int k = 0; k < 4; k++)
  {
    v[k] = dither_add(v[k], a[k], 1.0f / 16.0f, terms & DT_UL);
    v[k] = dither_add(v[k], b[k], 5.0f / 16.0f, terms & DT_U);
    v[k] = dither_add(v[k], c[k], 3.0f / 16.0f, terms & DT_UR);
    v[k] = dither_add(v[k], d[k], 7.0f / 16.0f, terms & DT_L);
  }
  float n[4];
  if(q.gray)
  { // _rgb_to_gray :185-188; every lane, alpha included, becomes the gray value
    const float g = dither_quantize(0.30f * v[0] + 0.59f * v[1] + 0.11f * v[2], q);
    n[0] = n[1] = n[2] = n[3] = g;
  }
  else
  {
#pragma unroll
    for(int k = 0; k < 4; k++) n[k] = dither_quantize(v[k], q);
  }
  *err = make_float4(v[0] - n[0], v[1] - n[1], v[2] - n[2], v[3] - n[3]);
  return make_float4(n[0], n[1], n[2], n[3]);
}

// the terms of pixel (j, i) of a width-w frame
__host__ __device__ __forceinline__ int dither_terms(const int j, const int i, const int w)
{
  const int left = i > 0 ? DT_L : 0;
  if(j == 0) return left;
  return left | (i > 0 ? DT_UL : 0) | DT_U | (i < w - 1 ? DT_UR : 0);
}

// hand-off of a row block's last row: published in chunks of D pixels; progress counts the pixels published
__host__ __device__ __forceinline__ bool dither_publish_due(const int i, const int w, const int D) { return (i + 1) % D == 0 || i + 1 == w; }
__host__ __device__ __forceinline__ int dither_chunk_need(const int c, const int w, const int D) { return (c + 1) * D < w ? (c + 1) * D : w; }

constexpr int DROWS = 32;             // rows per block: one warp
constexpr long long DSPIN = 1ll << 22; // polls before a wait gives up (each at least one L2 round trip and a 64 ns sleep: > 1 s)
enum
{
  DFAULT_NONE = 0,
  DFAULT_SPIN = 1
};

// get_dither_parameters :257-323 for the Floyd-Steinberg types: < 0 = copy the input untouched; scale = roi_in.scale
int dither_params(const b200_dither_data_t *d, const int pipe_type, const float scale, dither_q_t *q)
{
  int graymode = -1;
  unsigned levels = 65536;
  const int l1 = (int)floorf(1.0f + log2f(1.0f / scale)); // dt_log2f = log2f with glibc
  const int bds = (pipe_type != B200_PIPE_EXPORT) ? l1 * l1 : 1;
  switch(d->dither_type)
  {
    case B200_DITHER_FS1BIT:
      graymode = 1;
      levels = bds + 1 < 256 ? bds + 1 : 256;
      levels = levels > 2 ? levels : 2;
      break;
    case B200_DITHER_FS4BIT_GRAY:
      graymode = 1;
      levels = 15 * bds + 1 < 256 ? 15 * bds + 1 : 256;
      levels = levels > 16 ? levels : 16;
      break;
    case B200_DITHER_FS8BIT:
      graymode = 0;
      levels = 256;
      break;
    case B200_DITHER_FS16BIT:
      graymode = 0;
      levels = 65536;
      break;
    case B200_DITHER_FSAUTO:
      switch(d->levels & B200_IMAGEIO_CHANNEL_MASK)
      {
        case B200_IMAGEIO_RGB: graymode = 0; break;
        case B200_IMAGEIO_GRAY: graymode = 1; break;
      }
      switch(d->levels & B200_IMAGEIO_PREC_MASK)
      {
        case B200_IMAGEIO_INT8: levels = 256; break;
        case B200_IMAGEIO_INT12: levels = 4096; break;
        case B200_IMAGEIO_INT16: levels = 65536; break;
        case B200_IMAGEIO_BW: levels = 2; break;
        default: graymode = -1; break; // INT32, FLOAT
      }
      break;
  }
  q->f = (float)(levels - 1);
  q->rf = (float)(1.0 / q->f);
  q->gray = graymode;
  return graymode;
}

#ifndef B200_KERNELS_ON_CPU
// frames under 3 px either way: clipnan and nearest_color, no diffusion (:361-372)
__global__ void dither_tiny_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, const size_t n, const dither_q_t q, const int keep_alpha)
{
  const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if(k >= n) return;
  const float4 z = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  const float4 x = in[k];
  float4 e;
  float4 o = dither_pixel(x, z, z, z, z, 0, q, &e);
  if(keep_alpha) o.w = x.w; // dt_iop_alpha_copy :369-370
  out[k] = o;
}

struct dither_sync_t
{
  int *ticket;   // row-block tickets handed out so far
  int *progress; // per row block: pixels of its last row published in `edge`
  int *fault;    // DFAULT_*
  float4 *edge;  // per row block but the last: the errors of its last row
};

__device__ __forceinline__ float4 shfl_up4(const float4 v)
{
  return make_float4(__shfl_up_sync(0xffffffffu, v.x, 1), __shfl_up_sync(0xffffffffu, v.y, 1), __shfl_up_sync(0xffffffffu, v.z, 1),
                     __shfl_up_sync(0xffffffffu, v.w, 1));
}
__device__ __forceinline__ float4 shfl4(const float4 v, const int src)
{
  return make_float4(__shfl_sync(0xffffffffu, v.x, src), __shfl_sync(0xffffffffu, v.y, src), __shfl_sync(0xffffffffu, v.z, src),
                     __shfl_sync(0xffffffffu, v.w, src));
}

// lane 0: wait until `progress` reaches `need`; false once the bound is exceeded or another block has faulted
__device__ bool dither_wait(int *progress, const int need, int *fault)
{
  cuda::atomic_ref<int, cuda::thread_scope_device> p(*progress);
  for(long long it = 0;; it++)
  {
    if(p.load(cuda::memory_order_acquire) >= need) return true;
    if(*(volatile int *)fault != DFAULT_NONE) return false;
    if(it >= DSPIN)
    {
      atomicCAS(fault, DFAULT_NONE, DFAULT_SPIN);
      return false;
    }
    __nanosleep(64);
  }
}

// D: steps per batch = pixels per hand-off chunk (D <= 32)
template <int D>
__global__ void __launch_bounds__(DROWS) dither_fs_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, const int w, const int h,
                                                          const dither_q_t q, const int keep_alpha, const dither_sync_t S)
{
  static_assert(D >= 1 && D <= 32, "a hand-off chunk is held one pixel per lane");
  const int lane = threadIdx.x;
  int ticket = 0;
  if(lane == 0) ticket = atomicAdd(S.ticket, 1);
  const int blk = __shfl_sync(0xffffffffu, ticket, 0);
  const int j = blk * DROWS + lane;
  const bool row = j < h;
  const float4 *src = in + (size_t)(row ? j : 0) * w;
  float4 *dst = out + (size_t)(row ? j : 0) * w;
  const bool publish = row && lane == DROWS - 1 && j + 1 < h;
  float4 *edge_out = S.edge + (size_t)blk * w;
  const float4 *edge_in = S.edge + (size_t)(blk - 1) * w;
  int *prev_progress = S.progress + blk - 1;
  const int last = (h - 1 - blk * DROWS) < DROWS - 1 ? h - 1 - blk * DROWS : DROWS - 1; // last lane with a row
  const int s_end = w - 1 + 2 * last;                                                  // step of that lane's last pixel
  const float4 z = make_float4(0.0f, 0.0f, 0.0f, 0.0f);

  // lane 0 needs at step s the error of (j-1, s+1): batch b (steps bD-1 .. bD+D-2) reads chunk b of the row above
  float4 up_next = z;
  int ok = 1;
  if(blk > 0)
  {
    if(lane == 0) ok = dither_wait(prev_progress, dither_chunk_need(0, w, D), S.fault);
    ok = __shfl_sync(0xffffffffu, ok, 0);
    if(!ok) return;
    if(lane < D && lane < w) up_next = __ldcg(edge_in + lane);
  }
  float4 inb[D], inn[D];
#pragma unroll
  for(int k = 0; k < D; k++)
  {
    const int p = k - 1 - 2 * lane;
    inn[k] = (row && p >= 0 && p < w) ? __ldg(src + p) : z;
  }
  float4 E = z, U1 = z, U2 = z, U3 = z; // own last error; errors of (j-1, p+1), (j-1, p), (j-1, p-1)
  for(int b = 0; b * D - 1 <= s_end; b++)
  {
    const int s0 = b * D - 1;
    const float4 up_cur = up_next;
    if(blk > 0 && (b + 1) * D < w)
    {
      if(lane == 0) ok = dither_wait(prev_progress, dither_chunk_need(b + 1, w, D), S.fault);
      ok = __shfl_sync(0xffffffffu, ok, 0);
      if(!ok) return;
      if(lane < D && (b + 1) * D + lane < w) up_next = __ldcg(edge_in + (b + 1) * D + lane);
    }
#pragma unroll
    for(int k = 0; k < D; k++)
    {
      inb[k] = inn[k];
      const int p = s0 + D + k - 2 * lane;
      inn[k] = (row && p >= 0 && p < w) ? __ldg(src + p) : z;
    }
#pragma unroll
    for(int k = 0; k < D; k++)
    {
      const int p = s0 + k - 2 * lane;
      float4 up = shfl_up4(E);
      const float4 above = shfl4(up_cur, k);
      if(lane == 0) up = blk > 0 ? above : z;
      U3 = U2;
      U2 = U1;
      U1 = up;
      if(row && p >= 0 && p < w)
      {
        float4 e;
        float4 o = dither_pixel(inb[k], U3, U2, U1, E, dither_terms(j, p, w), q, &e);
        if(keep_alpha) o.w = inb[k].w; // dt_iop_alpha_copy :451-453
        dst[p] = o;
        E = e;
        if(publish)
        {
          __stcg(edge_out + p, e);
          if(dither_publish_due(p, w, D))
            cuda::atomic_ref<int, cuda::thread_scope_device>(S.progress[blk]).store(p + 1, cuda::memory_order_release);
        }
      }
    }
  }
}
#endif
} // namespace
} // namespace b200

#ifndef B200_KERNELS_ON_CPU
using namespace b200;

static int dither_check(const b200_piece_t *piece, const void *in, const void *out)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "dither: NULL argument");
  if(!piece->data || piece->data_size < sizeof(b200_dither_data_t)) return fail(B200_ERR_ARG, "dither: piece->data is not a b200_dither_data_t");
  if(in == out) return fail(B200_ERR_ARG, "dither: in-place processing is not supported");
  if(piece->roi_in.width < 1 || piece->roi_in.height < 1) return fail(B200_ERR_ARG, "dither: empty roi_in");
  const b200_dither_data_t *d = (const b200_dither_data_t *)piece->data;
  if(d->dither_type == B200_DITHER_RANDOM)
    return fail(B200_ERR_UNSUPPORTED, "dither: the random method is not built (the reference carries tea_state[1] from row to row of an "
                                      "OpenMP thread, so its output depends on the thread count and schedule)");
  if(d->dither_type < B200_DITHER_FS1BIT || d->dither_type > B200_DITHER_FSAUTO) return fail(B200_ERR_ARG, "dither: method %d", d->dither_type);
  return B200_OK;
}

extern "C" int b200_dither_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = dither_check(piece, d_in, d_out);
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  const int w = piece->roi_in.width, h = piece->roi_in.height;
  const size_t npx = (size_t)w * h;
  const int keep_alpha = (piece->mask_display & B200_DISPLAY_MASK) ? 1 : 0;
  dither_q_t q;
  if(dither_params((const b200_dither_data_t *)piece->data, piece->pipe_type, (float)piece->roi_in.scale, &q) < 0)
  { // no quantisation for this output: the buffer passes untouched (:346-354)
    B200_CUDA_TRY(cudaMemcpyAsync(d_out, d_in, npx * 16, cudaMemcpyDeviceToDevice, s));
    return B200_OK;
  }
  if(w < 3 || h < 3)
  {
    dither_tiny_kernel<<<(unsigned)((npx + 255) / 256), 256, 0, s>>>((const float4 *)d_in, (float4 *)d_out, npx, q, keep_alpha);
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
  }
  const int nblk = (h + DROWS - 1) / DROWS;
  void *sync = nullptr, *edge = nullptr;
  const size_t sync_bytes = sizeof(int) * (size_t)(nblk + 2);
  if((rc = scratch(SLOT_SMALL + 4, sync_bytes, &sync))) return rc;
  if(nblk > 1 && (rc = scratch(SLOT_TMP0, sizeof(float4) * (size_t)w * (nblk - 1), &edge))) return rc;
  B200_CUDA_TRY(cudaMemsetAsync(sync, 0, sync_bytes, s));
  int *ints = (int *)sync;
  const dither_sync_t S = { ints, ints + 2, ints + 1, (float4 *)edge };
  dither_fs_kernel<16><<<nblk, DROWS, 0, s>>>((const float4 *)d_in, (float4 *)d_out, w, h, q, keep_alpha, S);
  B200_CUDA_TRY(cudaGetLastError());
  int fault = DFAULT_NONE;
  B200_CUDA_TRY(cudaMemcpyAsync(&fault, ints + 1, sizeof(int), cudaMemcpyDeviceToHost, s));
  B200_CUDA_TRY(cudaStreamSynchronize(s));
  if(fault != DFAULT_NONE)
    return fail(B200_ERR_CUDA, "dither: a row block waited past its bound for the errors of the block above (%dx%d frame, %d row blocks)", w, h, nblk);
  return B200_OK;
}

extern "C" int b200_dither_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = dither_check(piece, in, out);
  if(rc) return rc;
  const size_t bytes = (size_t)piece->roi_in.width * piece->roi_in.height * 16;
  return through_device(piece, in, bytes, out, bytes, false, b200_dither_process_dev);
}

extern "C" void b200_dither_tiling(const b200_piece_t *piece, b200_tiling_t *t) { default_tiling(piece, t, 0, false); } // the module declares no tiling callback
#endif
