// The pointwise modules either side of the demosaic .. colorout path (SURVEY.md 8f ranks 1 and 2).
//
// Reference: iop/rawprepare.c process() :466-633 (compute_proper_crop :206-210, BL :413-418); iop/temperature.c process()
// :486-608; iop/highlights.c process() :679-789 with _hl_count_thresholds :232-253, _hl_count_clipped :266-292,
// iop/highlights/clip.c process_clip :60-85; iop/exposure.c process() :501-544; iop/gamma.c _copy_output :352-364;
// imageio/imageio_core.c :706-738 (the export's float -> uint8 / uint16 conversions).
//
// All of it is HBM-bound streaming: 2..16 bytes in, 4..16 bytes out per sample, a handful of flops.  One thread per
// four samples (vector loads and stores where the row geometry allows them).  The three raw-domain modules also exist
// as one fused pass over the sensor data (b200_rawfront_process_dev): 8 instead of 26 bytes per sample for uint16 input.
#ifndef B200_KERNELS_ON_CPU // tests/emul compiles the kernels of this file with g++ to check them against the oracle without a GPU
#include "runtime.h"
#include <initializer_list>
#endif
#include "x87.cuh"
#include <float.h>
#include <math.h>
#include <string.h>

namespace
{
constexpr int NT = 256;

// ---- the raw domain: one description of "what happens to a sensor sample" shared by the per-module and fused kernels ----
struct prepare_t
{ // rawprepare: the Bayer branches of process() :480-560 and the gain maps :592-630
  float sub[4], inv_div[4];
  int in_width;     // roi_in->width (samples per input row)
  int csx, csy;     // compute_proper_crop of the border trim
  int cfa_x, cfa_y; // roi_out origin + trim: phase of the 2x2 block
  int roi_x, roi_y; // roi_out origin (the gain maps are addressed in image coordinates)
  int gain;         // apply_gainmaps
  unsigned map_w, map_h;
  float im_to_rel_x, im_to_rel_y, rel_to_map_x, rel_to_map_y, map_origin_h, map_origin_v;
  const float *maps; // 4 planes of map_w * map_h gains, device memory
};
struct balance_t
{ // temperature on a Bayer mosaic :552-577
  float coeffs[4];
  unsigned filters;
  int roi_x, roi_y;
};
struct clip_t
{ // highlights: process_clip on a mosaic, and the bypass test
  float clip, raw_threshold;
};

__device__ __forceinline__ int fc(int row, int col, unsigned filters)
{ // develop/imageop_math.h:190-193
  return (filters >> ((((row << 1) & 14) + (col & 1)) << 1)) & 3;
}
__device__ __forceinline__ float divr(float a, float b)
{ // IEEE division, opaque to nvcc's x / c -> x * (1 / c) rewrite (see labglue.cu: divc)
#ifdef B200_KERNELS_ON_CPU
  return a / b;
#else
  float q;
  asm("div.rn.ftz.f32 %0, %1, %2;" : "=f"(q) : "f"(a), "f"(b));
  return q;
#endif
}

// bilinear gain of site `id` at output sample (j, i): rawprepare.c:603-626.  CLAMP and MIN mix float, int and uint32
// operands in the reference: every comparison there is a float comparison, every result a float.
__device__ __forceinline__ float gain_at(const prepare_t &P, int id, int j, int i)
{
  float y_map = ((float)(P.roi_y + P.csy + j) * P.im_to_rel_y - P.map_origin_v) * P.rel_to_map_y;
  y_map = y_map > (float)P.map_h ? (float)P.map_h : (y_map < 0.0f ? 0.0f : y_map);
  const unsigned y_i0 = (unsigned)(y_map < (float)(P.map_h - 1) ? y_map : (float)(P.map_h - 1));
  const unsigned y_i1 = (y_i0 + 1 < P.map_h - 1) ? y_i0 + 1 : P.map_h - 1;
  const float y_frac = y_map - (float)y_i0;
  float x_map = ((float)(P.roi_x + P.csx + i) * P.im_to_rel_x - P.map_origin_h) * P.rel_to_map_x;
  x_map = x_map > (float)P.map_w ? (float)P.map_w : (x_map < 0.0f ? 0.0f : x_map);
  const unsigned x_i0 = (unsigned)(x_map < (float)(P.map_w - 1) ? x_map : (float)(P.map_w - 1));
  const unsigned x_i1 = (x_i0 + 1 < P.map_w - 1) ? x_i0 + 1 : P.map_w - 1;
  const float x_frac = x_map - (float)x_i0;
  const float *plane = P.maps + (size_t)id * P.map_w * P.map_h;
  const float *row0 = plane + (size_t)y_i0 * P.map_w, *row1 = plane + (size_t)y_i1 * P.map_w;
  const float gain_top = (1.0f - x_frac) * row0[x_i0] + x_frac * row0[x_i1];
  const float gain_bottom = (1.0f - x_frac) * row1[x_i0] + x_frac * row1[x_i1];
  return (1.0f - y_frac) * gain_top + y_frac * gain_bottom;
}
// one of four kernel-parameter floats without dynamic indexing (which would copy the array to local memory)
__device__ __forceinline__ float pick4(const float (&a)[4], int k) { return (k & 2) ? ((k & 1) ? a[3] : a[2]) : ((k & 1) ? a[1] : a[0]); }
// four consecutive samples as floats: one 8- or 16-byte load when the address allows it
__device__ __forceinline__ void load4(const unsigned short *p, int n, float (&x)[4])
{
  if(n == 4 && ((size_t)p & 7) == 0)
  {
    const uint2 w = *(const uint2 *)p;
    x[0] = (float)(w.x & 0xffffu);
    x[1] = (float)(w.x >> 16);
    x[2] = (float)(w.y & 0xffffu);
    x[3] = (float)(w.y >> 16);
  }
  else
    for(int k = 0; k < 4; k++) x[k] = k < n ? (float)p[k] : 0.0f;
}
__device__ __forceinline__ void load4(const float *p, int n, float (&x)[4])
{
  if(n == 4 && ((size_t)p & 15) == 0)
  {
    const float4 w = *(const float4 *)p;
    x[0] = w.x;
    x[1] = w.y;
    x[2] = w.z;
    x[3] = w.w;
  }
  else
    for(int k = 0; k < 4; k++) x[k] = k < n ? p[k] : 0.0f;
}

// Four consecutive samples of one row per thread.  STAGES: bit 0 rawprepare, bit 1 temperature, bit 2 highlights clip.
// COUNT: no output, count the samples the highlights bypass test calls clipped (value after stages 0..1 > raw_threshold).
// Stage 2 reads the counter a previous COUNT launch filled: fewer than 25 -> the samples pass unclipped.
template <typename T, int STAGES, bool COUNT>
__global__ void __launch_bounds__(NT) raw_front_kernel(const T *__restrict__ in, float *__restrict__ out, int width, int height, prepare_t P,
                                                       balance_t B, clip_t H, unsigned long long *counter)
{
  const int i0 = (blockIdx.x * NT + threadIdx.x) * 4;
  const int j = blockIdx.y;
  int local = 0;
  if(i0 < width)
  {
    const size_t pin = (STAGES & 1) ? (size_t)P.in_width * (j + P.csy) + P.csx + i0 : (size_t)j * width + i0;
    const size_t pout = (size_t)j * width + i0;
    const int n = min(4, width - i0);
    bool clip_on = false;
    if((STAGES & 4) && !COUNT) clip_on = *counter >= 25ull; // DT_HL_MIN_CLIPPED_PIXELS, iop/highlights/common.h:218
    // the 2x2 period made explicit, as the reference's row loops do (:489-512, :556-577): two site ids and two
    // white-balance coefficients per row, alternating with the column (i0 is a multiple of 4)
    float sub[2] = { 0.f, 0.f }, inv[2] = { 0.f, 0.f }, wb[2] = { 0.f, 0.f };
    int id[2] = { 0, 0 };
    if(STAGES & 1)
    {
      const int row_phase = ((j + P.cfa_y) & 1) << 1;
      id[0] = row_phase + (P.cfa_x & 1);
      id[1] = row_phase + ((P.cfa_x & 1) ^ 1);
      for(int q = 0; q < 2; q++)
      {
        sub[q] = pick4(P.sub, id[q]);
        inv[q] = pick4(P.inv_div, id[q]);
      }
    }
    if(STAGES & 2)
      for(int q = 0; q < 2; q++) wb[q] = pick4(B.coeffs, fc(j + B.roi_y, q + B.roi_x, B.filters));
    float v[4];
    load4(in + pin, n, v);
#pragma unroll
    for(int k = 0; k < 4; k++)
      if(k < n)
      {
        float x = v[k];
        if(STAGES & 1)
        {
          x = (x - sub[k & 1]) * inv[k & 1];
          if(P.gain) x *= gain_at(P, id[k & 1], j, i0 + k);
        }
        if(STAGES & 2) x = x * wb[k & 1];
        if(COUNT)
          local += (x > H.raw_threshold) ? 1 : 0;
        else if((STAGES & 4) && clip_on)
          x = H.clip < x ? H.clip : x; // MIN(clip, in[k])
        v[k] = x;
      }
    if(!COUNT)
    {
      if(n == 4 && (pout & 3) == 0)
        *(float4 *)(out + pout) = make_float4(v[0], v[1], v[2], v[3]);
      else
        for(int k = 0; k < n; k++) out[pout + k] = v[k];
    }
  }
  if(COUNT)
  {
#ifdef B200_KERNELS_ON_CPU
    if(local) atomicAdd(counter, (unsigned long long)local);
#else
    local = __reduce_add_sync(0xffffffffu, local);
    if((threadIdx.x & 31) == 0 && local) atomicAdd(counter, (unsigned long long)local);
#endif
  }
}

// ---- flat kernels over n floats (4 per thread) -------------------------------------------------------------------------
enum
{
  OP_EXPOSURE = 1,       // (in - black) * scale
  OP_CLIP = 2,           // MIN(clip, in) when the counter says so
  OP_COPY = 3
};
template <int OP> __device__ __forceinline__ float flat_op(float x, float a, float b)
{
  if(OP == OP_EXPOSURE) return (x - a) * b;
  if(OP == OP_CLIP) return a < x ? a : x;
  return x;
}
// keep_alpha: lane 3 of every pixel is the input's (dt_iop_alpha_copy after the loop when a mask is displayed)
template <int OP> __global__ void __launch_bounds__(NT) flat_kernel(const float *__restrict__ in, float *__restrict__ out, size_t n, float a, float b,
                                                                    int keep_alpha, const unsigned long long *counter)
{
  const size_t k0 = ((size_t)blockIdx.x * NT + threadIdx.x) * 4;
  if(k0 >= n) return;
  bool on = true;
  if(OP == OP_CLIP) on = *counter >= 25ull;
  if(k0 + 4 <= n)
  {
    const float4 p = *(const float4 *)(in + k0);
    float4 o;
    o.x = on ? flat_op<OP>(p.x, a, b) : p.x;
    o.y = on ? flat_op<OP>(p.y, a, b) : p.y;
    o.z = on ? flat_op<OP>(p.z, a, b) : p.z;
    o.w = (on && !keep_alpha) ? flat_op<OP>(p.w, a, b) : p.w;
    *(float4 *)(out + k0) = o;
  }
  else
    for(size_t k = k0; k < n; k++) out[k] = on ? flat_op<OP>(in[k], a, b) : in[k];
}

// rawprepare's third branch with a crop: `ch` floats per pixel, one thread per float
__global__ void __launch_bounds__(NT) predownsampled_kernel(const float *__restrict__ in, float *__restrict__ out, int width, int height, int ch,
                                                            int in_width, int csx, int csy, float sub, float div)
{
  const size_t k = (size_t)blockIdx.x * NT + threadIdx.x;
  if(k >= (size_t)width * height * ch) return;
  const int c = (int)(k % ch);
  const size_t px = k / ch;
  const int i = (int)(px % width), j = (int)(px / width);
  out[k] = divr(in[(size_t)ch * ((size_t)in_width * (j + csy) + csx + i) + c] - sub, div);
}

// temperature on an X-Trans mosaic :504-549 and on `ch` floats per pixel :579-600
__global__ void __launch_bounds__(NT) balance_xtrans_kernel(const float *__restrict__ in, float *__restrict__ out, int width, int height, int roi_x,
                                                            int roi_y, const float *__restrict__ lut36)
{ // lut36[r * 6 + c] = coeffs[xtrans[r][c]]
  const int i = blockIdx.x * NT + threadIdx.x, j = blockIdx.y;
  if(i >= width) return;
  const size_t p = (size_t)j * width + i;
  out[p] = in[p] * lut36[((j + 600 + roi_y) % 6) * 6 + ((i % 12) + 600 + roi_x) % 6];
}
__global__ void __launch_bounds__(NT) balance_pixels_kernel(const float *__restrict__ in, float *__restrict__ out, size_t npixels, int ch, float c0,
                                                            float c1, float c2)
{
  const size_t k = (size_t)blockIdx.x * NT + threadIdx.x;
  if(k >= npixels) return;
  if(ch == 4)
  {
    const float4 p = ((const float4 *)in)[k];
    ((float4 *)out)[k] = make_float4(p.x * c0, p.y * c1, p.z * c2, p.w);
  }
  else
  { // the first three floats of every `ch`: the rest of the pixel is not written (:589-597)
    out[k * ch + 0] = in[k * ch + 0] * c0;
    out[k * ch + 1] = in[k * ch + 1] * c1;
    out[k * ch + 2] = in[k * ch + 2] * c2;
  }
}

// highlights on non-mosaic input: a pixel counts when any of its first three floats is over its threshold :278-290
__global__ void __launch_bounds__(NT) count_pixels_kernel(const float *__restrict__ in, size_t npixels, int ch, float t0, float t1, float t2,
                                                          unsigned long long *counter)
{
  const size_t k = (size_t)blockIdx.x * NT + threadIdx.x;
  int local = 0;
  if(k < npixels)
  {
    const float *p = in + k * ch;
    int over = p[0] > t0;
    if(ch > 1) over |= p[1] > t1;
    if(ch > 2) over |= p[2] > t2;
    local = over;
  }
#ifdef B200_KERNELS_ON_CPU
  if(local) atomicAdd(counter, (unsigned long long)local);
#else
  local = __reduce_add_sync(0xffffffffu, local);
  if((threadIdx.x & 31) == 0 && local) atomicAdd(counter, (unsigned long long)local);
#endif
}

// ---- highlights, colour inpainting on a Bayer mosaic (iop/highlights/inpaint.c:63-82, lch.c interpolate_color :206-303) ----
// Along a line, a running ratio between neighbouring sites (decayed over unclipped pairs) restores a clipped sample from its
// neighbour; the four directions (along the row both ways, along the column both ways) are summed in that order and divided by four.
// Each line of each direction is a serial recurrence, and nothing else is: the four directions run at once, one thread per line
// (2 x height + 2 x width threads), each into a plane of its own, and a pointwise pass sums the planes in the reference's order.
// A thread per ROW would make a warp touch 32 rows at once, so the row directions run on a transposed copy of the mosaic where
// neighbouring rows are neighbouring addresses, like the columns of the frame itself; their two planes come back through a second
// transposition that already adds them.  The operands of eight steps are fetched ahead of the recurrence.
struct inpaint_t
{
  float clips[4]; // 0.987 * clip * processed_maximum per colour
  unsigned filters; // ROI-shifted
  int width, height;
};
// one direction of one line.  dim 0: along row `other`, dim 1: down column `other`; (si, sj) = the strides of a column step and of a
// row step in `in` and `plane`.  Only clipped sites are written (what the reference adds to its output there).
__device__ void inpaint_chain(const float *__restrict__ in, float *__restrict__ plane, const inpaint_t &A, ptrdiff_t si, ptrdiff_t sj, int dim, int dir, int other)
{
  const int n = dim ? A.height : A.width, n_other = dim ? A.width : A.height;
  if(other == 0 || other == n_other - 1) return; // a border line :232-235
  const ptrdiff_t step = dim ? sj : si, line = (ptrdiff_t)other * (dim ? si : sj);
  const int beg = dir == 1 ? 0 : n - 1;
  float ratio = 1.0f;
  for(int base = 0; base < n; base += 8)
  {
    float v[9];
#pragma unroll
    for(int m = 0; m < 9; m++)
    {
      const int k = beg + min(base + m, n - 1) * dir;
      v[m] = __ldg(in + line + (ptrdiff_t)k * step);
    }
#pragma unroll
    for(int m = 0; m < 8; m++)
    {
      const int k = beg + (base + m) * dir;
      if(base + m >= n || k == 0 || k == n - 1) continue; // the ends of the line are border sites
      const int i = dim ? other : k, j = dim ? k : other;
      const float clip0 = pick4(A.clips, fc(j, i, A.filters));
      const float clip1 = pick4(A.clips, fc(dim ? (j + 1) : j, dim ? i : (i + 1), A.filters));
      const float v0 = v[m], v1 = v[m + 1];
      if(v0 < clip0 && v0 > 1e-5f && v1 < clip1 && v1 > 1e-5f)
      { // both unclipped: ratio = in[odd] / in[even], exponential decay
        if(k & 1)
          ratio = (3.0f * ratio + v0 / v1) / 4.0f;
        else
          ratio = (3.0f * ratio + v1 / v0) / 4.0f;
      }
      if(v0 >= clip0 - 1e-5f)
      {
        float add;
        if(v1 >= clip1 - 1e-5f)
          add = fmaxf(clip0, clip1);
        else if(k & 1)
          add = v1 * ratio;
        else
          add = v1 / ratio;
        plane[line + (ptrdiff_t)k * step] = add;
      }
    }
  }
}
// `counter`: the clipped-sample count of the bypass test; under 25 the frame is copied through (by the last kernel) and nothing else runs
// grid.y = the direction.  Rows: on the transposed mosaic (site (i, j) at i * height + j)
__global__ void __launch_bounds__(128) inpaint_rows_kernel(const float *__restrict__ t_in, float *__restrict__ t_fwd, float *__restrict__ t_bwd, inpaint_t A,
                                                           const unsigned long long *counter)
{
  const int j = blockIdx.x * 128 + threadIdx.x;
  if(j >= A.height || *counter < 25ull) return;
  inpaint_chain(t_in, blockIdx.y ? t_bwd : t_fwd, A, A.height, 1, 0, blockIdx.y ? -1 : 1, j);
}
__global__ void __launch_bounds__(128) inpaint_cols_kernel(const float *__restrict__ in, float *__restrict__ down, float *__restrict__ up, inpaint_t A,
                                                           const unsigned long long *counter)
{
  const int i = blockIdx.x * 128 + threadIdx.x;
  if(i >= A.width || *counter < 25ull) return;
  inpaint_chain(in, blockIdx.y ? up : down, A, 1, A.width, 1, blockIdx.y ? -1 : 1, i);
}
// out[x][y] = a[y][x] (+ b[y][x]): `a` has `cols` floats per row and `rows` rows.  32x32 tiles, block (32, 8).
template <bool ADD>
__global__ void __launch_bounds__(256) transpose_kernel(const float *__restrict__ a, const float *__restrict__ b, float *__restrict__ out, int cols, int rows,
                                                        const unsigned long long *counter)
{
  if(*counter < 25ull) return;
#ifdef B200_KERNELS_ON_CPU // the harness runs threads one after the other: no staging through shared memory there
  const int x = (int)blockIdx.x * 32 + (int)threadIdx.x % 32, y0 = (int)blockIdx.y * 32;
  for(int y = y0 + (int)threadIdx.x / 32; y < min(y0 + 32, rows); y += 8)
    if(x < cols) out[(size_t)x * rows + y] = ADD ? a[(size_t)y * cols + x] + b[(size_t)y * cols + x] : a[(size_t)y * cols + x];
#else
  __shared__ float tile[32][33];
  const int tx = threadIdx.x % 32, ty = threadIdx.x / 32;
  const int x = blockIdx.x * 32 + tx;
  for(int r = ty; r < 32; r += 8)
  {
    const int y = blockIdx.y * 32 + r;
    if(x < cols && y < rows) tile[r][tx] = ADD ? __ldg(a + (size_t)y * cols + x) + __ldg(b + (size_t)y * cols + x) : __ldg(a + (size_t)y * cols + x);
  }
  __syncthreads();
  const int oy = blockIdx.y * 32 + tx; // the source row this lane writes
  for(int r = ty; r < 32; r += 8)
  {
    const int ox = blockIdx.x * 32 + r;
    if(ox < cols && oy < rows) out[(size_t)ox * rows + oy] = tile[tx][r];
  }
#endif
}
// the sum of the four directions in the reference's order, ((rows forward + rows backward) + down) + up, a quarter of it at the clipped
// sites, the input elsewhere (:232-235, :290-299).  `down` may be `out`.
__global__ void __launch_bounds__(NT) inpaint_sum_kernel(const float *__restrict__ in, const float *__restrict__ rows, const float *down, const float *__restrict__ up,
                                                         float *out, inpaint_t A, const unsigned long long *counter)
{
  const int i = blockIdx.x * NT + threadIdx.x, j = blockIdx.y;
  if(i >= A.width) return;
  const size_t p = (size_t)j * A.width + i;
  const float v0 = __ldg(in + p);
  float o = v0;
  if(*counter >= 25ull && i > 0 && i < A.width - 1 && j > 0 && j < A.height - 1 && v0 >= pick4(A.clips, fc(j, i, A.filters)) - 1e-5f)
    o = (((__ldg(rows + p)) + down[p]) + __ldg(up + p)) / 4.0f;
  out[p] = o;
}

// ---- highlights, LCh reconstruction on a Bayer mosaic (iop/highlights/lch.c:315-411) --------------------------------------------
// Every 2x2 block with a clipped sample is rebuilt from the lightness / chroma / hue of its clipped and unclipped values.  The
// reference multiplies and divides by long double constants (SQRT3, SQRT12): x87.cuh performs those three operations exactly.
// filters: the sensor's word, the ROI origin enters through x0 / y0 (process_lch_bayer reads piece->dsc_in.filters).
__global__ void __launch_bounds__(NT) lch_bayer_kernel(const float *__restrict__ ivoid, float *__restrict__ ovoid, int width, int height, int x0, int y0,
                                                       unsigned filters, float clip, const unsigned long long *counter)
{
  const int i = blockIdx.x * NT + threadIdx.x, j = blockIdx.y;
  if(i >= width) return;
  const float *in = ivoid + (size_t)width * j + i;
  float *out = ovoid + (size_t)width * j + i;
  if(*counter < 25ull)
  { // the bypass: fewer than DT_HL_MIN_CLIPPED_PIXELS samples over the threshold, the frame is copied through
    out[0] = in[0];
    return;
  }
  if(i == width - 1 || j == height - 1)
  {
    out[0] = clip < in[0] ? clip : in[0];
    return;
  }
  bool clipped = false;
  float R = 0.0f, Gmin = FLT_MAX, Gmax = -FLT_MAX, B = 0.0f;
#pragma unroll
  for(int jj = 0; jj <= 1; jj++)
#pragma unroll
    for(int ii = 0; ii <= 1; ii++)
    {
      const float val = in[(size_t)jj * width + ii];
      clipped = clipped || (val > clip);
      const int c = fc(j + jj + y0, i + ii + x0, filters);
      if(c == 0)
        R = val;
      else if(c == 1)
      {
        Gmin = Gmin < val ? Gmin : val;
        Gmax = Gmax > val ? Gmax : val;
      }
      else if(c == 2)
        B = val;
    }
  if(!clipped)
  {
    out[0] = in[0];
    return;
  }
  const float Ro = R < clip ? R : clip, Go = Gmin < clip ? Gmin : clip, Bo = B < clip ? B : clip;
  const float L = divr(R + Gmax + B, 3.0f);
  float C = x87::mul_sqrt3(R - Gmax);
  float H = 2.0f * B - Gmax - R;
  const float Co = x87::mul_sqrt3(Ro - Go);
  const float Ho = 2.0f * Bo - Go - Ro;
  if(R != Gmax && Gmax != B)
  {
    const float ratio = sqrtf((Co * Co + Ho * Ho) / (C * C + H * H));
    C *= ratio;
    H *= ratio;
  }
  const float t = L - divr(H, 6.0f);
  const int c = fc(j + y0, i + x0, filters);
  float v;
  if(c == 0)
    v = x87::add_div_sqrt12(t, C, +1);
  else if(c == 1)
    v = x87::add_div_sqrt12(t, C, -1);
  else
    v = L + divr(H, 3.0f);
  out[0] = v;
}

// ---- the X-Trans variants of the two reconstructions (lch.c:66-204, :412-537; inpaint.c:84-104) -------------------------------------
struct xtable_t
{
  unsigned char v[36]; // piece->dsc_in.xtrans
  int x0, y0;          // roi_in origin
};
__device__ __forceinline__ int fcx(const xtable_t &X, int row, int col) { return X.v[((row + 600 + X.y0) % 6) * 6 + (col + 600 + X.x0) % 6]; } // FCxtrans
__device__ __forceinline__ float pick4r(const float *a, int k) { return (k & 2) ? ((k & 1) ? a[3] : a[2]) : ((k & 1) ? a[1] : a[0]); }
__device__ __forceinline__ void set4r(float *a, int k, float v)
{
  if(k == 1) a[1] = v;
  else if(k == 2) a[2] = v;
  else if(k == 3) a[3] = v;
}
// interp_pix_xtrans :66-88
__device__ __forceinline__ float interp_pix_xtrans(int ratio_next, float next, float clip0, float clip_next, const float *ratios)
{
  const float clip_val = fmaxf(clip0, clip_next);
  if(next >= clip_next - 1e-5f) return clip_val;
  if(ratio_next > 0) return fminf(next / pick4r(ratios, ratio_next), clip_val);
  return fminf(next * pick4r(ratios, -ratio_next), clip_val);
}
// the colour-transition table roff[f0][f1] :104: RG 1, RB 2, GB 3, negative = inverted
__device__ __forceinline__ int roff(int f0, int f1) { return f0 == f1 ? 0 : (f0 < f1 ? -(f0 + f1) : (f0 + f1)); }
// interpolate_color_xtrans :90-204: three running ratios (one per colour pair) instead of Bayer's one; one direction of one line, laid out and
// fetched like inpaint_chain (the Bayer one): only clipped sites are written
__device__ void inpaint_chain_xtrans(const float *__restrict__ in, float *__restrict__ plane, const inpaint_t &A, const xtable_t &X, ptrdiff_t si, ptrdiff_t sj,
                                     int dim, int dir, int other)
{
  const int n = dim ? A.height : A.width, n_other = dim ? A.width : A.height;
  if(other == 0 || other == n_other - 1) return; // a border line :118-121
  const ptrdiff_t step = dim ? sj : si, across = dim ? si : sj, line = (ptrdiff_t)other * across;
  const int beg = dir == 1 ? 0 : n - 1;
  float ratios[4] = { 1.0f, 1.0f, 1.0f, 1.0f };
  for(int base = 0; base < n; base += 8)
  {
    float v[9];
#pragma unroll
    for(int m = 0; m < 9; m++)
    {
      const int k = beg + min(base + m, n - 1) * dir;
      v[m] = __ldg(in + line + (ptrdiff_t)k * step);
    }
#pragma unroll
    for(int m = 0; m < 8; m++)
    {
      const int k = beg + (base + m) * dir;
      if(base + m >= n || k == 0 || k == n - 1) continue;
      const int i = dim ? other : k, j = dim ? k : other;
      const int f0 = fcx(X, j, i), f1 = fcx(X, dim ? (j + dir) : j, dim ? i : (i + dir));
      const float clip0 = pick4(A.clips, f0), clip1 = pick4(A.clips, f1);
      const float v0 = v[m], v1 = v[m + 1];
      if((f0 != f1) && (v0 < clip0 && v0 > 1e-5f) && (v1 < clip1 && v1 > 1e-5f))
      {
        const int r = roff(f0, f1);
        if(r > 0)
          set4r(ratios, r, (3.f * pick4r(ratios, r) + (v1 / v0)) / 4.f);
        else
          set4r(ratios, -r, (3.f * pick4r(ratios, -r) + (v0 / v1)) / 4.f);
      }
      if(v0 >= clip0 - 1e-5f)
      {
        float add;
        if(f0 != f1)
          add = interp_pix_xtrans(roff(f0, f1), v1, clip0, clip1, ratios);
        else
        { // at the start of a 2x2 green block: look diagonally (one step on, one line to either side)
          const int fl = fcx(X, dim ? (j + dir) : (j - 1), dim ? (i - 1) : (i + dir)), fr = fcx(X, dim ? (j + dir) : (j + 1), dim ? (i + 1) : (i + dir));
          const float *next = in + line + (ptrdiff_t)(k + dir) * step;
          add = (fl != f0) ? interp_pix_xtrans(roff(f0, fl), __ldg(next - across), clip0, pick4(A.clips, fl), ratios)
                           : interp_pix_xtrans(roff(f0, fr), __ldg(next + across), clip0, pick4(A.clips, fr), ratios);
        }
        plane[line + (ptrdiff_t)k * step] = add;
      }
    }
  }
}
__global__ void __launch_bounds__(128) inpaint_rows_xtrans_kernel(const float *__restrict__ t_in, float *__restrict__ t_fwd, float *__restrict__ t_bwd, inpaint_t A,
                                                                  xtable_t X, const unsigned long long *counter)
{ // on the transposed mosaic, like inpaint_rows_kernel
  const int j = blockIdx.x * 128 + threadIdx.x;
  if(j >= A.height || *counter < 25ull) return;
  inpaint_chain_xtrans(t_in, blockIdx.y ? t_bwd : t_fwd, A, X, A.height, 1, 0, blockIdx.y ? -1 : 1, j);
}
__global__ void __launch_bounds__(128) inpaint_cols_xtrans_kernel(const float *__restrict__ in, float *__restrict__ down, float *__restrict__ up, inpaint_t A,
                                                                  xtable_t X, const unsigned long long *counter)
{
  const int i = blockIdx.x * 128 + threadIdx.x;
  if(i >= A.width || *counter < 25ull) return;
  inpaint_chain_xtrans(in, blockIdx.y ? up : down, A, X, 1, A.width, 1, blockIdx.y ? -1 : 1, i);
}
// the four directions summed in the reference's order, capped at the largest clip value :114, :196-199
__global__ void __launch_bounds__(NT) inpaint_sum_xtrans_kernel(const float *__restrict__ in, const float *__restrict__ rows, const float *down,
                                                                const float *__restrict__ up, float *out, inpaint_t A, xtable_t X, const unsigned long long *counter)
{
  const int i = blockIdx.x * NT + threadIdx.x, j = blockIdx.y;
  if(i >= A.width) return;
  const size_t p = (size_t)j * A.width + i;
  const float v0 = __ldg(in + p);
  float o = v0;
  if(*counter >= 25ull)
  {
    const float clip_max = fmaxf(fmaxf(A.clips[0], A.clips[1]), A.clips[2]);
    if(i == 0 || i == A.width - 1 || j == 0 || j == A.height - 1)
      o = fminf(clip_max, v0);
    else if(v0 >= pick4(A.clips, fcx(X, j, i)) - 1e-5f)
      o = fminf(clip_max, (((__ldg(rows + p)) + down[p]) + __ldg(up + p)) / 4.0f);
  }
  out[p] = o;
}
// process_lch_xtrans :412-537.  The reference's ring buffer `cl` says whether any of this and the two previous columns has a
// clipped sample in rows j-1..j+1: recomputed per pixel here.
__global__ void __launch_bounds__(NT) lch_xtrans_kernel(const float *__restrict__ ivoid, float *__restrict__ ovoid, int width, int height, xtable_t X, float clip,
                                                        const unsigned long long *counter)
{
  const int i = blockIdx.x * NT + threadIdx.x, j = blockIdx.y;
  if(i >= width) return;
  const float *in = ivoid + (size_t)width * j + i;
  float *out = ovoid + (size_t)width * j + i;
  if(*counter < 25ull)
  {
    out[0] = in[0];
    return;
  }
  if(i < 2 || i > width - 3 || j < 2 || j > height - 3)
  {
    out[0] = clip < in[0] ? clip : in[0];
    return;
  }
  bool clipped = in[0] > clip;
  if(!clipped)
  {
    bool cl = false;
    for(int ii = -2; ii <= 0; ii++) cl = cl || (in[-width + ii] > clip) || (in[ii] > clip) || (in[width + ii] > clip);
    clipped = cl;
    if(clipped)
      for(int offset_j = -2; offset_j <= 0; offset_j++)
        for(int offset_i = -2; offset_i <= 0; offset_i++)
          if(clipped)
          { // a 3x3 block touching the pixel without any clipping: no reconstruction
            clipped = false;
            for(int jj = offset_j; jj <= offset_j + 2; jj++)
              for(int ii = offset_i; ii <= offset_i + 2; ii++) clipped = clipped || (in[(ptrdiff_t)jj * width + ii] > clip);
          }
  }
  if(!clipped)
  {
    out[0] = in[0];
    return;
  }
  float mean[3] = { 0.0f, 0.0f, 0.0f }, mx[3] = { -FLT_MAX, -FLT_MAX, -FLT_MAX };
  int cnt[3] = { 0, 0, 0 };
  for(int jj = -1; jj <= 1; jj++)
    for(int ii = -1; ii <= 1; ii++)
    {
      const float val = in[(ptrdiff_t)jj * width + ii];
      const int c = fcx(X, j + jj, i + ii);
#pragma unroll
      for(int q = 0; q < 3; q++)
        if(q == c)
        {
          mean[q] += val;
          cnt[q]++;
          mx[q] = mx[q] > val ? mx[q] : val;
        }
    }
  const float m0 = mean[0] / (float)cnt[0], m1 = mean[1] / (float)cnt[1], m2 = mean[2] / (float)cnt[2];
  const float Ro = m0 < clip ? m0 : clip, Go = m1 < clip ? m1 : clip, Bo = m2 < clip ? m2 : clip;
  const float R = mx[0], G = mx[1], B = mx[2];
  const float L = divr(R + G + B, 3.0f);
  float C = x87::mul_sqrt3(R - G);
  float H = 2.0f * B - G - R;
  const float Co = x87::mul_sqrt3(Ro - Go);
  const float Ho = 2.0f * Bo - Go - Ro;
  if(R != G && G != B)
  {
    const float ratio = sqrtf((Co * Co + Ho * Ho) / (C * C + H * H));
    C *= ratio;
    H *= ratio;
  }
  const float t = L - divr(H, 6.0f);
  const int c = fcx(X, j, i);
  out[0] = c == 0 ? x87::add_div_sqrt12(t, C, +1) : (c == 1 ? x87::add_div_sqrt12(t, C, -1) : L + divr(H, 3.0f));
}

// ---- the float -> integer ends ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned gamma_byte(float x)
{ // (uint8_t)(fminf(roundf(255.0f * fmaxf(in, 0.0f)), 255.0f)), gamma.c:361
  return (unsigned)(int)fminf(roundf(255.0f * fmaxf(x, 0.0f)), 255.0f);
}
// BGR into bytes 0..2 of every output pixel; byte 3 keeps what the buffer held
__global__ void __launch_bounds__(NT) gamma_kernel(const float4 *__restrict__ in, unsigned *__restrict__ out, size_t npixels)
{
  const size_t k = (size_t)blockIdx.x * NT + threadIdx.x;
  if(k >= npixels) return;
  const float4 p = in[k];
  out[k] = (out[k] & 0xff000000u) | (gamma_byte(p.x) << 16) | (gamma_byte(p.y) << 8) | gamma_byte(p.z);
}
__device__ __forceinline__ unsigned export_byte(float x)
{ // (uint8_t)CLAMPF(roundf(x * 255.f), 0.f, 255.f) with CLAMPF of math/math.h:91: NaN -> 0
  const float r = roundf(x * 255.f);
  return (unsigned)(int)(r >= 0.f ? (r <= 255.f ? r : 255.f) : 0.f);
}
__device__ __forceinline__ unsigned export_word(float x)
{ // (uint16_t)CLAMP(roundf(x * 65535.f), 0.f, 65535.f) with glib's CLAMP: NaN reaches the conversion, which yields
  // INT_MIN on the reference's hardware (cvttss2si), whose low 16 bits are 0
  const float r = roundf(x * 65535.f);
  const float c = r > 65535.f ? 65535.f : (r < 0.f ? 0.f : r);
  return (c != c) ? 0u : (unsigned)(int)c;
}
template <int FORMAT> __global__ void __launch_bounds__(NT) export_kernel(const float4 *__restrict__ in, void *__restrict__ out, size_t npixels)
{
  const size_t k = (size_t)blockIdx.x * NT + threadIdx.x;
  if(k >= npixels) return;
  const float4 p = in[k];
  if(FORMAT == B200_EXPORT_UINT8)
    ((unsigned *)out)[k] = export_byte(p.x) | (export_byte(p.y) << 8) | (export_byte(p.z) << 16) | (export_byte(p.w) << 24);
  else if(FORMAT == B200_EXPORT_UINT8_SWAP)
    ((unsigned *)out)[k] = export_byte(p.z) | (export_byte(p.y) << 8) | (export_byte(p.x) << 16) | (export_byte(p.w) << 24);
  else
    ((uint2 *)out)[k] = make_uint2(export_word(p.x) | (export_word(p.y) << 16), export_word(p.z) | (export_word(p.w) << 16));
}

// ---- host-side set-up shared with tests/emul: pure functions of the piece ----------------------------------------------------
int proper_crop(const b200_piece_t *piece, int value)
{ // compute_proper_crop, rawprepare.c:206-210: the double product becomes roundf's float argument
  return (int)roundf((float)((double)value * piece->roi_in.scale));
}
bool is_mosaic(const b200_piece_t *p) { return p->filters && p->channels == 1; }
bool bayer_typed(const b200_piece_t *p) { return is_mosaic(p) && (p->datatype == B200_TYPE_UINT16 || p->datatype == B200_TYPE_FLOAT); }

// everything of prepare_t but the device copy of the gain maps; 0 = ok, 1 = the crop does not fit, 2 = bad gain maps
int fill_prepare(const b200_piece_t *piece, prepare_t *P)
{
  const b200_rawprepare_data_t *d = (const b200_rawprepare_data_t *)piece->data;
  memset(P, 0, sizeof(*P));
  for(int k = 0; k < 4; k++)
  {
    P->sub[k] = d->sub[k];
    P->inv_div[k] = 1.0f / d->div[k]; // :483, on the host in the reference too
  }
  P->in_width = piece->roi_in.width;
  P->csx = proper_crop(piece, d->x);
  P->csy = proper_crop(piece, d->y);
  P->roi_x = piece->roi_out.x;
  P->roi_y = piece->roi_out.y;
  P->cfa_x = P->roi_x + d->x;
  P->cfa_y = P->roi_y + d->y;
  if(P->csx < 0 || P->csy < 0 || P->csx + piece->roi_out.width > piece->roi_in.width || P->csy + piece->roi_out.height > piece->roi_in.height) return 1;
  if(d->apply_gainmaps && is_mosaic(piece))
  {
    const b200_dng_gain_map_t *g0 = d->gainmaps[0];
    if(!g0 || !d->gainmaps[1] || !d->gainmaps[2] || !d->gainmaps[3]) return 2;
    if(g0->map_points_h < 1 || g0->map_points_v < 1 || piece->buf_in_width < 1 || piece->buf_in_height < 1) return 2;
    for(int f = 1; f < 4; f++)
      if(d->gainmaps[f]->map_points_h != g0->map_points_h || d->gainmaps[f]->map_points_v != g0->map_points_v) return 2;
    P->gain = 1;
    P->map_w = g0->map_points_h;
    P->map_h = g0->map_points_v;
    P->im_to_rel_x = 1.0f / (float)piece->buf_in_width;
    P->im_to_rel_y = 1.0f / (float)piece->buf_in_height;
    P->rel_to_map_x = (float)(1.0 / g0->map_spacing_h); // 1.0f / double: a double division, rounded to float on assignment
    P->rel_to_map_y = (float)(1.0 / g0->map_spacing_v);
    P->map_origin_h = (float)g0->map_origin_h;
    P->map_origin_v = (float)g0->map_origin_v;
  }
  return 0;
}
void make_balance(const b200_piece_t *piece, balance_t *B)
{
  const b200_temperature_data_t *d = (const b200_temperature_data_t *)piece->data;
  for(int k = 0; k < 4; k++) B->coeffs[k] = d->coeffs[k];
  B->filters = piece->filters;
  B->roi_x = piece->roi_out.x;
  B->roi_y = piece->roi_out.y;
}
// thresholds of the bypass test and the clip value, highlights.c:716-729
void make_thresholds(const b200_piece_t *piece, float thresholds[4], float *clip)
{
  const b200_highlights_data_t *d = (const b200_highlights_data_t *)piece->data;
  float pmax[4];
  for(int c = 0; c < 4; c++) pmax[c] = (piece->processed_maximum[c] > 0.f) ? piece->processed_maximum[c] : 1.0f;
  *clip = d->clip * fminf(pmax[0], fminf(pmax[1], pmax[2]));
  float factor = 0.f;
  if(d->mode == B200_HIGHLIGHTS_INPAINT) factor = 0.987f;
  if(d->mode == B200_HIGHLIGHTS_LAPLACIAN || d->mode == B200_HIGHLIGHTS_HARMONIC) factor = 0.995f;
  for(int c = 0; c < 3; c++) thresholds[c] = (factor > 0.f) ? factor * d->clip * pmax[c] : *clip;
  thresholds[3] = *clip;
}
} // namespace

#ifndef B200_KERNELS_ON_CPU
using namespace b200;

namespace
{
size_t rawprepare_in_bytes(const b200_piece_t *p)
{
  const size_t n = (size_t)p->roi_in.width * p->roi_in.height;
  return bayer_typed(p) && p->datatype == B200_TYPE_UINT16 ? n * 2 : n * 4 * p->channels;
}

int check_piece(const char *op, const b200_piece_t *piece, const void *in, const void *out, size_t data_size)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "%s: NULL argument", op);
  if(data_size && (!piece->data || piece->data_size < data_size)) return fail(B200_ERR_ARG, "%s: piece->data is not the module's data block", op);
  if(in == out) return fail(B200_ERR_ARG, "%s: in-place processing is not supported", op);
  if(piece->roi_out.width < 1 || piece->roi_out.height < 1 || piece->roi_out.height > 65535)
    return fail(B200_ERR_ARG, "%s: roi_out %d x %d", op, piece->roi_out.width, piece->roi_out.height);
  return B200_OK;
}

// fill prepare_t from a rawprepare piece and upload the gain maps (stream-ordered) when there are any
int make_prepare(const b200_piece_t *piece, prepare_t *P, cudaStream_t s)
{
  const b200_rawprepare_data_t *d = (const b200_rawprepare_data_t *)piece->data;
  switch(fill_prepare(piece, P))
  {
    case 0: break;
    case 1:
      return fail(B200_ERR_ARG, "rawprepare: roi_out %dx%d at crop %d,%d does not fit roi_in %dx%d", piece->roi_out.width, piece->roi_out.height, P->csx,
                  P->csy, piece->roi_in.width, piece->roi_in.height);
    default: return fail(B200_ERR_ARG, "rawprepare: apply_gainmaps needs four maps of one non-empty size and a non-empty buf_in");
  }
  if(P->gain)
  {
    const size_t plane = (size_t)P->map_w * P->map_h;
    void *dm = nullptr;
    int rc = scratch(SLOT_SMALL + 3, plane * 4 * sizeof(float), &dm);
    if(rc) return rc;
    for(int f = 0; f < 4; f++)
      B200_CUDA_TRY(cudaMemcpyAsync((float *)dm + f * plane, d->gainmaps[f]->map_gain, plane * sizeof(float), cudaMemcpyHostToDevice, s));
    P->maps = (const float *)dm;
  }
  return B200_OK;
}
dim3 row_grid(int width, int height) { return dim3((unsigned)((width + 4 * NT - 1) / (4 * NT)), (unsigned)height); }
unsigned flat_grid(size_t n) { return (unsigned)((n + 4 * NT - 1) / (4 * NT)); }

int counter_buffer(unsigned long long **counter, cudaStream_t s)
{
  void *p = nullptr;
  int rc = scratch(SLOT_SMALL + 2, 256, &p);
  if(rc) return rc;
  B200_CUDA_TRY(cudaMemsetAsync(p, 0, sizeof(unsigned long long), s));
  *counter = (unsigned long long *)p;
  return B200_OK;
}

template <typename T, int STAGES, bool COUNT>
int launch_front(const void *d_in, void *d_out, int width, int height, const prepare_t &P, const balance_t &B, const clip_t &H, unsigned long long *counter,
                 cudaStream_t s)
{
  raw_front_kernel<T, STAGES, COUNT><<<row_grid(width, height), NT, 0, s>>>((const T *)d_in, (float *)d_out, width, height, P, B, H, counter);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
} // namespace

// ---- rawprepare ------------------------------------------------------------------------------------------------------------
extern "C" int b200_rawprepare_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = check_piece("rawprepare", piece, d_in, d_out, sizeof(b200_rawprepare_data_t));
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  const b200_rawprepare_data_t *d = (const b200_rawprepare_data_t *)piece->data;
  const int width = piece->roi_out.width, height = piece->roi_out.height;
  prepare_t P;
  if((rc = make_prepare(piece, &P, s))) return rc;
  if(bayer_typed(piece))
  {
    const balance_t B = {};
    const clip_t H = {};
    if(piece->datatype == B200_TYPE_UINT16) return launch_front<unsigned short, 1, false>(d_in, d_out, width, height, P, B, H, nullptr, s);
    return launch_front<float, 1, false>(d_in, d_out, width, height, P, B, H, nullptr, s);
  }
  if(is_mosaic(piece) && d->apply_gainmaps)
    return fail(B200_ERR_UNSUPPORTED, "rawprepare: gain maps on a mosaic that is neither uint16 nor float (datatype %d)", piece->datatype);
  if(piece->channels < 1) return fail(B200_ERR_ARG, "rawprepare: %u channels", piece->channels);
  const size_t n = (size_t)width * height * piece->channels;
  predownsampled_kernel<<<(unsigned)((n + NT - 1) / NT), NT, 0, s>>>((const float *)d_in, (float *)d_out, width, height, (int)piece->channels,
                                                                      piece->roi_in.width, P.csx, P.csy, d->sub[0], d->div[0]);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
extern "C" int b200_rawprepare_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_piece("rawprepare", piece, in, out, sizeof(b200_rawprepare_data_t));
  if(rc) return rc;
  return through_device(piece, in, rawprepare_in_bytes(piece), out, (size_t)piece->roi_out.width * piece->roi_out.height * 4 * piece->channels, false,
                        b200_rawprepare_process_dev);
}
extern "C" void b200_rawprepare_tiling(const b200_piece_t *piece, b200_tiling_t *t) { default_tiling(piece, t, 4, true); }

// ---- temperature -------------------------------------------------------------------------------------------------------------
extern "C" int b200_temperature_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = check_piece("temperature", piece, d_in, d_out, sizeof(b200_temperature_data_t));
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  const b200_temperature_data_t *d = (const b200_temperature_data_t *)piece->data;
  const int width = piece->roi_out.width, height = piece->roi_out.height;
  if(piece->filters == 9u)
  {
    float lut[36];
    for(int r = 0; r < 6; r++)
      for(int c = 0; c < 6; c++)
      {
        if(piece->xtrans[r][c] > 3) return fail(B200_ERR_ARG, "temperature: xtrans[%d][%d] = %d", r, c, piece->xtrans[r][c]);
        lut[r * 6 + c] = d->coeffs[piece->xtrans[r][c]];
      }
    void *dl = nullptr;
    if((rc = scratch(SLOT_SMALL + 3, sizeof(lut), &dl))) return rc;
    B200_CUDA_TRY(cudaMemcpyAsync(dl, lut, sizeof(lut), cudaMemcpyHostToDevice, s)); // pageable source: staged before the call returns
    balance_xtrans_kernel<<<dim3((unsigned)((width + NT - 1) / NT), (unsigned)height), NT, 0, s>>>((const float *)d_in, (float *)d_out, width, height,
                                                                                                 piece->roi_out.x, piece->roi_out.y, (const float *)dl);
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
  }
  if(piece->filters)
  {
    prepare_t P = {};
    balance_t B;
    make_balance(piece, &B);
    const clip_t H = {};
    return launch_front<float, 2, false>(d_in, d_out, width, height, P, B, H, nullptr, s);
  }
  if(piece->channels < 3) return fail(B200_ERR_ARG, "temperature: %u channels on non-mosaic input", piece->channels);
  if((piece->mask_display & 1) && piece->channels != 4)
    return fail(B200_ERR_UNSUPPORTED, "temperature: mask display on %u-channel input (the reference's alpha copy assumes 4)", piece->channels);
  const size_t npx = (size_t)width * height;
  balance_pixels_kernel<<<(unsigned)((npx + NT - 1) / NT), NT, 0, s>>>((const float *)d_in, (float *)d_out, npx, (int)piece->channels, d->coeffs[0],
                                                                        d->coeffs[1], d->coeffs[2]);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
extern "C" int b200_temperature_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_piece("temperature", piece, in, out, sizeof(b200_temperature_data_t));
  if(rc) return rc;
  const size_t bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 4 * (piece->filters ? 1 : piece->channels);
  // channel counts other than 4 leave part of every output pixel unwritten: carry what the caller's buffer holds
  return through_device(piece, in, bytes, out, bytes, !piece->filters && piece->channels != 4, b200_temperature_process_dev);
}
extern "C" void b200_temperature_tiling(const b200_piece_t *piece, b200_tiling_t *t) { default_tiling(piece, t, 0, true); }

// ---- highlights --------------------------------------------------------------------------------------------------------------
// colour inpainting, both mosaics: the mosaic transposed, the two row directions on the copy and the two column directions on the frame, the row
// planes transposed back (and added on the way), the sum.  X = NULL: Bayer
static int inpaint_sequence(const void *d_in, void *d_out, const inpaint_t &A, const xtable_t *X, const unsigned long long *counter, cudaStream_t s)
{
  const int width = A.width, height = A.height;
  const size_t npx = (size_t)width * height;
  void *t[4];
  int rc;
  for(int k = 0; k < 4; k++)
    if((rc = scratch(SLOT_TMP0 + k, npx * sizeof(float), &t[k]))) return rc;
  float *t_in = (float *)t[0], *t_fwd = (float *)t[1], *t_bwd = (float *)t[2], *up = (float *)t[3], *rows = t_in, *down = (float *)d_out;
  const dim3 tiles((unsigned)((width + 31) / 32), (unsigned)((height + 31) / 32)), tiles_t((unsigned)((height + 31) / 32), (unsigned)((width + 31) / 32));
  const dim3 by_row((unsigned)((height + 127) / 128), 2), by_col((unsigned)((width + 127) / 128), 2), px((unsigned)((width + NT - 1) / NT), (unsigned)height);
  transpose_kernel<false><<<tiles, 256, 0, s>>>((const float *)d_in, nullptr, t_in, width, height, counter);
  B200_CUDA_TRY(cudaGetLastError());
  if(X)
  {
    inpaint_rows_xtrans_kernel<<<by_row, 128, 0, s>>>(t_in, t_fwd, t_bwd, A, *X, counter);
    inpaint_cols_xtrans_kernel<<<by_col, 128, 0, s>>>((const float *)d_in, down, up, A, *X, counter);
  }
  else
  {
    inpaint_rows_kernel<<<by_row, 128, 0, s>>>(t_in, t_fwd, t_bwd, A, counter);
    inpaint_cols_kernel<<<by_col, 128, 0, s>>>((const float *)d_in, down, up, A, counter);
  }
  B200_CUDA_TRY(cudaGetLastError());
  transpose_kernel<true><<<tiles_t, 256, 0, s>>>(t_fwd, t_bwd, rows, height, width, counter); // back to the frame's layout, the two row directions added
  B200_CUDA_TRY(cudaGetLastError());
  if(X)
    inpaint_sum_xtrans_kernel<<<px, NT, 0, s>>>((const float *)d_in, rows, down, up, (float *)d_out, A, *X, counter);
  else
    inpaint_sum_kernel<<<px, NT, 0, s>>>((const float *)d_in, rows, down, up, (float *)d_out, A, counter);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
namespace b200
{ // highlights_laplacian.cu
int highlights_laplacian_dev(const b200_piece_t *piece, const b200_highlights_data_t *d, const void *d_in, void *d_out, const float clips[4],
                             const float *normalization, cudaStream_t s);
}
extern "C" int b200_highlights_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = check_piece("highlights", piece, d_in, d_out, sizeof(b200_highlights_data_t));
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  const b200_highlights_data_t *d = (const b200_highlights_data_t *)piece->data;
  if(d->mode < B200_HIGHLIGHTS_CLIP || d->mode > B200_HIGHLIGHTS_HARMONIC) return fail(B200_ERR_ARG, "highlights: mode %d", d->mode);
  const int width = piece->roi_out.width, height = piece->roi_out.height;
  const bool mosaic = piece->filters != 0;
  const int ch = mosaic ? 1 : (int)piece->channels;
  if(ch < 1) return fail(B200_ERR_ARG, "highlights: %d channels", ch);
  if((piece->mask_display & 1) && (mosaic || ch != 4))
    return fail(B200_ERR_UNSUPPORTED, "highlights: mask display on %s input (the reference's alpha copy runs past the buffers)", mosaic ? "mosaic" : "non-RGBA");
  float thresholds[4], clip;
  make_thresholds(piece, thresholds, &clip);
  const size_t npx = (size_t)width * height, n = npx * ch;
  unsigned long long *counter = nullptr;
  if((rc = counter_buffer(&counter, s))) return rc;
  if(mosaic)
  {
    const prepare_t P = {};
    const balance_t B = {};
    const clip_t H = { clip, fminf(fminf(thresholds[0], thresholds[1]), thresholds[2]) };
    if((rc = launch_front<float, 0, true>(d_in, nullptr, width, height, P, B, H, counter, s))) return rc;
  }
  else
  {
    count_pixels_kernel<<<(unsigned)((npx + NT - 1) / NT), NT, 0, s>>>((const float *)d_in, npx, ch, thresholds[0], thresholds[1], thresholds[2], counter);
    B200_CUDA_TRY(cudaGetLastError());
  }
  // what runs past the bypass: process_clip for CLIP, and for LCh / colour inpainting on non-mosaic input (:739-757)
  const bool clip_mode = d->mode == B200_HIGHLIGHTS_CLIP || (!mosaic && (d->mode == B200_HIGHLIGHTS_LCH || d->mode == B200_HIGHLIGHTS_INPAINT));
  if(clip_mode)
  { // count and branch stay on the device
    flat_kernel<OP_CLIP><<<flat_grid(n), NT, 0, s>>>((const float *)d_in, (float *)d_out, n, clip, 0.0f, (piece->mask_display & 1) ? 1 : 0, counter);
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
  }
  if(mosaic && piece->filters == 9u && (d->mode == B200_HIGHLIGHTS_LCH || d->mode == B200_HIGHLIGHTS_INPAINT))
  { // the X-Trans variants :735-757; FCxtrans takes roi_in
    xtable_t X;
    for(int r = 0; r < 6; r++)
      for(int c = 0; c < 6; c++)
      {
        if(piece->xtrans[r][c] > 2) return fail(B200_ERR_ARG, "highlights: xtrans[%d][%d] = %d", r, c, piece->xtrans[r][c]);
        X.v[r * 6 + c] = piece->xtrans[r][c];
      }
    X.x0 = piece->roi_in.x;
    X.y0 = piece->roi_in.y;
    if(d->mode == B200_HIGHLIGHTS_LCH)
      lch_xtrans_kernel<<<dim3((unsigned)((width + NT - 1) / NT), (unsigned)height), NT, 0, s>>>((const float *)d_in, (float *)d_out, width, height, X, clip, counter);
    else
    {
      float pmax[4];
      for(int c = 0; c < 4; c++) pmax[c] = (piece->processed_maximum[c] > 0.f) ? piece->processed_maximum[c] : 1.0f;
      const inpaint_t A = { { 0.987f * d->clip * pmax[0], 0.987f * d->clip * pmax[1], 0.987f * d->clip * pmax[2], clip }, 9u, width, height };
      if((rc = inpaint_sequence(d_in, d_out, A, &X, counter, s))) return rc;
    }
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
  }
  if(mosaic && piece->filters != 9u && d->mode == B200_HIGHLIGHTS_LCH)
  { // process() :748-757; the kernel reads the counter for the bypass
    lch_bayer_kernel<<<dim3((unsigned)((width + NT - 1) / NT), (unsigned)height), NT, 0, s>>>((const float *)d_in, (float *)d_out, width, height, piece->roi_out.x,
                                                                                             piece->roi_out.y, piece->filters, clip, counter);
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
  }
  if(mosaic && piece->filters != 9u && d->mode == B200_HIGHLIGHTS_INPAINT)
  { // process() :735-746; the bypass stays on the device: the kernels read the counter
    float pmax[4];
    for(int c = 0; c < 4; c++) pmax[c] = (piece->processed_maximum[c] > 0.f) ? piece->processed_maximum[c] : 1.0f;
    inpaint_t A = { { 0.987f * d->clip * pmax[0], 0.987f * d->clip * pmax[1], 0.987f * d->clip * pmax[2], clip },
                    b200_roi_filters(piece->filters, piece->roi_in.x, piece->roi_in.y), width, height };
    return inpaint_sequence(d_in, d_out, A, nullptr, counter, s);
  }
  // another reconstruction mode: only its bypass is built, so the host has to know which way the frame goes
  unsigned long long n_clipped = 0;
  B200_CUDA_TRY(cudaMemcpyAsync(&n_clipped, counter, sizeof(n_clipped), cudaMemcpyDeviceToHost, s));
  B200_CUDA_TRY(cudaStreamSynchronize(s));
  if(n_clipped >= 25ull && d->mode == B200_HIGHLIGHTS_LAPLACIAN) // process() :759-769: the thresholds of the count are the clips it hands over
    return highlights_laplacian_dev(piece, d, d_in, d_out, thresholds, nullptr, s);
  if(n_clipped >= 25ull)
    return fail(B200_ERR_UNSUPPORTED, "highlights: mode %d with %llu clipped samples (harmonic transposition is not built, only its bypass)", d->mode,
                n_clipped);
  flat_kernel<OP_COPY><<<flat_grid(n), NT, 0, s>>>((const float *)d_in, (float *)d_out, n, 0.0f, 0.0f, 0, counter);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
extern "C" int b200_highlights_laplacian_dev(const b200_piece_t *piece, const void *d_in, void *d_out, const float *normalization, void *stream)
{
  int rc = check_piece("highlights", piece, d_in, d_out, sizeof(b200_highlights_data_t));
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  const b200_highlights_data_t *d = (const b200_highlights_data_t *)piece->data;
  if(d->mode != B200_HIGHLIGHTS_LAPLACIAN) return fail(B200_ERR_ARG, "highlights: mode %d is not the guided laplacians", d->mode);
  float thresholds[4], clip;
  make_thresholds(piece, thresholds, &clip);
  return highlights_laplacian_dev(piece, d, d_in, d_out, thresholds, normalization, (cudaStream_t)stream);
}
extern "C" int b200_highlights_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_piece("highlights", piece, in, out, sizeof(b200_highlights_data_t));
  if(rc) return rc;
  const size_t bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 4 * (piece->filters ? 1 : piece->channels);
  return through_device(piece, in, bytes, out, bytes, false, b200_highlights_process_dev);
}
extern "C" void b200_highlights_tiling(const b200_piece_t *piece, b200_tiling_t *t)
{ // highlights.c:575-644
  if(!piece || !t || !piece->data) return;
  const b200_highlights_data_t *d = (const b200_highlights_data_t *)piece->data;
  const unsigned filters = piece->filters;
  if((d->mode == B200_HIGHLIGHTS_LAPLACIAN || d->mode == B200_HIGHLIGHTS_HARMONIC) && filters)
  { // DS_FACTOR 4, MAX_NUM_SCALES 12 (iop/highlights/common.h)
    const float DS = 4.0f;
    const float scale = DS * (float)((double)(float)piece->iscale / piece->roi_in.scale);
    const float final_radius = (float)((int)(1 << d->scales)) / scale;
    int scales = (int)ceilf(log2f(final_radius));
    scales = scales < 1 ? 1 : (scales > 12 ? 12 : scales);
    const int max_filter_radius = 1 << scales;
    t->factor = 2.f + 2.f * 4 + 6.f * 4 / DS;
    t->factor_cl = 2.f + 3.f * 4 + 6.f * 4 / DS;
    t->maxbuf = 1.f / piece->roi_in.height * 4.f / DS;
    t->maxbuf_cl = 1.0f;
    t->overhead = 0;
    t->overlap = (unsigned)(max_filter_radius * 1.5f / DS);
    t->xalign = t->yalign = (filters == 9u) ? 6 : 2;
    return;
  }
  t->factor = 2.0f;
  t->maxbuf = 1.0f;
  t->overhead = 0;
  const unsigned lch = d->mode == B200_HIGHLIGHTS_LCH;
  if(filters == 9u)
  {
    t->xalign = t->yalign = 6;
    t->overlap = lch ? 2 : 0;
  }
  else if(filters)
  {
    t->xalign = t->yalign = 2;
    t->overlap = lch ? 1 : 0;
  }
  else
  {
    t->xalign = t->yalign = 1;
    t->overlap = 0;
  }
}

// ---- rawprepare -> temperature -> highlights(clip) in one pass ------------------------------------------------------------------
extern "C" int b200_rawfront_process_dev(const b200_piece_t *rawprepare, const b200_piece_t *temperature, const b200_piece_t *highlights, const void *d_in,
                                         void *d_out, void *stream)
{
  int rc = check_piece("rawfront", rawprepare, d_in, d_out, sizeof(b200_rawprepare_data_t));
  if(rc) return rc;
  if(!bayer_typed(rawprepare) || rawprepare->filters == 9u) return fail(B200_ERR_UNSUPPORTED, "rawfront: a uint16 or float Bayer mosaic is required");
  const int width = rawprepare->roi_out.width, height = rawprepare->roi_out.height;
  for(const b200_piece_t *p : { temperature, highlights })
    if(p && (p->roi_out.width != width || p->roi_out.height != height || p->filters != rawprepare->filters || p->devid != rawprepare->devid))
      return fail(B200_ERR_ARG, "rawfront: the pieces do not describe one buffer");
  if(temperature && (!temperature->data || temperature->data_size < sizeof(b200_temperature_data_t))) return fail(B200_ERR_ARG, "rawfront: temperature data");
  if(highlights)
  {
    if(!highlights->data || highlights->data_size < sizeof(b200_highlights_data_t)) return fail(B200_ERR_ARG, "rawfront: highlights data");
    if(((const b200_highlights_data_t *)highlights->data)->mode != B200_HIGHLIGHTS_CLIP)
      return fail(B200_ERR_UNSUPPORTED, "rawfront: only the clip mode of highlights fuses (run the modules one by one)");
    if(highlights->mask_display & 1) return fail(B200_ERR_UNSUPPORTED, "rawfront: mask display");
  }
  if((rc = bind_device(rawprepare->devid))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  prepare_t P;
  if((rc = make_prepare(rawprepare, &P, s))) return rc;
  balance_t B = {};
  if(temperature) make_balance(temperature, &B);
  clip_t H = {};
  unsigned long long *counter = nullptr;
  const bool u16 = rawprepare->datatype == B200_TYPE_UINT16;
#define FRONT(ST, CNT)                                                                                                   \
  (u16 ? launch_front<unsigned short, ST, CNT>(d_in, d_out, width, height, P, B, H, counter, s)                          \
       : launch_front<float, ST, CNT>(d_in, d_out, width, height, P, B, H, counter, s))
  if(highlights)
  {
    float thresholds[4];
    make_thresholds(highlights, thresholds, &H.clip);
    H.raw_threshold = fminf(fminf(thresholds[0], thresholds[1]), thresholds[2]);
    if((rc = counter_buffer(&counter, s))) return rc;
    if(temperature)
    {
      if((rc = FRONT(3, true))) return rc;
      return FRONT(7, false);
    }
    if((rc = FRONT(1, true))) return rc;
    return FRONT(5, false);
  }
  return temperature ? FRONT(3, false) : FRONT(1, false);
#undef FRONT
}

// ---- exposure ----------------------------------------------------------------------------------------------------------------
extern "C" int b200_exposure_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = check_piece("exposure", piece, d_in, d_out, sizeof(b200_exposure_data_t));
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  const b200_exposure_data_t *d = (const b200_exposure_data_t *)piece->data;
  if(piece->channels < 1) return fail(B200_ERR_ARG, "exposure: %u channels", piece->channels);
  if((piece->mask_display & 1) && piece->channels != 4)
    return fail(B200_ERR_UNSUPPORTED, "exposure: mask display on %u-channel input (the reference's alpha copy assumes 4)", piece->channels);
  const size_t n = (size_t)piece->roi_out.width * piece->roi_out.height * piece->channels;
  flat_kernel<OP_EXPOSURE><<<flat_grid(n), NT, 0, (cudaStream_t)stream>>>((const float *)d_in, (float *)d_out, n, d->black, d->scale,
                                                                          (piece->mask_display & 1) ? 1 : 0, nullptr);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
extern "C" int b200_exposure_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_piece("exposure", piece, in, out, sizeof(b200_exposure_data_t));
  if(rc) return rc;
  const size_t bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 4 * piece->channels;
  return through_device(piece, in, bytes, out, bytes, false, b200_exposure_process_dev);
}
extern "C" void b200_exposure_tiling(const b200_piece_t *piece, b200_tiling_t *t) { default_tiling(piece, t, 0, false); }

// ---- gamma and the export conversions -------------------------------------------------------------------------------------------
extern "C" int b200_gamma_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = check_piece("gamma", piece, d_in, d_out, 0);
  if(rc) return rc;
  if(piece->mask_display) return fail(B200_ERR_UNSUPPORTED, "gamma: mask and channel displays (GUI previews) are not built");
  if((rc = bind_device(piece->devid))) return rc;
  const size_t npx = (size_t)piece->roi_out.width * piece->roi_out.height;
  gamma_kernel<<<(unsigned)((npx + NT - 1) / NT), NT, 0, (cudaStream_t)stream>>>((const float4 *)d_in, (unsigned *)d_out, npx);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
extern "C" int b200_gamma_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_piece("gamma", piece, in, out, 0);
  if(rc) return rc;
  const size_t npx = (size_t)piece->roi_out.width * piece->roi_out.height;
  return through_device(piece, in, npx * 16, out, npx * 4, true, b200_gamma_process_dev); // the fourth byte of every pixel is the caller's
}
extern "C" void b200_gamma_tiling(const b200_piece_t *piece, b200_tiling_t *t) { default_tiling(piece, t, 0, false); }

extern "C" int b200_export_convert_dev(const void *d_in, void *d_out, size_t width, size_t height, int format, void *stream)
{
  if(!d_in || !d_out || !width || !height) return fail(B200_ERR_ARG, "export_convert: NULL or empty argument");
  const size_t npx = width * height;
  const unsigned grid = (unsigned)((npx + NT - 1) / NT);
  cudaStream_t s = (cudaStream_t)stream;
  switch(format)
  {
    case B200_EXPORT_UINT8: export_kernel<B200_EXPORT_UINT8><<<grid, NT, 0, s>>>((const float4 *)d_in, d_out, npx); break;
    case B200_EXPORT_UINT8_SWAP: export_kernel<B200_EXPORT_UINT8_SWAP><<<grid, NT, 0, s>>>((const float4 *)d_in, d_out, npx); break;
    case B200_EXPORT_UINT16: export_kernel<B200_EXPORT_UINT16><<<grid, NT, 0, s>>>((const float4 *)d_in, d_out, npx); break;
    default: return fail(B200_ERR_ARG, "export_convert: format %d", format);
  }
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
extern "C" int b200_export_convert_host(const void *in, void *out, size_t width, size_t height, int format)
{
  if(!in || !out || !width || !height) return fail(B200_ERR_ARG, "export_convert: NULL or empty argument");
  if(format < B200_EXPORT_UINT8 || format > B200_EXPORT_UINT16) return fail(B200_ERR_ARG, "export_convert: format %d", format);
  const size_t npx = width * height;
  return through_device(-1, in, npx * 16, out, npx * (format == B200_EXPORT_UINT16 ? 8 : 4), false,
                        [=](const void *d_in, void *d_out, void *stream) { return b200_export_convert_dev(d_in, d_out, width, height, format, stream); });
}
#endif // B200_KERNELS_ON_CPU
