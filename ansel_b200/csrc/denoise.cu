// denoise (profiled): variance-stabilising transform + edge-aware a-trous wavelets (+ NLM, see nlm.cu).
//
// Reference: src/iop/denoiseprofile.c  process_wavelets :1289-1447, variance_stabilizing_xform
// :1223-1286, compute_wb_factors :1098-1129, set_up_conversion_matrices :1170-1221, the VST pairs
// :852-1089;  src/pixel/eaw.c  eaw_dn_decompose :242-326 (dn_weight :181-195, fast_mexp2f
// math/math.h:303-317), eaw_synthesize :157-175.
//
// Parity contract: C-standard float semantics of that source (no contraction, IEEE division, FTZ),
// glibc's powf/logf/log2f (flt32_math.cuh on the device, the host libm in the plan below).  One
// deliberate difference, the same as in the oracle: the per-channel sum of squared detail
// coefficients is accumulated in FP64 by a fixed-order two-stage reduction and rounded once, where
// the reference's float OpenMP reduction depends on its thread count (eaw.c:236,253).
//
// Cost model per scale (45 MP): decompose reads the input through L1/L2 (25 taps), writes coarse +
// detail (32 B/px), ~1 k instructions/px -> instruction bound; synthesize streams 48 B/px.
#include "runtime.h"
#include "packed_f32.cuh"
#include "flt32_math.cuh"
#include <math.h>
#include <string.h>

namespace
{
#define MAXF(a, b) ((a) > (b) ? (a) : (b))

// math/math.h:303-317, the variant eaw.c uses
__device__ __forceinline__ float mexp2_float(float x)
{
  const float i1 = (float)0x3f800000u, i2 = (float)0x3f000000u;
  const float k0 = i1 + x * (i2 - i1);
  const int ki = k0 >= (float)0x800000u ? (int)k0 : 0;
  return __int_as_float(ki);
}

constexpr int DEC_BX = 32, DEC_BY = 8;

// max(0, t) the way `(0 > t) ? 0 : t` reads for a NaN (it stays one; fmaxf would drop it)
__device__ __forceinline__ float max0_keep_nan(float t)
{
  float r;
  asm("max.NaN.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(t), "f"(0.0f));
  return r;
}

// eaw.c:242-326: one thread per pixel, taps rows-outer / columns-inner, clamp-to-edge.  The two channel pairs of a pixel
// (x y | z w) are the lanes of the packed FP32 instructions: they sit in adjacent registers as the 16-byte load delivers them.
__global__ void __launch_bounds__(DEC_BX *DEC_BY)
    eaw_decompose_kernel(float4 *__restrict__ coarse, const float4 *__restrict__ in, float4 *__restrict__ detail,
                         double *__restrict__ partial, int mult, float inv_sigma2, int width, int height)
{
  const int i = blockIdx.x * DEC_BX + threadIdx.x, j = blockIdx.y * DEC_BY + threadIdx.y;
  double sq[4] = { 0.0, 0.0, 0.0, 0.0 };
  if(i < width && j < height)
  {
    const float4 px = __ldg(in + (size_t)j * width + i);
    // the 25 taps, clamped to the frame: five row pointers, five column offsets
    const float4 *row[5];
    int xs[5];
#pragma unroll
    for(int k = 0; k < 5; k++)
    {
      row[k] = in + (size_t)min(max(j + mult * (k - 2), 0), height - 1) * width;
      xs[k] = min(max(i + mult * (k - 2), 0), width - 1);
    }
    constexpr float filter[5] = { 1.0f / 16.0f, 4.0f / 16.0f, 6.0f / 16.0f, 4.0f / 16.0f, 1.0f / 16.0f };
    f2 sxy = mk2(0.f, 0.f), szw = mk2(0.f, 0.f); // sum[0..1], sum[2..3]
    float wgt = 0.f;                              // the four wgt lanes of the reference hold the same number
    const f2 pxy = mk2(px.x, px.y);
#pragma unroll
    for(int jj = 0; jj < 5; jj++)
    {
#pragma unroll
      for(int ii = 0; ii < 5; ii++)
      {
        const float4 q = __ldg(row[jj] + xs[ii]);
        const f2 dxy = sub2(pxy, mk2(q.x, q.y));
        const float d2 = px.z - q.z;
        const float dot = (dxy.x * dxy.x + dxy.y * dxy.y + d2 * d2) * inv_sigma2;
        const float t = max0_keep_nan(dot * 0.02f - 9.0f);
        // mexp2_float(), math/math.h:303-317
        const float k0 = (float)0x3f800000u + t * ((float)0x3f000000u - (float)0x3f800000u);
        const float w = (filter[ii] * filter[jj]) * __int_as_float(k0 >= (float)0x800000u ? (int)k0 : 0);
        wgt += w;
        sxy = add2(sxy, mk2(w * q.x, w * q.y)); // products per lane, sums packed
        szw = add2(szw, mk2(w * q.z, w * q.w));
      }
    }
    float4 c, d;
    c.x = sxy.x / wgt;
    c.y = sxy.y / wgt;
    c.z = szw.x / wgt;
    c.w = szw.y / wgt;
    d.x = px.x - c.x;
    d.y = px.y - c.y;
    d.z = px.z - c.z;
    d.w = px.w - c.w;
    coarse[(size_t)j * width + i] = c;
    detail[(size_t)j * width + i] = d;
    sq[0] = (double)(d.x * d.x);
    sq[1] = (double)(d.y * d.y);
    sq[2] = (double)(d.z * d.z);
    sq[3] = (double)(d.w * d.w);
  }
  // fixed-order block reduction in FP64: lanes by shuffle tree, then warps in index order
  __shared__ double wsum[DEC_BY][4];
#pragma unroll
  for(int c = 0; c < 4; c++)
  {
    double v = sq[c];
#pragma unroll
    for(int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if(threadIdx.x == 0) wsum[threadIdx.y][c] = v;
  }
  __syncthreads();
  if(threadIdx.x < 4 && threadIdx.y == 0)
  {
    double v = 0.0;
    for(int k = 0; k < DEC_BY; k++) v += wsum[k][threadIdx.x];
    partial[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 4 + threadIdx.x] = v;
  }
}

// second stage: one block sums the per-block partials in a fixed order (strided chunks, then a tree)
__global__ void __launch_bounds__(1024) reduce_partials_kernel(const double *__restrict__ partial, size_t n_blocks, double *__restrict__ out)
{
  __shared__ double sm[1024];
  for(int c = 0; c < 4; c++)
  {
    double v = 0.0;
    for(size_t k = threadIdx.x; k < n_blocks; k += 1024) v += partial[k * 4 + c];
    sm[threadIdx.x] = v;
    __syncthreads();
    for(int s = 512; s > 0; s >>= 1)
    {
      if((int)threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
      __syncthreads();
    }
    if(threadIdx.x == 0) out[c] = sm[0];
    __syncthreads();
  }
}

struct thr_args_t
{
  float sb2, nm1;
  float adjt[4];
};
// variance_stabilizing_xform(), denoiseprofile.c:1223-1286: the data-dependent tail
__global__ void thresholds_kernel(const double *__restrict__ sums, thr_args_t a, float *__restrict__ thrs)
{
  if(threadIdx.x < 4)
  {
    const int c = threadIdx.x;
    float std_x = 1.0f;
    if(c < 3)
    {
      const float var_y = (float)sums[c] / a.nm1;
      std_x = sqrtf(MAXF(1e-6f, var_y - a.sb2));
    }
    thrs[c] = a.adjt[c] * a.sb2 / std_x;
  }
}

// eaw.c:157-175 with the threshold read from device memory
__global__ void __launch_bounds__(256) eaw_synthesize_kernel(float4 *out, const float4 *in, const float4 *__restrict__ detail,
                                                             const float *__restrict__ thrs, float4 boost, size_t npx)
{
  const size_t k = (size_t)blockIdx.x * 256 + threadIdx.x;
  if(k >= npx) return;
  const float t0 = thrs[0], t1 = thrs[1], t2 = thrs[2], t3 = thrs[3];
  const float4 d = __ldcs(detail + k);
  const float4 a = in[k];
  float4 o;
#define SOFT(dv, tv) (MAXF((dv) - (tv), 0.0f) + (((dv) + (tv)) < 0.0f ? ((dv) + (tv)) : 0.0f))
  o.x = a.x + boost.x * SOFT(d.x, t0);
  o.y = a.y + boost.y * SOFT(d.y, t1);
  o.z = a.z + boost.z * SOFT(d.z, t2);
  o.w = a.w + boost.w * SOFT(d.w, t3);
#undef SOFT
  out[k] = o;
}

// ---- variance-stabilising transforms -----------------------------------------------------------
struct vst_args_t
{
  int mode; // 0 = old (precondition/backtransform), 1 = v2 RGB, 2 = Y0U0V0
  float wb[4], expon[4], denom[4], scale[4], bias_wb[4];
  float aa[4], s38[4], s18[4];
  float b, bias, sqrt_3_2;
  float m[3][4]; // toY0U0V0 (forward) or toRGB (backward)
};

__device__ __forceinline__ float lane(const float4 &v, int c) { return c == 0 ? v.x : (c == 1 ? v.y : (c == 2 ? v.z : v.w)); }

__global__ void __launch_bounds__(256) vst_forward_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, size_t npx, const vst_args_t a)
{
  __shared__ double tabs[f32m::SMEM_DOUBLES];
  const f32m::tables_t tb = f32m::stage_tables(tabs, threadIdx.x, 256);
  __syncthreads();
  const size_t k = (size_t)blockIdx.x * 256 + threadIdx.x;
  if(k >= npx) return;
  const float4 p = __ldcs(in + k);
  float o[4];
  if(a.mode == 0)
  { // precondition(), :852-870
#pragma unroll
    for(int c = 0; c < 4; c++) o[c] = 2.0f * sqrtf(fmaxf(0.0f, lane(p, c) / a.aa[c] + a.s38[c]));
  }
  else if(a.mode == 1)
  { // precondition_v2(), :925-941
#pragma unroll
    for(int c = 0; c < 4; c++)
    {
      const float v = lane(p, c) / a.wb[c] + a.b;
      o[c] = 2.0f * f32m::powf_(tb, MAXF(v, 0.0f), a.expon[c]) / a.denom[c];
    }
  }
  else
  { // precondition_Y0U0V0(), :1026-1054
    float tmp[4];
#pragma unroll
    for(int c = 0; c < 4; c++) tmp[c] = f32m::powf_(tb, MAXF(lane(p, c) + a.b, 0.0f), a.expon[c]) * a.scale[c];
#pragma unroll
    for(int c = 0; c < 3; c++)
    {
      float sum = 0.0f;
#pragma unroll
      for(int j = 0; j < 4; j++) sum += a.m[c][j] * tmp[j];
      o[c] = sum;
    }
    o[3] = 0.0f;
  }
  out[k] = make_float4(o[0], o[1], o[2], o[3]);
}

// out = backtransform(acc + residual); residual may be null (NLM path transforms in place)
__global__ void __launch_bounds__(256)
    vst_backward_kernel(const float4 *acc, const float4 *__restrict__ residual, float4 *out, size_t npx, const vst_args_t a)
{
  __shared__ double tabs[f32m::SMEM_DOUBLES];
  const f32m::tables_t tb = f32m::stage_tables(tabs, threadIdx.x, 256);
  __syncthreads();
  const size_t k = (size_t)blockIdx.x * 256 + threadIdx.x;
  if(k >= npx) return;
  float4 p = acc[k];
  if(residual)
  { // "add in the final residue", :1421-1424
    const float4 r = __ldcs(residual + k);
    p.x += r.x;
    p.y += r.y;
    p.z += r.z;
    p.w += r.w;
  }
  float o[4];
  if(a.mode == 0)
  { // backtransform(), :873-899
#pragma unroll
    for(int c = 0; c < 4; c++)
    {
      const float x = lane(p, c), x2 = x * x;
      o[c] = (x < 0.5f) ? 0.0f
                        : a.aa[c] * (1.f / 4.f * x2 + 1.f / 4.f * a.sqrt_3_2 / x - 11.f / 8.f / x2
                                     + 5.f / 8.f * a.sqrt_3_2 / (x * x2) - a.s18[c]);
    }
  }
  else if(a.mode == 1)
  { // backtransform_v2(), :1003-1023
#pragma unroll
    for(int c = 0; c < 4; c++)
    {
      const float x = MAXF(lane(p, c), 0.0f);
      const float delta = x * x + a.bias;
      const float z1 = (x + sqrtf(MAXF(delta, 0.0f))) / a.denom[c];
      o[c] = a.wb[c] * (f32m::powf_(tb, z1, a.expon[c]) - a.b);
    }
  }
  else
  { // backtransform_Y0U0V0(), :1057-1089
    float rgb[4] = { 0.f, 0.f, 0.f, 0.f };
#pragma unroll
    for(int j = 0; j < 3; j++)
#pragma unroll
      for(int c = 0; c < 4; c++) rgb[j] += a.m[j][c] * lane(p, c);
#pragma unroll
    for(int c = 0; c < 4; c++)
    {
      const float x = MAXF(rgb[c], 0.0f);
      const float delta = x * x + a.bias_wb[c];
      const float z1 = (x + sqrtf(MAXF(delta, 0.0f))) * a.scale[c];
      o[c] = f32m::powf_(tb, z1, a.expon[c]) - a.b;
    }
  }
  out[k] = make_float4(o[0], o[1], o[2], o[3]);
}

__global__ void copy_alpha_kernel(const float4 *__restrict__ in, float4 *out, size_t npx)
{
  const size_t k = (size_t)blockIdx.x * 256 + threadIdx.x;
  if(k < npx) out[k].w = in[k].w;
}

// ---- host-side plan (plain C float arithmetic, the host libm) ----------------------------------
struct plan_t
{
  int max_scale;
  float wb[4], p[4];
  float a_eff, b, bias_eff;
  float toY[3][4], toRGB[3][4];
  float aa[4], bb[4];
  float sigma_band[B200_DENOISE_BANDS];
};

// compute_wb_factors(), :1098-1129
void wb_factors(float wb[4], const b200_denoiseprofile_data_t *d, const float coeffs[4], const float pm[4], const float weights[4])
{
  const float wb_mean = (coeffs[0] + coeffs[1] + coeffs[2]) / 3.0f;
  wb[0] = wb[1] = wb[2] = wb[3] = wb_mean;
  if(d->fix_anscombe_and_nlmeans_norm)
  {
    if(wb_mean != 0.0f && d->wb_adaptive_anscombe)
      for(int i = 0; i < 3; i++) wb[i] = coeffs[i];
    else if(wb_mean == 0.0f)
      for(int i = 0; i < 4; i++) wb[i] = 1.0f;
  }
  else
    for(int i = 0; i < 4; i++) wb[i] = weights[i] * pm[i];
}

// invert_matrix(), :1132-1166
bool invert3(float in[3][4], float out[3][4])
{
  const float biga = in[1][1] * in[2][2] - in[1][2] * in[2][1];
  const float bigb = -in[1][0] * in[2][2] + in[1][2] * in[2][0];
  const float bigc = in[1][0] * in[2][1] - in[1][1] * in[2][0];
  const float bigd = -in[0][1] * in[2][2] + in[0][2] * in[2][1];
  const float bige = in[0][0] * in[2][2] - in[0][2] * in[2][0];
  const float bigf = -in[0][0] * in[2][1] + in[0][1] * in[2][0];
  const float bigg = in[0][1] * in[1][2] - in[0][2] * in[1][1];
  const float bigh = -in[0][0] * in[1][2] + in[0][2] * in[1][0];
  const float bigi = in[0][0] * in[1][1] - in[0][1] * in[1][0];
  const float det = in[0][0] * biga + in[0][1] * bigb + in[0][2] * bigc;
  if(det == 0.0f) return false;
  const float cof[3][3] = { { biga, bigd, bigg }, { bigb, bige, bigh }, { bigc, bigf, bigi } };
  for(int r = 0; r < 3; r++)
  {
    for(int c = 0; c < 3; c++) out[r][c] = 1.0f / det * cof[r][c];
    out[r][3] = 0.0f;
  }
  return true;
}

// set_up_conversion_matrices(), :1170-1221
void conversion_matrices(float toY[3][4], float toRGB[3][4], const float wb[4])
{
  float sum_invwb = 1.0f / wb[0] + 1.0f / wb[1] + 1.0f / wb[2];
  sum_invwb *= sqrtf(3);
  toY[0][0] = sum_invwb / wb[0];
  toY[0][1] = sum_invwb / wb[1];
  toY[0][2] = sum_invwb / wb[2];
  toY[0][3] = 0.0f;
  const float sdU = sqrtf(0.5f * 0.5f * wb[0] * wb[0] + 0.5f * 0.5f * wb[2] * wb[2]);
  const float sdV = sqrtf(0.25f * 0.25f * wb[0] * wb[0] + 0.5f * 0.5f * wb[1] * wb[1] + 0.25f * 0.25f * wb[2] * wb[2]);
  for(int c = 0; c < 3; c++)
  {
    toY[1][c] /= sdU;
    toY[2][c] /= sdV;
  }
  toY[1][3] = toY[2][3] = 0.0f;
  if(!invert3(toY, toRGB))
  {
    const float sdY = sqrtf(1.0f / 9.0f * (wb[0] * wb[0] + wb[1] * wb[1] + wb[2] * wb[2]));
    toY[0][0] = toY[0][1] = toY[0][2] = 1.0f / (3.0f * sdY);
    toY[0][3] = 0.0f;
    invert3(toY, toRGB);
  }
}

// the scale-count loop of process_wavelets :1301-1317 and tiling_callback :818-836
int wavelet_max_scale(float roi_scale, int buf_w, int buf_h)
{
  int max_scale = 0;
  const float in_scale = fminf(roi_scale, 1.0f);
  const float big = (float)MAXF(buf_h, buf_w) * 0.2f;
  const float cap = (float)(2 * (2u << (B200_DENOISE_BANDS - 1)) + 1);
  const float supp0 = cap < big ? cap : big;
  const float i0 = log2f((supp0 - 1.0f) * .5f);
  for(; max_scale < B200_DENOISE_BANDS; max_scale++)
  {
    const float supp = (float)(2 * (2u << max_scale) + 1);
    const float supp_in = supp * (1.0f / in_scale);
    const float i_in = log2f((supp_in - 1) * .5f) - 1.0f;
    const float t = 1.0f - (i_in + .5f) / i0;
    if(t < 0.0f) break;
  }
  return max_scale;
}

void make_plan(plan_t *pl, const b200_denoiseprofile_data_t *d, const b200_piece_t *piece, bool nlm)
{
  memset(pl, 0, sizeof(*pl));
  const float roi_scale = (float)piece->roi_in.scale;
  pl->max_scale = wavelet_max_scale(roi_scale, piece->buf_in_width, piece->buf_in_height);
  // wavelets: in_scale = min(scale, 1) :1305; NLM: min(min(scale, 2), 1) :1615 -- the same number
  const float in_scale = fminf(roi_scale, 1.0f);
  const float ww[4] = { 2.0f, 1.0f, 2.0f, 0.0f }, wn[4] = { 1.0f, 1.0f, 1.0f, 0.0f };
  wb_factors(pl->wb, d, piece->wb_coeffs, piece->processed_maximum, nlm ? wn : ww);
  for(int c = 0; c < 3; c++)
  { // MAX(d->shadows + 0.1 * logf(..), 0.0f): the 0.1 makes the expression double, :1348-1351,1514-1516
    const double v = (double)d->shadows + 0.1 * (double)logf(in_scale / pl->wb[c]);
    pl->p[c] = (float)(v > 0.0 ? v : 0.0);
  }
  pl->p[3] = 0.0f;
  const float compensate_p = 0.05f / powf(0.05f, d->shadows);
  if(nlm)
  { // nlmeans_precondition(), :1519-1524
    for(int i = 0; i < 4; i++)
    {
      pl->wb[i] *= d->strength * in_scale;
      pl->aa[i] = d->a[1] * pl->wb[i];
      pl->bb[i] = d->b[1] * pl->wb[i];
    }
  }
  else
  {
    float toY[3][4] = { { 1.0f / 3.0f, 1.0f / 3.0f, 1.0f / 3.0f, 0 }, { 0.5f, 0.0f, -0.5f, 0 }, { 0.25f, -0.5f, 0.25f, 0 } };
    float toRGB[3][4] = { { 0 } };
    conversion_matrices(toY, toRGB, pl->wb);
    const float cs = (d->wavelet_color_mode == B200_DENOISE_RGB) ? 1.0f : 2.5f;
    for(int k = 0; k < 3; k++)
      for(int c = 0; c < 4; c++)
      {
        toY[k][c] /= (d->strength * cs * in_scale);
        toRGB[k][c] *= (d->strength * cs * in_scale);
      }
    for(int i = 0; i < 4; i++) pl->wb[i] *= d->strength * cs * in_scale;
    memcpy(pl->toY, toY, sizeof(toY));
    memcpy(pl->toRGB, toRGB, sizeof(toRGB));
    for(int c = 0; c < 3; c++)
    {
      pl->aa[c] = d->a[1] * pl->wb[c];
      pl->bb[c] = d->b[1] * pl->wb[c];
    }
  }
  pl->a_eff = d->a[1] * compensate_p;
  pl->b = d->b[1];
  pl->bias_eff = (float)((double)d->bias - 0.5 * (double)logf(in_scale));
  const float varf = sqrtf(2.0f + 2.0f * 4.0f * 4.0f + 6.0f * 6.0f) / 16.0f;
  for(int s = 0; s < B200_DENOISE_BANDS; s++) pl->sigma_band[s] = powf(varf, (float)s) * 1.0f;
}

void vst_args(vst_args_t *v, const plan_t *pl, const b200_denoiseprofile_data_t *d, bool forward, bool nlm)
{
  memset(v, 0, sizeof(*v));
  v->mode = !d->use_new_vst ? 0 : ((nlm || d->wavelet_color_mode == B200_DENOISE_RGB) ? 1 : 2);
  const float sa = sqrtf(pl->a_eff);
  for(int c = 0; c < 4; c++)
  {
    v->wb[c] = pl->wb[c];
    v->aa[c] = pl->aa[c];
  }
  for(int c = 0; c < 3; c++)
  {
    v->s38[c] = (pl->bb[c] / pl->aa[c]) * (pl->bb[c] / pl->aa[c]) + 3.f / 8.f;
    v->s18[c] = (pl->bb[c] / pl->aa[c]) * (pl->bb[c] / pl->aa[c]) + 1.f / 8.f;
    if(forward)
    {
      v->expon[c] = -pl->p[c] / 2 + 1;
      v->denom[c] = (-pl->p[c] + 2) * sa;
      v->scale[c] = 2.0f / ((-pl->p[c] + 2) * sa);
    }
    else
    {
      v->expon[c] = 1.0f / (1.0f - pl->p[c] / 2.0f);
      v->denom[c] = 4.0f / (sa * (2.0f - pl->p[c]));
      v->scale[c] = (sa * (2.0f - pl->p[c])) / 4.0f;
      v->bias_wb[c] = pl->bias_eff * pl->wb[c];
    }
  }
  v->expon[3] = v->denom[3] = v->scale[3] = 1.0f;
  v->b = pl->b;
  v->bias = pl->bias_eff;
  v->sqrt_3_2 = sqrtf(3.0f / 2.0f);
  memcpy(v->m, forward ? pl->toY : pl->toRGB, sizeof(v->m));
}

// the parameter-dependent head of variance_stabilizing_xform(), :1223-1283
void threshold_args(thr_args_t *t, int scale, int max_scale, size_t npixels, float sigma_band, const b200_denoiseprofile_data_t *d)
{
  t->sb2 = sigma_band * sigma_band;
  t->nm1 = (float)npixels - 1.0f;
  float adjt[4] = { 8.0f, 8.0f, 8.0f, 0.0f };
  const int offset_scale = B200_DENOISE_BANDS - max_scale;
  const int band = B200_DENOISE_BANDS - (scale + offset_scale + 1);
  if(d->wavelet_color_mode == B200_DENOISE_RGB)
  {
    float f = d->force[B200_DENOISE_CH_ALL][band];
    f *= f;
    f *= 4;
    for(int c = 0; c < 4; c++) adjt[c] *= f;
    for(int c = 0; c < 3; c++)
    {
      f = d->force[B200_DENOISE_CH_R + c][band];
      f *= f;
      f *= 4;
      adjt[c] *= f;
    }
  }
  else
  {
    float f = d->force[B200_DENOISE_CH_Y0][band];
    f *= f;
    f *= 4;
    adjt[0] *= f;
    f = d->force[B200_DENOISE_CH_U0V0][band];
    f *= f;
    f *= 4;
    adjt[1] *= f;
    adjt[2] *= f;
  }
  memcpy(t->adjt, adjt, sizeof(adjt));
}

int decompose_launch(float4 *coarse, const float4 *in, float4 *detail, double *partial, double *sums, int scale,
                     float inv_sigma2, int width, int height, cudaStream_t s)
{
  using namespace b200;
  const dim3 grid((width + DEC_BX - 1) / DEC_BX, (height + DEC_BY - 1) / DEC_BY), block(DEC_BX, DEC_BY);
  eaw_decompose_kernel<<<grid, block, 0, s>>>(coarse, in, detail, partial, 1 << scale, inv_sigma2, width, height);
  B200_CUDA_TRY(cudaGetLastError());
  reduce_partials_kernel<<<1, 1024, 0, s>>>(partial, (size_t)grid.x * grid.y, sums);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
size_t partial_bytes(int width, int height)
{
  return (size_t)((width + DEC_BX - 1) / DEC_BX) * ((height + DEC_BY - 1) / DEC_BY) * 4 * sizeof(double) + 64;
}
} // namespace

namespace b200
{
int denoiseprofile_nlmeans_dev(const b200_piece_t *piece, const b200_denoiseprofile_data_t *d, const float *d_in, float *d_out,
                               cudaStream_t s);
int nlmeans_denoise_dev(const float *d_in, float *d_out, int width, int height, float scattering, float scale, float luma,
                        float chroma, float center_weight, float sharpness, int radius, int search_radius, int decimate,
                        const float norm[4], cudaStream_t stream);

// shared with nlm.cu: forward / backward VST for the NLM mode of denoiseprofile (:1500-1597)
int denoise_vst_forward(const b200_piece_t *piece, const b200_denoiseprofile_data_t *d, const float *d_in, float *d_out,
                        size_t npx, bool nlm, cudaStream_t s)
{
  plan_t pl;
  make_plan(&pl, d, piece, nlm);
  vst_args_t v;
  vst_args(&v, &pl, d, true, nlm);
  vst_forward_kernel<<<(unsigned)((npx + 255) / 256), 256, 0, s>>>((const float4 *)d_in, (float4 *)d_out, npx, v);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
int denoise_vst_backward(const b200_piece_t *piece, const b200_denoiseprofile_data_t *d, float *d_buf, size_t npx, bool nlm,
                         cudaStream_t s)
{
  plan_t pl;
  make_plan(&pl, d, piece, nlm);
  vst_args_t v;
  vst_args(&v, &pl, d, false, nlm);
  vst_backward_kernel<<<(unsigned)((npx + 255) / 256), 256, 0, s>>>((const float4 *)d_buf, nullptr, (float4 *)d_buf, npx, v);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
// dt_iop_alpha_copy() as both modes of denoiseprofile end with it when a mask is displayed (denoiseprofile.c:1645-1646)
int denoise_alpha_copy(const float *d_in, float *d_out, size_t npx, cudaStream_t s)
{
  copy_alpha_kernel<<<(unsigned)((npx + 255) / 256), 256, 0, s>>>((const float4 *)d_in, (float4 *)d_out, npx);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
} // namespace b200

using namespace b200;

extern "C" int b200_eaw_dn_decompose_dev(void *d_coarse, const void *d_in, void *d_detail, double *d_sum_squared, int scale,
                                         float inv_sigma2, int width, int height, void *stream)
{
  if(!d_coarse || !d_in || !d_detail || !d_sum_squared || scale < 0 || scale > 12 || width <= 0 || height <= 0)
    return fail(B200_ERR_ARG, "eaw_dn_decompose: bad arguments");
  int rc = bind_device(-1);
  if(rc) return rc;
  void *partial = nullptr;
  if((rc = scratch(SLOT_SMALL, partial_bytes(width, height), &partial))) return rc;
  return decompose_launch((float4 *)d_coarse, (const float4 *)d_in, (float4 *)d_detail, (double *)partial, d_sum_squared, scale,
                          inv_sigma2, width, height, (cudaStream_t)stream);
}

extern "C" int b200_eaw_synthesize_dev(void *d_out, const void *d_in, const void *d_detail, const float threshold[4],
                                       const float boost[4], int width, int height, void *stream)
{
  if(!d_out || !d_in || !d_detail || !threshold || !boost || width <= 0 || height <= 0)
    return fail(B200_ERR_ARG, "eaw_synthesize: bad arguments");
  int rc = bind_device(-1);
  if(rc) return rc;
  void *small = nullptr;
  if((rc = scratch(SLOT_SMALL, 4096, &small))) return rc;
  float *d_thr = (float *)((char *)small + 2048);
  cudaStream_t s = (cudaStream_t)stream;
  B200_CUDA_TRY(cudaMemcpyAsync(d_thr, threshold, 16, cudaMemcpyHostToDevice, s));
  const size_t npx = (size_t)width * height;
  eaw_synthesize_kernel<<<(unsigned)((npx + 255) / 256), 256, 0, s>>>((float4 *)d_out, (const float4 *)d_in, (const float4 *)d_detail,
                                                                     d_thr, make_float4(boost[0], boost[1], boost[2], boost[3]), npx);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}

// nlmeans_denoise(), pixel/nlmeans_core.c:315-532, on device RGBA buffers (d_in != d_out)
extern "C" int b200_nlmeans_denoise_dev(const void *d_in, void *d_out, int width, int height, float scattering, float scale,
                                        float luma, float chroma, float center_weight, float sharpness, int patch_radius,
                                        int search_radius, int decimate, const float norm[4], void *stream)
{
  if(!d_in || !d_out || d_in == d_out || width <= 0 || height <= 0 || !norm) return fail(B200_ERR_ARG, "nlmeans_denoise: bad arguments");
  int rc = bind_device(-1);
  if(rc) return rc;
  return nlmeans_denoise_dev((const float *)d_in, (float *)d_out, width, height, scattering, scale, luma, chroma, center_weight,
                             sharpness, patch_radius, search_radius, decimate, norm, (cudaStream_t)stream);
}

// process_wavelets(), denoiseprofile.c:1289-1447
static int process_wavelets_dev(const b200_piece_t *piece, const b200_denoiseprofile_data_t *d, const float *d_in, float *d_out,
                                cudaStream_t s)
{
  const int width = piece->roi_in.width, height = piece->roi_in.height;
  const size_t npx = (size_t)width * height, bytes = npx * 16;
  plan_t pl;
  make_plan(&pl, d, piece, false);
  const int max_mult = 1 << (pl.max_scale - 1);
  if(pl.max_scale < 1 || width < 2 * max_mult || height < 2 * max_mult)
  { // "corner case of extremely small image": plain copy (:1323-1329)
    if(d_in != d_out) B200_CUDA_TRY(cudaMemcpyAsync(d_out, d_in, bytes, cudaMemcpyDeviceToDevice, s));
    return B200_OK;
  }
  int rc;
  void *precond, *tmp, *buf, *small;
  if((rc = scratch(SLOT_TMP0, bytes, &precond))) return rc;
  if((rc = scratch(SLOT_TMP1, bytes, &tmp))) return rc;
  if((rc = scratch(SLOT_TMP2, bytes, &buf))) return rc;
  if((rc = scratch(SLOT_SMALL, partial_bytes(width, height) + 4096, &small))) return rc;
  double *partial = (double *)small;
  double *sums = (double *)((char *)small + partial_bytes(width, height));
  float *thrs = (float *)(sums + 8);

  vst_args_t v;
  vst_args(&v, &pl, d, true, false);
  vst_forward_kernel<<<(unsigned)((npx + 255) / 256), 256, 0, s>>>((const float4 *)d_in, (float4 *)precond, npx, v);
  B200_CUDA_TRY(cudaGetLastError());
  B200_CUDA_TRY(cudaMemsetAsync(d_out, 0, bytes, s));

  float4 *buf1 = (float4 *)precond, *buf2 = (float4 *)tmp;
  for(int sc = 0; sc < pl.max_scale; sc++)
  {
    const float sb = pl.sigma_band[sc];
    if((rc = decompose_launch(buf2, buf1, (float4 *)buf, partial, sums, sc, 1.0f / (sb * sb), width, height, s))) return rc;
    thr_args_t t;
    threshold_args(&t, sc, pl.max_scale, npx, sb, d);
    thresholds_kernel<<<1, 32, 0, s>>>(sums, t, thrs);
    B200_CUDA_TRY(cudaGetLastError());
    eaw_synthesize_kernel<<<(unsigned)((npx + 255) / 256), 256, 0, s>>>((float4 *)d_out, (const float4 *)d_out, (const float4 *)buf, thrs,
                                                                       make_float4(1.f, 1.f, 1.f, 1.f), npx);
    B200_CUDA_TRY(cudaGetLastError());
    float4 *t3 = buf2;
    buf2 = buf1;
    buf1 = t3;
  }
  vst_args(&v, &pl, d, false, false);
  vst_backward_kernel<<<(unsigned)((npx + 255) / 256), 256, 0, s>>>((const float4 *)d_out, buf1, (float4 *)d_out, npx, v);
  B200_CUDA_TRY(cudaGetLastError());
  if(piece->mask_display & B200_DISPLAY_MASK)
  {
    copy_alpha_kernel<<<(unsigned)((npx + 255) / 256), 256, 0, s>>>((const float4 *)d_in, (float4 *)d_out, npx);
    B200_CUDA_TRY(cudaGetLastError());
  }
  return B200_OK;
}

static int check_dn(const b200_piece_t *piece, const void *in, void *out)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "denoiseprofile: NULL argument");
  if(!piece->data || piece->data_size < sizeof(b200_denoiseprofile_data_t))
    return fail(B200_ERR_ARG, "denoiseprofile: piece->data is not a b200_denoiseprofile_data_t");
  if(piece->roi_in.width != piece->roi_out.width || piece->roi_in.height != piece->roi_out.height)
    return fail(B200_ERR_ARG, "denoiseprofile: roi_in and roi_out differ");
  if(in == out) return fail(B200_ERR_ARG, "denoiseprofile: in-place processing is not supported");
  return B200_OK;
}

extern "C" int b200_denoiseprofile_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = check_dn(piece, d_in, d_out);
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  const b200_denoiseprofile_data_t *d = (const b200_denoiseprofile_data_t *)piece->data;
  cudaStream_t s = (cudaStream_t)stream;
  if(d->mode == B200_DENOISE_WAVELETS || d->mode == B200_DENOISE_WAVELETS_AUTO)
    return process_wavelets_dev(piece, d, (const float *)d_in, (float *)d_out, s);
  if(d->mode == B200_DENOISE_NLMEANS || d->mode == B200_DENOISE_NLMEANS_AUTO)
    return denoiseprofile_nlmeans_dev(piece, d, (const float *)d_in, (float *)d_out, s);
  return fail(B200_ERR_UNSUPPORTED, "denoiseprofile: variance-measurement mode (GUI aid) is not built");
}

extern "C" int b200_denoiseprofile_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_dn(piece, in, out);
  if(rc) return rc;
  const size_t bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 16;
  return through_device(piece, in, bytes, out, bytes, false, b200_denoiseprofile_process_dev);
}

// tiling_callback(), denoiseprofile.c:796-849
extern "C" void b200_denoiseprofile_tiling(const b200_piece_t *piece, b200_tiling_t *tiling)
{
  if(!piece || !tiling || !piece->data) return;
  const b200_denoiseprofile_data_t *d = (const b200_denoiseprofile_data_t *)piece->data;
  const float rs = (float)piece->roi_in.scale;
  if(d->mode == B200_DENOISE_NLMEANS || d->mode == B200_DENOISE_NLMEANS_AUTO)
  {
    const int P = (int)ceilf(d->radius * fminf(fminf(rs, 2.0f), 1.0f));
    const int K = (int)ceilf(d->nbhood * fminf(fminf(rs, 2.0f), 1.0f));
    const int K_scattered = (int)ceilf(d->scattering * (K * K * K + 7.0 * K * sqrt((double)K)) / 6.0) + K;
    (void)P;
    tiling->factor = 2.0f + 0.25f;
    tiling->factor_cl = 4.0f + 0.25f * 4; // NUM_BUCKETS 4, denoiseprofile.c:104
    tiling->maxbuf = 1.0f;
    tiling->maxbuf_cl = 1.0f;
    tiling->overhead = 0;
    tiling->overlap = P + K_scattered;
    tiling->xalign = 1;
    tiling->yalign = 1;
  }
  else
  {
    const int max_scale = wavelet_max_scale(rs, piece->buf_in_width, piece->buf_in_height);
    tiling->factor = 5.0f;
    tiling->factor_cl = 3.5f + max_scale;
    tiling->maxbuf = 1.0f;
    tiling->maxbuf_cl = 1.0f;
    tiling->overhead = 0;
    tiling->overlap = 1u << max_scale;
    tiling->xalign = 1;
    tiling->yalign = 1;
  }
}
