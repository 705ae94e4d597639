// local contrast module, local-Laplacian mode: Gaussian pyramid of the padded L channel, six remapped
// pyramids, coarse-to-fine assembly with per-pixel interpolation between the two nearest remappings.
//
// Reference: src/iop/bilat.c process :336-360 (commit_params :296-311: tiling disabled);
// src/pixel/locallaplacian.c  dl :53-58, ll_expand_gaussian :80-118, ll_fill_boundary1/2 :120-145,
// pad_by_replication :147-159, gauss_expand :160-171, gauss_reduce :173-200, ll_pad_input :204-280,
// ll_laplacian :283-293, curve_scalar :295-327, apply_curve :329-352, local_laplacian_internal :354-563.
//
// Every boundary-fill pass of the reference copies already computed neighbours, so each buffer is a pure
// function "value at clamped coordinates": one kernel per pyramid operation, no separate fill passes.
// Mixed precision kept (the 4./256., 24.0, 4.0, 2.0 literals make those expressions double); expf is
// glibc's (flt32_math.cuh).  Bit-identical to the oracle, which is bit-identical to the reference file
// compiled in place.  Whole-image dependency (pad = 2^(levels-1)): no tiling, like the reference.
// Traffic: 8 pyramids x 4/3 x padded frame; HBM-streaming stencils, the curve pass is expf-bound.
#include "runtime.h"
#include "flt32_math.cuh"
#include <math.h>

namespace
{
constexpr int NUM_GAMMA = 6;  // locallaplacian.c:48
constexpr int MAX_LEVELS = 30; // :46
#define CLAMPS(A, L, H) ((A) > (L) ? ((A) < (H) ? (A) : (H)) : (L))

__host__ __device__ inline int dl(int size, int level)
{
  for(int l = 0; l < level; l++) size = (size - 1) / 2 + 1;
  return size;
}
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// ll_expand_gaussian(), :80-118, at interior coordinates of a fine grid of width wd
__device__ __forceinline__ float expand_at(const float *__restrict__ coarse, int i, int j, int wd)
{
  const int cw = (wd - 1) / 2 + 1;
  const float *c = coarse + (size_t)(j / 2) * cw + i / 2;
  switch((i & 1) + 2 * (j & 1))
  {
    case 0:
      return (float)(4. / 256. * (double)(6.0f * (c[-cw] + c[-1] + 6.0f * c[0] + c[1] + c[cw]) + c[-cw - 1] + c[-cw + 1] + c[cw - 1] + c[cw + 1]));
    case 1:
      return (float)(4. / 256. * (24.0 * (double)(c[0] + c[1]) + 4.0 * (double)(c[-cw] + c[-cw + 1] + c[cw] + c[cw + 1])));
    case 2:
      return (float)(4. / 256. * (24.0 * (double)(c[0] + c[cw]) + 4.0 * (double)(c[-1] + c[1] + c[cw - 1] + c[cw + 1])));
    default:
      return .25f * (c[0] + c[1] + c[cw] + c[cw + 1]);
  }
}
__device__ __forceinline__ float expand_clamped(const float *__restrict__ coarse, int i, int j, int wd, int ht)
{
  return expand_at(coarse, clampi(i, 1, ((wd - 1) & ~1) - 1), clampi(j, 1, ((ht - 1) & ~1) - 1), wd);
}

// ll_pad_input(), replication branch :262-273 + pad_by_replication
__global__ void ll_pad_kernel(const float4 *__restrict__ in, float *__restrict__ padded, int wd, int ht, int w, int h, int max_supp)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
  if(i >= w || j >= h) return;
  const int sj = clampi(j - max_supp, 0, ht - 1), si = clampi(i - max_supp, 0, wd - 1);
  padded[(size_t)j * w + i] = __ldg(in + (size_t)sj * wd + si).x * 0.01f;
}

struct reduce_batch_t
{
  const float *in[NUM_GAMMA];
  float *out[NUM_GAMMA];
};
// gauss_reduce() + ll_fill_boundary1, :173-200,120-129; blockIdx.z picks one of up to six pyramids
__global__ void ll_reduce_kernel(const reduce_batch_t b, int wd, int ht)
{
  const int cw = (wd - 1) / 2 + 1, ch = (ht - 1) / 2 + 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
  if(i >= cw || j >= ch) return;
  const float *__restrict__ input = b.in[blockIdx.z];
  const int cj = clampi(j, 1, ch - 2), ci = clampi(i, 1, cw - 2);
  const float w[5] = { 1.f / 16.f, 4.f / 16.f, 6.f / 16.f, 4.f / 16.f, 1.f / 16.f };
  float acc = 0.0f;
  if(ch > 2 && cw > 2)
  {
#pragma unroll
    for(int jj = -2; jj <= 2; jj++)
#pragma unroll
      for(int ii = -2; ii <= 2; ii++) acc += __ldg(input + (size_t)(2 * cj + jj) * wd + 2 * ci + ii) * w[ii + 2] * w[jj + 2];
  }
  b.out[blockIdx.z][(size_t)j * cw + i] = acc;
}

struct curve_args_t
{
  float *out[NUM_GAMMA];
  float gamma[NUM_GAMMA];
  float sigma, shadows, highlights, clarity;
};
// curve_scalar(), :295-327
__device__ __forceinline__ float curve(const f32m::tables_t &tb, float x, float g, float sigma, float shadows, float highlights, float clarity)
{
  const float c = x - g;
  float val;
  if(c > 2 * sigma)
    val = g + sigma + shadows * (c - sigma);
  else if(c < -2 * sigma)
    val = g - sigma + highlights * (c + sigma);
  else if(c > 0.0f)
  {
    const float t = CLAMPS(c / (2.0f * sigma), 0.0f, 1.0f);
    const float t2 = t * t;
    const float mt = 1.0f - t;
    val = g + sigma * 2.0f * mt * t + t2 * (sigma + sigma * shadows);
  }
  else
  {
    const float t = CLAMPS(-c / (2.0f * sigma), 0.0f, 1.0f);
    const float t2 = t * t;
    const float mt = 1.0f - t;
    val = g - sigma * 2.0f * mt * t + t2 * (-sigma - sigma * highlights);
  }
  val += clarity * c * f32m::expf_(tb, (float)((double)(-c * c) / (2.0 * (double)sigma * (double)sigma / (double)3.0f)));
  return val;
}
// apply_curve(), :329-352, for all six gammas at once
__global__ void __launch_bounds__(256) ll_curve_kernel(const float *__restrict__ padded, const curve_args_t a, int w, int h, int max_supp)
{
  __shared__ double tabs[f32m::SMEM_DOUBLES];
  const f32m::tables_t tb = f32m::stage_tables(tabs, threadIdx.y * blockDim.x + threadIdx.x, 256);
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
  if(i >= w || j >= h) return;
  const int cj = clampi(j, max_supp, h - max_supp - 1), ci = clampi(i, max_supp, w - max_supp - 1);
  const float x = __ldg(padded + (size_t)cj * w + ci);
#pragma unroll
  for(int k = 0; k < NUM_GAMMA; k++) a.out[k][(size_t)j * w + i] = curve(tb, x, a.gamma[k], a.sigma, a.shadows, a.highlights, a.clarity);
}

struct assemble_args_t
{
  const float *coarse_out; // output[l+1]
  float *fine_out;         // output[l]
  const float *padded;     // padded[l]
  const float *fine[NUM_GAMMA], *coarse[NUM_GAMMA]; // buf[k][l], buf[k][l+1]
  float gamma[NUM_GAMMA];
};
// gauss_expand + the coefficient loop of local_laplacian_internal, :508-531
__global__ void ll_assemble_kernel(const assemble_args_t a, int pw, int ph)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
  if(i >= pw || j >= ph) return;
  float o = expand_clamped(a.coarse_out, i, j, pw, ph);
  const float v = __ldg(a.padded + (size_t)j * pw + i);
  int hi = 1;
  for(; hi < NUM_GAMMA - 1 && a.gamma[hi] <= v; hi++)
    ;
  const int lo = hi - 1;
  const float al = CLAMPS((v - a.gamma[lo]) / (a.gamma[hi] - a.gamma[lo]), 0.0f, 1.0f);
  const float l0 = __ldg(a.fine[lo] + (size_t)j * pw + i) - expand_clamped(a.coarse[lo], i, j, pw, ph);
  const float l1 = __ldg(a.fine[hi] + (size_t)j * pw + i) - expand_clamped(a.coarse[hi], i, j, pw, ph);
  o += l0 * (1.0f - al) + l1 * al;
  a.fine_out[(size_t)j * pw + i] = o;
}

// :532-538; alpha: the reference leaves it as found in the output buffer -- here the input's alpha is
// carried through (which is also what dt_iop_alpha_copy does when the pipe displays a mask)
__global__ void ll_writeback_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, const float *__restrict__ out0, int wd, int ht, int w, int max_supp)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
  if(i >= wd || j >= ht) return;
  const float4 p = __ldg(in + (size_t)j * wd + i);
  out[(size_t)j * wd + i] = make_float4(100.0f * out0[(size_t)(j + max_supp) * w + max_supp + i], p.y, p.z, p.w);
}
} // namespace

namespace b200
{
int bilateral_grid_dev(const float *d_in, float *d_out, int width, int height, float sigma_s, float sigma_r, float detail, cudaStream_t s);
size_t bilateral_grid_bytes(int width, int height, float sigma_s, float sigma_r);
}
using namespace b200;

// dt_iop_bilat_params_t == dt_iop_bilat_data_t, iop/bilat.c:78-110
static int check_bl(const b200_piece_t *piece, const void *in, void *out)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "bilat: NULL argument");
  if(!piece->data || piece->data_size < sizeof(b200_bilat_data_t)) return fail(B200_ERR_ARG, "bilat: piece->data is not a b200_bilat_data_t");
  const b200_bilat_data_t *d = (const b200_bilat_data_t *)piece->data;
  if(d->mode != B200_BILAT_LOCAL_LAPLACIAN && d->mode != B200_BILAT_BILATERAL) return fail(B200_ERR_ARG, "bilat: mode %d", d->mode);
  if(in == out) return fail(B200_ERR_ARG, "bilat: in-place processing is not supported");
  return B200_OK;
}

extern "C" int b200_bilat_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = check_bl(piece, d_in, d_out);
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  const b200_bilat_data_t *d = (const b200_bilat_data_t *)piece->data;
  cudaStream_t s = (cudaStream_t)stream;
  const int wd = piece->roi_in.width, ht = piece->roi_in.height;
  if(d->mode == B200_BILAT_BILATERAL)
  { // bilat.c:341-353; the alpha copy of :361 is what the slice already does
    const float scale = (float)((double)(float)piece->iscale / piece->roi_in.scale); // dt_dev_get_module_scale: float / double
    return bilateral_grid_dev((const float *)d_in, (float *)d_out, wd, ht, d->sigma_s / scale, d->sigma_r, d->detail, s);
  }
  // local_laplacian(i, o, w, h, d->midtone, d->sigma_s, d->sigma_r, d->detail, 0), bilat.c:354
  const float sigma = d->midtone, shadows = d->sigma_s, highlights = d->sigma_r, clarity = d->detail;
  if(wd <= 1 || ht <= 1) return B200_OK; // :366: returns without touching the output
  const int mn = wd < ht ? wd : ht;
  int num_levels = 31 - __builtin_clz((unsigned)mn);
  if(num_levels > MAX_LEVELS) num_levels = MAX_LEVELS;
  // min(wd,ht) in {2,3} gives a single level and the reference then reads padded[-1] (:417): undefined there
  if(num_levels < 2) return fail(B200_ERR_UNSUPPORTED, "bilat: frames narrower than 4 px are undefined in the reference");
  const int last = num_levels - 1, max_supp = 1 << last;
  const int w = 2 * max_supp + wd, h = 2 * max_supp + ht;

  size_t level_px[MAX_LEVELS], total = 0;
  for(int l = 0; l <= last; l++)
  {
    level_px[l] = (((size_t)dl(w, l) * dl(h, l)) + 63) & ~(size_t)63;
    total += level_px[l];
  }
  void *base = nullptr;
  if((rc = scratch(SLOT_TMP0, total * (2 + NUM_GAMMA) * sizeof(float), &base))) return rc;
  float *padded[MAX_LEVELS], *output[MAX_LEVELS], *buf[NUM_GAMMA][MAX_LEVELS];
  {
    float *p = (float *)base;
    for(int l = 0; l <= last; l++)
    {
      padded[l] = p;
      p += level_px[l];
    }
    for(int l = 0; l <= last; l++)
    {
      output[l] = p;
      p += level_px[l];
    }
    for(int k = 0; k < NUM_GAMMA; k++)
      for(int l = 0; l <= last; l++)
      {
        buf[k][l] = p;
        p += level_px[l];
      }
  }
  const dim3 blk(32, 8);
  auto grid = [&](int gw, int gh, int gz = 1) { return dim3((gw + 31) / 32, (gh + 7) / 8, gz); };

  ll_pad_kernel<<<grid(w, h), blk, 0, s>>>((const float4 *)d_in, padded[0], wd, ht, w, h, max_supp);
  B200_CUDA_TRY(cudaGetLastError());
  for(int l = 1; l <= last; l++)
  { // the padded pyramid; its coarsest level is written straight into output[last] (:417-419)
    reduce_batch_t b = {};
    b.in[0] = padded[l - 1];
    b.out[0] = (l < last) ? padded[l] : output[last];
    const int fw = dl(w, l - 1), fh = dl(h, l - 1);
    ll_reduce_kernel<<<grid((fw - 1) / 2 + 1, (fh - 1) / 2 + 1), blk, 0, s>>>(b, fw, fh);
    B200_CUDA_TRY(cudaGetLastError());
  }
  float gamma[NUM_GAMMA];
  for(int k = 0; k < NUM_GAMMA; k++) gamma[k] = (k + .5f) / (float)NUM_GAMMA;
  {
    curve_args_t c;
    for(int k = 0; k < NUM_GAMMA; k++)
    {
      c.out[k] = buf[k][0];
      c.gamma[k] = gamma[k];
    }
    c.sigma = sigma;
    c.shadows = shadows;
    c.highlights = highlights;
    c.clarity = clarity;
    ll_curve_kernel<<<grid(w, h), blk, 0, s>>>(padded[0], c, w, h, max_supp);
    B200_CUDA_TRY(cudaGetLastError());
  }
  for(int l = 1; l <= last; l++)
  {
    reduce_batch_t b;
    for(int k = 0; k < NUM_GAMMA; k++)
    {
      b.in[k] = buf[k][l - 1];
      b.out[k] = buf[k][l];
    }
    const int fw = dl(w, l - 1), fh = dl(h, l - 1);
    ll_reduce_kernel<<<grid((fw - 1) / 2 + 1, (fh - 1) / 2 + 1, NUM_GAMMA), blk, 0, s>>>(b, fw, fh);
    B200_CUDA_TRY(cudaGetLastError());
  }
  for(int l = last - 1; l >= 0; l--)
  {
    assemble_args_t a;
    a.coarse_out = output[l + 1];
    a.fine_out = output[l];
    a.padded = padded[l];
    for(int k = 0; k < NUM_GAMMA; k++)
    {
      a.fine[k] = buf[k][l];
      a.coarse[k] = buf[k][l + 1];
      a.gamma[k] = gamma[k];
    }
    const int pw = dl(w, l), ph = dl(h, l);
    ll_assemble_kernel<<<grid(pw, ph), blk, 0, s>>>(a, pw, ph);
    B200_CUDA_TRY(cudaGetLastError());
  }
  ll_writeback_kernel<<<grid(wd, ht), blk, 0, s>>>((const float4 *)d_in, (float4 *)d_out, output[0], wd, ht, w, max_supp);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}

extern "C" int b200_bilat_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_bl(piece, in, out);
  if(rc) return rc;
  const size_t bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 16;
  return through_device(piece, in, bytes, out, bytes, false, b200_bilat_process_dev);
}

// bilat.c:296-311: the local Laplacian cannot be tiled (process_tiling_ready = 0); the numbers below are
// what default_tiling_callback would report and local_laplacian_memory_use() (:566-580) as overhead
extern "C" void b200_bilat_tiling(const b200_piece_t *piece, b200_tiling_t *tiling)
{
  if(!piece || !tiling) return;
  if(piece->data && ((const b200_bilat_data_t *)piece->data)->mode == B200_BILAT_BILATERAL)
  { // bilat.c:259-280.  The reference's figures add three grid rows per OpenMP thread of scratch; the device needs the grid only
    const b200_bilat_data_t *d = (const b200_bilat_data_t *)piece->data;
    const float scale = (float)((double)(float)piece->iscale / piece->roi_in.scale);
    const float sigma_s = d->sigma_s / scale;
    const size_t basebuffer = sizeof(float) * piece->channels * (size_t)piece->roi_in.width * piece->roi_in.height;
    const size_t grid = bilateral_grid_bytes(piece->roi_in.width, piece->roi_in.height, sigma_s, d->sigma_r);
    tiling->factor = 2.0f + (float)grid / basebuffer;
    tiling->factor_cl = 2.0f + (float)(2 * grid) / basebuffer; // dt_bilateral_memory_use with OpenCL: two grids
    tiling->maxbuf = fmaxf(1.0f, (float)grid / basebuffer);
    tiling->maxbuf_cl = tiling->maxbuf;
    tiling->overhead = 0;
    tiling->overlap = (unsigned)ceilf(4 * sigma_s);
    tiling->xalign = 1;
    tiling->yalign = 1;
    return;
  }
  tiling->factor = 2.0f;
  tiling->factor_cl = 2.0f;
  tiling->maxbuf = 1.0f;
  tiling->maxbuf_cl = 1.0f;
  tiling->overlap = 0;
  tiling->xalign = 1;
  tiling->yalign = 1;
  const int width = piece->roi_in.width, height = piece->roi_in.height;
  size_t mem = 0;
  if(width > 1 && height > 1)
  {
    const int mn = width < height ? width : height;
    int num_levels = 31 - __builtin_clz((unsigned)mn);
    if(num_levels > MAX_LEVELS) num_levels = MAX_LEVELS;
    const int max_supp = 1 << (num_levels - 1);
    for(int l = 0; l < num_levels; l++) mem += sizeof(float) * (2 + NUM_GAMMA) * (size_t)dl(width + 2 * max_supp, l) * dl(height + 2 * max_supp, l);
  }
  tiling->overhead = mem > 0xffffffffu ? 0xffffffffu : (unsigned)mem;
}
