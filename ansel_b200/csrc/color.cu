// colorin / colorout: matrix + tone-curve colour conversion, pointwise RGBA -> RGBA.
//
// Reference arithmetic: src/colorprofiles/conversion.c  _apply_matrix :593-682,
// _apply_target_curves :546-583, _clamp_unit :536-543; dt_mat3x4_mul_vec4 system/simd.h:188-197;
// dt_ioppr_eval_trc / extrapolate_lut / eval_exp colorprofiles/iop_profile.h:536-580.
// Callers: iop/colorin.c:711-734, iop/colorout.c:373-389.
//
// Roofline: pure streaming, 16 B in + 16 B out per pixel (32 B/px algorithmic, SURVEY.md 8d); the
// 768 KB of tone curves stay in L2.  The reference makes a second pass over the output for the
// target curves; the per-pixel arithmetic is identical when fused, so it is one pass here.
// 3x3 (x4 lanes) per pixel is ~21 flop per 32 B: three orders of magnitude under the tensor-core
// ridge, and TF32 inputs would break bit parity, so this is CUDA-core FMA by design.
//
// Rounding flavours (include/b200iop.h B200_FP_*): CONTRACT reproduces, operation for operation,
// what gcc 13 makes of the reference's release flags on FMA hardware -- fma(r2,z, fma(r0,x, r1*y))
// for the matrix, fma(l1,1-f, l2*f) for the target-curve lerp, fma(l2,f, l1*(1-f)) for the
// source-curve lerp -- and is pinned bit-for-bit against oracle/_ref/libref_fast.so; STRICT rounds
// every multiply and add (pinned against libref_strict.so).  The library is compiled with
// --fmad=false, so the only fused operations are the explicit ones below.
#include "runtime.h"
#include "flt32_math.cuh"
#include "trc.cuh"
#include <mutex>

namespace
{
struct conv_args_t
{
  const float4 *in;
  float4 *out;
  unsigned long long npx;
  float m[9], cm[9];
  const float *lut_s[3]; // device pointers, nullptr = channel passes through
  const float *lut_t[3];
  float co_s[9], co_t[9];
  int decode, encode, clip, copy_alpha;
  // further destinations of the same pixels: peer GPUs' copies of the frame (b200_apply_conversion_scatter_dev)
  int n_mirror;
  float4 *mirror[B200_MAX_SCATTER - 1];
};

template <bool CONTRACT> __device__ __forceinline__ float4 mat4(const float *m, float x, float y, float z)
{
  float o[4];
#pragma unroll
  for(int i = 0; i < 4; i++)
  {
    // lane 3 multiplies zeros like the padded dt_colormatrix_t row does (sign of zero and NaN included)
    const float a = i < 3 ? m[3 * i] : 0.0f, b = i < 3 ? m[3 * i + 1] : 0.0f, c = i < 3 ? m[3 * i + 2] : 0.0f;
    float acc;
    if(CONTRACT)
    {
      acc = __fmaf_rn(a, x, __fmul_rn(b, y));
      acc = __fmaf_rn(c, z, acc);
    }
    else
    {
      acc = __fadd_rn(__fmul_rn(a, x), __fmul_rn(b, y));
      acc = __fadd_rn(__fmul_rn(c, z), acc);
    }
    o[i] = acc;
  }
  return make_float4(o[0], o[1], o[2], o[3]);
}

__device__ __forceinline__ float clamp01(float v) { return v > 1.0f ? 1.0f : (v < 0.0f ? 0.0f : v); }

constexpr int CONV_THREADS = 256;
constexpr int CONV_PER_THREAD = 4;

template <bool CONTRACT> __global__ void __launch_bounds__(CONV_THREADS) convert_kernel(const conv_args_t a)
{
  const f32m::tables_t tb = f32m::global_tables();
  const unsigned long long base = (unsigned long long)blockIdx.x * (CONV_THREADS * CONV_PER_THREAD) + threadIdx.x;
  float4 px[CONV_PER_THREAD];
#pragma unroll
  for(int j = 0; j < CONV_PER_THREAD; j++)
  {
    const unsigned long long k = base + (unsigned long long)j * CONV_THREADS;
    if(k < a.npx) px[j] = __ldcs(a.in + k);
  }
#pragma unroll
  for(int j = 0; j < CONV_PER_THREAD; j++)
  {
    const unsigned long long k = base + (unsigned long long)j * CONV_THREADS;
    if(k >= a.npx) continue;
    float4 p = px[j];
    const float alpha_in = p.w;
    if(a.decode)
    {
      if(a.lut_s[0]) p.x = eval_trc<CONTRACT, true>(tb, p.x, a.lut_s[0], a.co_s + 0);
      if(a.lut_s[1]) p.y = eval_trc<CONTRACT, true>(tb, p.y, a.lut_s[1], a.co_s + 3);
      if(a.lut_s[2]) p.z = eval_trc<CONTRACT, true>(tb, p.z, a.lut_s[2], a.co_s + 6);
    }
    float4 v = mat4<CONTRACT>(a.m, p.x, p.y, p.z);
    if(a.clip) v = mat4<CONTRACT>(a.cm, clamp01(v.x), clamp01(v.y), clamp01(v.z));
    if(a.encode)
    {
      if(a.lut_t[0]) v.x = eval_trc<CONTRACT, false>(tb, v.x, a.lut_t[0], a.co_t + 0);
      if(a.lut_t[1]) v.y = eval_trc<CONTRACT, false>(tb, v.y, a.lut_t[1], a.co_t + 3);
      if(a.lut_t[2]) v.z = eval_trc<CONTRACT, false>(tb, v.z, a.lut_t[2], a.co_t + 6);
    }
    if(a.copy_alpha) v.w = alpha_in; // dt_iop_alpha_copy when the pipe displays a mask
    __stcs(a.out + k, v);
    // the all-gather of the finished band, done by the producer: plain stores into the peers' frames over NVLink
    for(int m = 0; m < a.n_mirror; m++) a.mirror[m][k] = v;
  }
}

// ---- device copies of tone curves, keyed by dt_colorspaces_conversion_identity() ---------------
struct lut_entry_t
{
  uint64_t identity;
  int dev;
  int side; // 0 = source, 1 = target
  float *d;  // 3 * LUTN floats
  unsigned long long stamp;
};
constexpr int LUT_CACHE = 16;
lut_entry_t g_luts[LUT_CACHE];
unsigned long long g_stamp = 0;
std::mutex g_lut_mu;

} // namespace

// returns a device pointer holding the three curves of one side (3*LUTN floats)
int b200::device_curves(const float *const host[3], uint64_t identity, int side, cudaStream_t stream, const float **out)
{
  using namespace b200;
  int dev = 0;
  B200_CUDA_TRY(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(g_lut_mu);
  int slot = -1;
  if(identity)
    for(int k = 0; k < LUT_CACHE; k++)
      if(g_luts[k].d && g_luts[k].identity == identity && g_luts[k].dev == dev && g_luts[k].side == side)
      {
        g_luts[k].stamp = ++g_stamp;
        *out = g_luts[k].d;
        return B200_OK;
      }
  // pick a free slot on this device, else the least recently used one of this device, else any free
  unsigned long long best = ~0ull;
  for(int k = 0; k < LUT_CACHE; k++)
    if(!g_luts[k].d)
    {
      slot = k;
      break;
    }
  if(slot < 0)
    for(int k = 0; k < LUT_CACHE; k++)
      if(g_luts[k].dev == dev && g_luts[k].stamp < best)
      {
        best = g_luts[k].stamp;
        slot = k;
      }
  if(slot < 0) return fail(B200_ERR_NOMEM, "tone-curve cache exhausted by other devices");
  if(!g_luts[slot].d)
  {
    cudaError_t e = cudaMalloc(&g_luts[slot].d, sizeof(float) * 3 * LUTN);
    if(e != cudaSuccess)
    {
      g_luts[slot].d = nullptr;
      return fail(B200_ERR_NOMEM, "cudaMalloc(tone curves) failed: %s", cudaGetErrorString(e));
    }
  }
  else
  {
    // reuse: whoever used this buffer last may still be running on another stream
    B200_CUDA_TRY(cudaDeviceSynchronize());
  }
  for(int c = 0; c < 3; c++)
    B200_CUDA_TRY(cudaMemcpyAsync(g_luts[slot].d + (size_t)c * LUTN, host[c], sizeof(float) * LUTN, cudaMemcpyHostToDevice, stream));
  // The entry is published to every stream of this device, so the upload has to have landed first: another pipe (preview and
  // full start together, each on its own non-blocking stream) may hit the cache and launch before this stream got to the copy.
  // Once per profile; it also makes pinned host arrays safe to change after return.
  B200_CUDA_TRY(cudaStreamSynchronize(stream));
  g_luts[slot].identity = identity;
  g_luts[slot].dev = dev;
  g_luts[slot].side = side;
  g_luts[slot].stamp = ++g_stamp;
  *out = g_luts[slot].d;
  return B200_OK;
}

using namespace b200;

static int apply_conversion(const b200_conversion_t *c, const void *d_in, void *d_out, int n_mirror, void *const *mirrors, size_t width,
                            size_t height, int copy_alpha, void *stream_);
extern "C" int b200_apply_conversion_dev(const b200_conversion_t *c, const void *d_in, void *d_out, size_t width,
                                         size_t height, int copy_alpha, void *stream_)
{
  return apply_conversion(c, d_in, d_out, 0, nullptr, width, height, copy_alpha, stream_);
}
extern "C" int b200_apply_conversion_scatter_dev(const b200_conversion_t *c, const void *d_in, int n_out, void *const *d_outs,
                                                 size_t width, size_t height, int copy_alpha, void *stream_)
{
  if(n_out < 1 || n_out > B200_MAX_SCATTER || !d_outs) return fail(B200_ERR_ARG, "apply_conversion_scatter: 1..%d destinations", B200_MAX_SCATTER);
  for(int k = 0; k < n_out; k++)
    if(!d_outs[k]) return fail(B200_ERR_ARG, "apply_conversion_scatter: NULL destination");
  return apply_conversion(c, d_in, d_outs[0], n_out - 1, d_outs + 1, width, height, copy_alpha, stream_);
}
static int apply_conversion(const b200_conversion_t *c, const void *d_in, void *d_out, int n_mirror, void *const *mirrors, size_t width,
                            size_t height, int copy_alpha, void *stream_)
{
  if(!c || !d_in || !d_out) return fail(B200_ERR_ARG, "apply_conversion: NULL argument");
  if(!c->is_matrix)
    return fail(B200_ERR_UNSUPPORTED, "apply_conversion: lcms2 (non-matrix) conversions are not built (SURVEY.md 8c iii)");
  int rc = bind_device(-1);
  if(rc) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  const unsigned long long npx = (unsigned long long)width * height;
  if(!npx) return B200_OK;

  conv_args_t a;
  a.in = (const float4 *)d_in;
  a.out = (float4 *)d_out;
  a.npx = npx;
  a.n_mirror = n_mirror;
  for(int k = 0; k < B200_MAX_SCATTER - 1; k++) a.mirror[k] = k < n_mirror ? (float4 *)mirrors[k] : nullptr;
  for(int i = 0; i < 3; i++)
    for(int j = 0; j < 3; j++)
    {
      a.m[3 * i + j] = c->matrix[i][j];
      a.cm[3 * i + j] = c->clip_matrix[i][j];
      a.co_s[3 * i + j] = c->coeffs_source[i][j];
      a.co_t[3 * i + j] = c->coeffs_target[i][j];
    }
  a.clip = c->has_clipping ? 1 : 0;
  a.copy_alpha = copy_alpha ? 1 : 0;
  // conversion.c:610-611: a side is active when it has curves and at least one is non-linear
  int n_s = 0, n_t = 0;
  const bool have_s = c->lut_source[0] && c->lut_source[1] && c->lut_source[2];
  const bool have_t = c->lut_target[0] && c->lut_target[1] && c->lut_target[2];
  for(int k = 0; k < 3; k++)
  {
    if(have_s && c->lut_source[k][0] >= 0.0f) n_s++;
    if(have_t && c->lut_target[k][0] >= 0.0f) n_t++;
  }
  a.decode = have_s && n_s > 0;
  a.encode = have_t && n_t > 0;
  const float *ds = nullptr, *dt = nullptr;
  if(a.decode && (rc = device_curves(c->lut_source, c->identity, 0, stream, &ds))) return rc;
  if(a.encode && (rc = device_curves(c->lut_target, c->identity, 1, stream, &dt))) return rc;
  for(int k = 0; k < 3; k++)
  {
    a.lut_s[k] = (a.decode && c->lut_source[k][0] >= 0.0f) ? ds + (size_t)k * LUTN : nullptr;
    a.lut_t[k] = (a.encode && c->lut_target[k][0] >= 0.0f) ? dt + (size_t)k * LUTN : nullptr;
  }
  const unsigned long long per_block = CONV_THREADS * CONV_PER_THREAD;
  const unsigned blocks = (unsigned)((npx + per_block - 1) / per_block);
  if(c->fp_mode == B200_FP_STRICT)
    convert_kernel<false><<<blocks, CONV_THREADS, 0, stream>>>(a);
  else
    convert_kernel<true><<<blocks, CONV_THREADS, 0, stream>>>(a);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}

namespace
{
int passthrough(const void *d_in, void *d_out, size_t bytes, cudaStream_t s)
{
  if(d_in != d_out) B200_CUDA_TRY(cudaMemcpyAsync(d_out, d_in, bytes, cudaMemcpyDeviceToDevice, s));
  return B200_OK;
}

// shared body of colorin.c:711-734 and colorout.c:373-389
int color_process_dev(const b200_piece_t *piece, const b200_conversion_t *conv, int type, const void *d_in, void *d_out,
                      void *stream)
{
  int rc = bind_device(piece->devid);
  if(rc) return rc;
  const size_t w = piece->roi_out.width, h = piece->roi_out.height;
  if(type == B200_COLORSPACE_LAB || !conv) // Lab in means Lab out / nothing to convert: dt_iop_image_copy_by_size
    return passthrough(d_in, d_out, w * h * 4 * sizeof(float), (cudaStream_t)stream);
  return b200_apply_conversion_dev(conv, d_in, d_out, w, h, piece->mask_display & B200_DISPLAY_MASK, stream);
}
} // namespace

#define COLOR_CHECK(op, T)                                                                         \
  if(!piece || !in || !out) return fail(B200_ERR_ARG, op ": NULL argument");                      \
  if(!piece->data || piece->data_size < sizeof(T)) return fail(B200_ERR_ARG, op ": piece->data is not a " #T); \
  const T *d = (const T *)piece->data;

extern "C" int b200_colorin_process_dev(const b200_piece_t *piece, const void *in, void *out, void *stream)
{
  COLOR_CHECK("colorin", b200_colorin_data_t)
  if(d->blue_mapping) return fail(B200_ERR_UNSUPPORTED, "colorin: the legacy blue-mapping hook (v1/v2 history) is not built");
  return color_process_dev(piece, d->conversion, d->type, in, out, stream);
}
extern "C" int b200_colorin_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  COLOR_CHECK("colorin", b200_colorin_data_t)
  if(d->blue_mapping) return fail(B200_ERR_UNSUPPORTED, "colorin: the legacy blue-mapping hook (v1/v2 history) is not built");
  const size_t bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 16;
  return through_device(piece, in, bytes, out, bytes, false, b200_colorin_process_dev);
}
extern "C" int b200_colorout_process_dev(const b200_piece_t *piece, const void *in, void *out, void *stream)
{
  COLOR_CHECK("colorout", b200_colorout_data_t)
  return color_process_dev(piece, d->conversion, d->type, in, out, stream);
}
// colorout as the last module of a banded chain: the band goes straight into every GPU's frame
extern "C" int b200_colorout_process_scatter_dev(const b200_piece_t *piece, const void *in, int n_out, void *const *outs, void *stream)
{
  void *out = (n_out > 0 && outs) ? outs[0] : nullptr;
  COLOR_CHECK("colorout", b200_colorout_data_t)
  if(d->type == B200_COLORSPACE_LAB || !d->conversion) return fail(B200_ERR_UNSUPPORTED, "colorout scatter: pass-through conversions are not scattered");
  return b200_apply_conversion_scatter_dev(d->conversion, in, n_out, outs, piece->roi_out.width, piece->roi_out.height,
                                           piece->mask_display & B200_DISPLAY_MASK, stream);
}
extern "C" int b200_colorout_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  COLOR_CHECK("colorout", b200_colorout_data_t)
  (void)d;
  const size_t bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 16;
  return through_device(piece, in, bytes, out, bytes, false, b200_colorout_process_dev);
}
extern "C" void b200_colorin_tiling(const b200_piece_t *piece, b200_tiling_t *t) { default_tiling(piece, t, 0, false); }
extern "C" void b200_colorout_tiling(const b200_piece_t *piece, b200_tiling_t *t) { default_tiling(piece, t, 0, false); }

// dt_ioppr_init_unbounded_coeffs(), colorprofiles/iop_profile.c:303-329, with dt_iop_estimate_exp
// (develop/imageop_math.h:135-165) and extrapolate_lut (iop_profile.h:536-545).  Host-side set-up
// called from commit_params; plain C float arithmetic with the C library's logf.
static float host_lut_at(const float *lut, float v)
{
  const float scaled = v * (float)(LUTN - 1);
  const float ft = scaled > 0.0f ? (scaled < (float)(LUTN - 1) ? scaled : (float)(LUTN - 1)) : 0.0f;
  const int t = (ft < (float)(LUTN - 2)) ? (int)ft : LUTN - 2;
  const float f = ft - (float)t;
  return lut[t] * (1.0f - f) + lut[t + 1] * f;
}
extern "C" int b200_fit_unbounded_coeffs(const float *const lut[3], float coeffs[3][3])
{
  int nonlinear = 0;
  for(int k = 0; k < 3; k++)
  {
    if(lut[k] && lut[k][0] >= 0.0f)
    {
      const float x[4] = { 0.7f, 0.8f, 0.9f, 1.0f };
      float y[4];
      for(int j = 0; j < 4; j++) y[j] = host_lut_at(lut[k], x[j]);
      const float x0 = x[3], y0 = y[3];
      float g = 0.0f;
      int cnt = 0;
      for(int j = 0; j < 3; j++)
      {
        const float yy = y[j] / y0, xx = x[j] / x0;
        if(yy > 0.0f && xx > 0.0f)
        {
          g += logf(y[j] / y0) / logf(x[j] / x0);
          cnt++;
        }
      }
      g = cnt ? g * (1.0f / cnt) : 1.0f;
      coeffs[k][0] = 1.0f / x0;
      coeffs[k][1] = y0;
      coeffs[k][2] = g;
      nonlinear++;
    }
    else
      coeffs[k][0] = -1.0f;
  }
  return nonlinear;
}
