// RGB <-> Lab glue between modules whose default_colorspace() differs, and the denoise (non-local means) iop.
//
// Reference: colorprofiles/iop_profile.c _transform_rgb_to_lab_matrix :376-420, _transform_lab_to_rgb_matrix
// :422-464; common/colorspaces_inline_conversions.h :51-106 (cbrt_5f bit trick + one Halley step, D50);
// iop/nlmeans.c process_cpu :416-456, tiling_callback :400-414.
// Pointwise, 32 B/px at the boundary: HBM-bound streaming kernels (float4 in, float4 out).
#include "runtime.h"
#include "trc.cuh"
#include <math.h>

namespace b200
{
int nlmeans_denoise_dev(const float *d_in, float *d_out, int width, int height, float scattering, float scale, float luma,
                        float chroma, float center_weight, float sharpness, int radius, int search_radius, int decimate,
                        const float norm[4], cudaStream_t stream);
}

namespace
{
struct m3_t
{
  float m[9];
};
// IEEE division by a compile-time constant.  With -ftz=true nvcc rewrites `x / c` into `x * (1/c)` even under
// -prec-div=true (seen in SASS as FMUL.FTZ by 1.0371291 for `/ 0.9642f`; 1-ulp differences in 18 % of the
// pixels); the PTX instruction is opaque to that rewrite.  Divisions by powers of two are exact either way.
__device__ __forceinline__ float divc(float a, float b)
{
  float q;
  asm("div.rn.ftz.f32 %0, %1, %2;" : "=f"(q) : "f"(a), "f"(b));
  return q;
}
__device__ __forceinline__ float cbrt_5f(float f) { return __uint_as_float(__float_as_uint(f) / 3u + 709921077u); }
__device__ __forceinline__ float cbrta_halleyf(float a, float R)
{
  const float a3 = a * a * a;
  return a * (a3 + R + R) / (a3 + a3 + R);
}
__device__ __forceinline__ float lab_f(float x)
{
  const float epsilon = 216.0f / 24389.0f, kappa = 24389.0f / 27.0f;
  return (x > epsilon) ? cbrta_halleyf(cbrt_5f(x), x) : divc(kappa * x + 16.0f, 116.0f);
}
__device__ __forceinline__ float lab_f_inv(float x)
{
  const float epsilon = 0.20689655172413796f, kappa = 24389.0f / 27.0f;
  return (x > epsilon) ? x * x * x : divc(116.0f * x - 16.0f, kappa);
}
__device__ __forceinline__ float row(const float *m, float x, float y, float z)
{ // dt_mat3x4_mul_vec4, system/simd.h:188-197
  float acc = m[0] * x;
  acc = m[1] * y + acc;
  acc = m[2] * z + acc;
  return acc;
}
__global__ void __launch_bounds__(256) rgb_to_lab_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, size_t n, const m3_t M)
{
  const size_t k = (size_t)blockIdx.x * 256 + threadIdx.x;
  if(k >= n) return;
  const float4 p = in[k];
  const float fx = lab_f(divc(row(M.m + 0, p.x, p.y, p.z), 0.9642f));
  const float fy = lab_f(row(M.m + 3, p.x, p.y, p.z));
  const float fz = lab_f(divc(row(M.m + 6, p.x, p.y, p.z), 0.8249f));
  out[k] = make_float4(116.0f * fy - 16.0f, 500.0f * (fx - fy), 200.0f * (fy - fz), p.w);
}
__global__ void __launch_bounds__(256) lab_to_rgb_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, size_t n, const m3_t M)
{
  const size_t k = (size_t)blockIdx.x * 256 + threadIdx.x;
  if(k >= n) return;
  const float4 p = in[k];
  const float fy = divc(p.x + 16.0f, 116.0f);
  const float fx = divc(p.y, 500.0f) + fy;
  const float fz = fy - divc(p.z, 200.0f);
  const float X = 0.9642f * lab_f_inv(fx), Y = 1.0f * lab_f_inv(fy), Z = 0.8249f * lab_f_inv(fz);
  out[k] = make_float4(row(M.m + 0, X, Y, Z), row(M.m + 3, X, Y, Z), row(M.m + 6, X, Y, Z), p.w);
}
// the same two conversions for a profile with tone curves (_apply_tonecurves :332-373): lut_in before the matrix,
// lut_out after it, each only on the channels that have a curve (nullptr = linear channel)
struct curves_t
{
  const float *lut[3];
  float co[9];
};
__global__ void __launch_bounds__(256) rgb_to_lab_trc_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, size_t n, const m3_t M, const curves_t cv)
{
  const size_t k = (size_t)blockIdx.x * 256 + threadIdx.x;
  if(k >= n) return;
  const f32m::tables_t tb = f32m::global_tables();
  float4 p = in[k];
  if(cv.lut[0]) p.x = eval_trc<false, true>(tb, p.x, cv.lut[0], cv.co + 0);
  if(cv.lut[1]) p.y = eval_trc<false, true>(tb, p.y, cv.lut[1], cv.co + 3);
  if(cv.lut[2]) p.z = eval_trc<false, true>(tb, p.z, cv.lut[2], cv.co + 6);
  const float fx = lab_f(divc(row(M.m + 0, p.x, p.y, p.z), 0.9642f));
  const float fy = lab_f(row(M.m + 3, p.x, p.y, p.z));
  const float fz = lab_f(divc(row(M.m + 6, p.x, p.y, p.z), 0.8249f));
  out[k] = make_float4(116.0f * fy - 16.0f, 500.0f * (fx - fy), 200.0f * (fy - fz), p.w);
}
__global__ void __launch_bounds__(256) lab_to_rgb_trc_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, size_t n, const m3_t M, const curves_t cv)
{
  const size_t k = (size_t)blockIdx.x * 256 + threadIdx.x;
  if(k >= n) return;
  const f32m::tables_t tb = f32m::global_tables();
  const float4 p = in[k];
  const float fy = divc(p.x + 16.0f, 116.0f);
  const float fx = divc(p.y, 500.0f) + fy;
  const float fz = fy - divc(p.z, 200.0f);
  const float X = 0.9642f * lab_f_inv(fx), Y = 1.0f * lab_f_inv(fy), Z = 0.8249f * lab_f_inv(fz);
  float4 o = make_float4(row(M.m + 0, X, Y, Z), row(M.m + 3, X, Y, Z), row(M.m + 6, X, Y, Z), p.w);
  if(cv.lut[0]) o.x = eval_trc<false, false>(tb, o.x, cv.lut[0], cv.co + 0);
  if(cv.lut[1]) o.y = eval_trc<false, false>(tb, o.y, cv.lut[1], cv.co + 3);
  if(cv.lut[2]) o.z = eval_trc<false, false>(tb, o.z, cv.lut[2], cv.co + 6);
  out[k] = o;
}
__global__ void copy_alpha_kernel2(const float4 *__restrict__ in, float4 *__restrict__ out, size_t n)
{
  const size_t k = (size_t)blockIdx.x * 256 + threadIdx.x;
  if(k < n) out[k].w = in[k].w;
}
} // namespace

using namespace b200;

static int transform(const void *d_in, void *d_out, int width, int height, int cst_from, int cst_to, const b200_profile_matrices_t *wp,
                     const b200_profile_curves_t *curves, int nonlinearlut, void *stream);
extern "C" int b200_colorspace_transform_dev(const void *d_in, void *d_out, int width, int height, int cst_from, int cst_to,
                                             const b200_profile_matrices_t *wp, int nonlinearlut, void *stream)
{
  return transform(d_in, d_out, width, height, cst_from, cst_to, wp, nullptr, nonlinearlut, stream);
}
extern "C" int b200_colorspace_transform_trc_dev(const void *d_in, void *d_out, int width, int height, int cst_from, int cst_to,
                                                 const b200_profile_matrices_t *wp, const b200_profile_curves_t *curves, void *stream)
{
  if(!curves) return fail(B200_ERR_ARG, "colorspace_transform_trc: NULL curves");
  for(int k = 0; k < 3; k++)
    if(!curves->lut_in[k] || !curves->lut_out[k]) return fail(B200_ERR_ARG, "colorspace_transform_trc: NULL curve");
  // dt_ioppr_init_unbounded_coeffs, iop_profile.c:303-329: the flag counts the INPUT curves only and gates both directions
  int nonlinearlut = 0;
  for(int k = 0; k < 3; k++) nonlinearlut += curves->lut_in[k][0] >= 0.0f;
  return transform(d_in, d_out, width, height, cst_from, cst_to, wp, nonlinearlut ? curves : nullptr, 0, stream);
}
static int transform(const void *d_in, void *d_out, int width, int height, int cst_from, int cst_to, const b200_profile_matrices_t *wp,
                     const b200_profile_curves_t *curves, int nonlinearlut, void *stream)
{
  if(!d_in || !d_out || !wp) return fail(B200_ERR_ARG, "colorspace_transform: NULL argument");
  if(width <= 0 || height <= 0) return B200_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t n = (size_t)width * height;
  if(cst_from == cst_to)
  { // dt_colorspaces_apply_profile :1305-1309: nothing to do (the caller keeps using the input buffer)
    if(d_in != d_out) B200_CUDA_TRY(cudaMemcpyAsync(d_out, d_in, n * 16, cudaMemcpyDeviceToDevice, s));
    return B200_OK;
  }
  if(nonlinearlut) return fail(B200_ERR_UNSUPPORTED, "colorspace_transform: a work profile with tone curves goes through b200_colorspace_transform_trc_dev");
  if(isnan(wp->matrix_in[0][0]) || isnan(wp->matrix_out[0][0]))
    return fail(B200_ERR_UNSUPPORTED, "colorspace_transform: not a matrix profile (the reference falls back to lcms2)");
  m3_t M;
  const unsigned grid = (unsigned)((n + 255) / 256);
  if(cst_from == B200_CS_RGB && cst_to == B200_CS_LAB)
  {
    for(int i = 0; i < 3; i++)
      for(int j = 0; j < 3; j++) M.m[3 * i + j] = wp->matrix_in[i][j];
    if(curves)
    {
      curves_t cv;
      const float *d = nullptr;
      int rc = device_curves(curves->lut_in, curves->identity, 2, s, &d);
      if(rc) return rc;
      for(int k = 0; k < 3; k++)
      {
        cv.lut[k] = curves->lut_in[k][0] >= 0.0f ? d + (size_t)k * B200_LUT_SAMPLES : nullptr;
        for(int j = 0; j < 3; j++) cv.co[3 * k + j] = curves->unbounded_coeffs_in[k][j];
      }
      rgb_to_lab_trc_kernel<<<grid, 256, 0, s>>>((const float4 *)d_in, (float4 *)d_out, n, M, cv);
    }
    else
      rgb_to_lab_kernel<<<grid, 256, 0, s>>>((const float4 *)d_in, (float4 *)d_out, n, M);
  }
  else if(cst_from == B200_CS_LAB && cst_to == B200_CS_RGB)
  {
    for(int i = 0; i < 3; i++)
      for(int j = 0; j < 3; j++) M.m[3 * i + j] = wp->matrix_out[i][j];
    if(curves)
    {
      curves_t cv;
      const float *d = nullptr;
      int rc = device_curves(curves->lut_out, curves->identity, 3, s, &d);
      if(rc) return rc;
      for(int k = 0; k < 3; k++)
      {
        cv.lut[k] = curves->lut_out[k][0] >= 0.0f ? d + (size_t)k * B200_LUT_SAMPLES : nullptr;
        for(int j = 0; j < 3; j++) cv.co[3 * k + j] = curves->unbounded_coeffs_out[k][j];
      }
      lab_to_rgb_trc_kernel<<<grid, 256, 0, s>>>((const float4 *)d_in, (float4 *)d_out, n, M, cv);
    }
    else
      lab_to_rgb_kernel<<<grid, 256, 0, s>>>((const float4 *)d_in, (float4 *)d_out, n, M);
  }
  else
    return fail(B200_ERR_ARG, "colorspace_transform: invalid conversion from %d to %d", cst_from, cst_to); // :594
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}

// ---- denoise (non-local means) iop --------------------------------------------------------------
static int check_nl(const b200_piece_t *piece, const void *in, void *out)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "nlmeans: NULL argument");
  if(!piece->data || piece->data_size < sizeof(b200_nlmeans_data_t)) return fail(B200_ERR_ARG, "nlmeans: piece->data is not a b200_nlmeans_data_t");
  if(in == out) return fail(B200_ERR_ARG, "nlmeans: in-place processing is not supported");
  return B200_OK;
}
extern "C" int b200_nlmeans_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = check_nl(piece, d_in, d_out);
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  const b200_nlmeans_data_t *d = (const b200_nlmeans_data_t *)piece->data;
  cudaStream_t s = (cudaStream_t)stream;
  const int width = piece->roi_in.width, height = piece->roi_in.height;
  const float scale = (float)fmin(piece->roi_in.scale, (double)2.0f); // nlmeans.c:430
  const int P = (int)ceilf(d->radius * scale);
  const int K = (int)ceilf(7 * scale);
  const float sharpness = 3000.0f / (1.0f + d->strength);
  const float max_L = 120.0f, max_C = 512.0f;
  const float nL = 1.0f / max_L, nC = 1.0f / max_C;
  const float norm2[4] = { nL * nL, nC * nC, nC * nC, 1.0f };
  const int decimate = (piece->pipe_type == B200_PIPE_THUMBNAIL || piece->pipe_type == B200_PIPE_PREVIEW) ? 1 : 0;
  if((rc = nlmeans_denoise_dev((const float *)d_in, (float *)d_out, width, height, 0.0f, scale, d->luma, d->chroma, -1.0f, sharpness, P, K,
                               decimate, norm2, s)))
    return rc;
  if(piece->mask_display & B200_DISPLAY_MASK)
  {
    const size_t n = (size_t)width * height;
    copy_alpha_kernel2<<<(unsigned)((n + 255) / 256), 256, 0, s>>>((const float4 *)d_in, (float4 *)d_out, n);
    B200_CUDA_TRY(cudaGetLastError());
  }
  return B200_OK;
}
extern "C" int b200_nlmeans_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_nl(piece, in, out);
  if(rc) return rc;
  const size_t bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 16;
  return through_device(piece, in, bytes, out, bytes, false, b200_nlmeans_process_dev);
}
extern "C" void b200_nlmeans_tiling(const b200_piece_t *piece, b200_tiling_t *tiling)
{
  if(!piece || !tiling || !piece->data) return;
  const b200_nlmeans_data_t *d = (const b200_nlmeans_data_t *)piece->data;
  const int P = (int)ceilf((float)(d->radius * fmin(piece->roi_in.scale, (double)2.0f)));
  const int K = (int)ceilf((float)(7 * fmin(piece->roi_in.scale, (double)2.0f)));
  tiling->factor = (float)(2.0f + 1.0f + 0.25 * 4); // NUM_BUCKETS 4
  tiling->maxbuf = 1.0f;
  tiling->overhead = 0;
  tiling->overlap = P + K;
  tiling->xalign = 1;
  tiling->yalign = 1;
}
