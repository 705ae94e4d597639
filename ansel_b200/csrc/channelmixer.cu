// Colour calibration (channelmixerrgb): chromatic adaptation, channel mix, gamut compression, colourfulness / brightness.
//
// Reference: iop/channelmixerrgb.c loop_switch :765-959 (called from process() :2018-2066), gamut_mapping :641-706,
// luma_chroma :707-763; pixel/chromatic_adaptation.h (matrices :49-108, bradford_adapt_D50 :178-187, CAT16_adapt_D50
// :199-207, XYZ_adapt_D50 :217-223, _downscale/_upscale_vector_simd :277-290); math/math.h scalar_product :185-195,
// euclidean_norm :206-209.
//
// Pointwise, 32 bytes per pixel at the module boundary and ~150 flops with up to two powf (glibc's, restated in
// flt32_math.cuh, double-precision core): an HBM stream when the gamut compression exponent is 0, FP64-pipe bound
// otherwise.  One thread per pixel; the adaptation kind, version and clip flag are uniform branches.  Every operation in
// the reference's order, no contraction; divisions by literal constants through PTX (see labglue.cu: divc).
#ifndef B200_KERNELS_ON_CPU // tests/emul compiles the kernel of this file with g++ to check it against the oracle without a GPU
#include "runtime.h"
#endif
#include "flt32_math.cuh"
#include <math.h>
#include <string.h>

namespace
{
constexpr int CNT = 256;
#define CM_NORM_MIN 1.52587890625e-05f
#define CM_INVERSE_SQRT_3 0.5773502691896258f

struct cm_args_t
{
  float mix[9], r2x[9], x2r[9]; // rows of data->MIX, work_profile->matrix_in, ->matrix_out
  float saturation[3], lightness[3], grey[3], illuminant[3];
  float p, gamut;
  int apply_grey, clip, kind, version;
};
struct v3
{
  float x, y, z;
};

__device__ __forceinline__ float cm_div3(float a)
{ // a / 3.0f as an IEEE division (nvcc would multiply by the rounded reciprocal)
#ifdef B200_KERNELS_ON_CPU
  return a / 3.0f;
#else
  float q;
  asm("div.rn.ftz.f32 %0, %1, %2;" : "=f"(q) : "f"(a), "f"(3.0f));
  return q;
#endif
}
// dt_mat3x4_mul_vec4 (system/simd.h:188-197) with the rows of the untransposed matrix
__device__ __forceinline__ v3 mul(const float *m, v3 a)
{
  v3 o;
  o.x = m[2] * a.z + (m[1] * a.y + m[0] * a.x);
  o.y = m[5] * a.z + (m[4] * a.y + m[3] * a.x);
  o.z = m[8] * a.z + (m[7] * a.y + m[6] * a.x);
  return o;
}
__device__ __forceinline__ float max_zero(float v) { return ((__float_as_uint(v) & 0x7f800000u) != 0x7f800000u && v > 0.0f) ? v : 0.0f; }
__device__ __forceinline__ v3 max_zero3(v3 a) { return v3{ max_zero(a.x), max_zero(a.y), max_zero(a.z) }; }
__device__ __forceinline__ float scale_of(float Y) { return ((Y > CM_NORM_MIN) && !(Y != Y)) ? (Y + CM_NORM_MIN) : CM_NORM_MIN; }
__device__ __forceinline__ float sqf(float x) { return x * x; }
// scalar_product: the reference's `omp simd reduction(+)` over three products is evaluated as 0 + ((p0 + p2) + p1)
__device__ __forceinline__ float dot3(v3 a, const float *b) { return 0.f + ((a.x * b[0] + a.z * b[2]) + a.y * b[1]); }
__device__ __forceinline__ float norm3(v3 a) { return fmaxf(sqrtf(sqf(a.x) + sqf(a.y) + sqf(a.z)), CM_NORM_MIN); }

__device__ v3 gamut_mapping(const f32m::tables_t &tb, v3 in, float compression, int clip)
{
  const float sum = in.x + in.y + in.z;
  const float Y = in.y;
  if(!(sum > 0.f && Y > 0.f)) return v3{ 0.f, 0.f, 0.f };
  float x = in.x / sum, y = in.y / sum;
  const float uv_denominator = -2.f * x + 12.f * y + 3.f;
  float u = 4.f * x / uv_denominator, v = 9.f * y / uv_denominator;
  const float D50u = 0.20915914598542354f, D50v = 0.488075320769787f;
  const float du = D50u - u, dv = D50v - v;
  const float Delta = Y * (sqf(du) + sqf(dv));
  const float correction = (compression == 0.0f) ? 0.f : f32m::powf_(tb, Delta, compression);
  const float tmp_u = correction * du + u, tmp_v = correction * dv + v;
  u = (u > D50u) ? fmaxf(tmp_u, D50u) : fminf(tmp_u, D50u);
  v = (v > D50v) ? fmaxf(tmp_v, D50v) : fminf(tmp_v, D50v);
  const float xy_denominator = 6.f * u - 16.f * v + 12.f;
  x = 9.f * u / xy_denominator;
  y = 4.f * v / xy_denominator;
  if(clip)
  {
    x = fmaxf(x, 0.0f);
    y = fmaxf(y, 0.0f);
  }
  y = fmaxf(y, CM_NORM_MIN);
  const float scale = x + y;
  if(scale >= 1.f)
  {
    x /= scale;
    y /= scale;
  }
  return v3{ Y * x / y, Y, Y * (1.f - x - y) / y };
}

__device__ v3 luma_chroma(v3 in, const cm_args_t &a)
{
  float norm = norm3(in);
  const float avg = fmaxf(cm_div3(in.x + in.y + in.z), CM_NORM_MIN);
  if(!(norm > 0.f && avg > 0.f)) return in;
  const float mix = dot3(in, a.lightness);
  if(a.version == 2) norm *= CM_INVERSE_SQRT_3;
  v3 o = { in.x / norm, in.y / norm, in.z / norm };
  float coeff_ratio = 0.f;
  if(a.version == 0)
  {
    coeff_ratio += sqf(1.0f - o.x) * a.saturation[0];
    coeff_ratio += sqf(1.0f - o.y) * a.saturation[1];
    coeff_ratio += sqf(1.0f - o.z) * a.saturation[2];
  }
  else
    coeff_ratio = cm_div3(dot3(o, a.saturation));
  o.x = fmaxf((1.0f - o.x) * coeff_ratio + o.x, (o.x < 0.0f) ? o.x : 0.0f);
  o.y = fmaxf((1.0f - o.y) * coeff_ratio + o.y, (o.y < 0.0f) ? o.y : 0.0f);
  o.z = fmaxf((1.0f - o.z) * coeff_ratio + o.z, (o.z < 0.0f) ? o.z : 0.0f);
  if(a.version == 2) norm /= norm3(o) * CM_INVERSE_SQRT_3;
  norm *= fmaxf(1.f + mix / avg, 0.f);
  return v3{ o.x * norm, o.y * norm, o.z * norm };
}

__constant__ float c_lms[4][9] = {
  { 0.8951f, 0.2664f, -0.1614f, -0.7502f, 1.7135f, 0.0367f, 0.0389f, -0.0685f, 1.0296f },           // XYZ -> Bradford LMS
  { 0.9870f, -0.1471f, 0.1600f, 0.4323f, 0.5184f, 0.0493f, -0.0085f, 0.0400f, 0.9685f },            // and back
  { 0.401288f, 0.650173f, -0.051461f, -0.250268f, 1.204414f, 0.045854f, -0.002079f, 0.048952f, 0.953127f }, // XYZ -> CAT16 LMS
  { 1.862068f, -1.011255f, 0.149187f, 0.38752f, 0.621447f, -0.008974f, -0.015841f, -0.034123f, 1.049964f }  // and back
};

__global__ void __launch_bounds__(CNT) channelmixer_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, size_t npixels, const cm_args_t a)
{
  const size_t k = (size_t)blockIdx.x * CNT + threadIdx.x;
  if(k >= npixels) return;
  const f32m::tables_t tb = f32m::global_tables();
  const float4 px = in[k];
  const int kind = a.kind, clip = a.clip;
  const bool bradford = kind == B200_ADAPTATION_LINEAR_BRADFORD || kind == B200_ADAPTATION_FULL_BRADFORD;
  const bool lms = bradford || kind == B200_ADAPTATION_CAT16;
  const float *to_lms = c_lms[bradford ? 0 : 2], *to_xyz = c_lms[bradford ? 1 : 3];
  v3 two = { px.x, px.y, px.z }, one;
  if(clip) two = max_zero3(two);
  if(kind == B200_ADAPTATION_RGB)
  {
    one = mul(a.mix, two);
    one = mul(a.r2x, one);
  }
  else
  {
    one = mul(a.r2x, two);
    const float Y = one.y, s = scale_of(Y);
    if(kind == B200_ADAPTATION_XYZ)
    { // XYZ_adapt_D50
      two = v3{ one.x / s, one.y / s, one.z / s };
      two = v3{ two.x * 0.9642119944211994f / a.illuminant[0], two.y * 1.0f / a.illuminant[1], two.z * 0.8251882845188288f / a.illuminant[2] };
      two = v3{ two.x * s, two.y * s, two.z * s };
      one = mul(a.mix, two);
    }
    else
    {
      two = mul(to_lms, one);
      two = v3{ two.x / s, two.y / s, two.z / s };
      if(bradford)
      { // bradford_adapt_D50
        two = v3{ two.x / a.illuminant[0], two.y / a.illuminant[1], two.z / a.illuminant[2] };
        if(kind == B200_ADAPTATION_FULL_BRADFORD) two.z = (two.z > 0.f) ? f32m::powf_(tb, two.z, a.p) : two.z;
        two = v3{ 0.996078f * two.x, 1.020646f * two.y, 0.818155f * two.z };
      }
      else // CAT16_adapt_D50(.., 1.0f, TRUE)
        two = v3{ two.x * 0.994535f / a.illuminant[0], two.y * 1.000997f / a.illuminant[1], two.z * 0.833036f / a.illuminant[2] };
      one = v3{ two.x * s, two.y * s, two.z * s };
      two = mul(a.mix, one);
      one = mul(to_xyz, two);
    }
  }
  two = gamut_mapping(tb, one, a.gamut, clip);
  one = lms ? mul(to_lms, two) : (kind == B200_ADAPTATION_XYZ ? two : mul(a.x2r, two));
  if(clip) one = max_zero3(one);
  two = luma_chroma(one, a);
  if(clip) two = max_zero3(two);
  float4 o;
  if(a.apply_grey)
  {
    const float grey_mix = fmaxf(two.x * a.grey[0] + two.y * a.grey[1] + two.z * a.grey[2], 0.0f);
    o = make_float4(grey_mix, grey_mix, grey_mix, px.w);
  }
  else
  {
    one = lms ? mul(to_xyz, two) : (kind == B200_ADAPTATION_XYZ ? two : mul(a.r2x, two));
    if(clip) one = max_zero3(one);
    two = mul(a.x2r, one);
    if(clip) two = max_zero3(two);
    o = make_float4(two.x, two.y, two.z, px.w);
  }
  out[k] = o;
}

// flatten the piece into kernel arguments; false = an adaptation the reference's switch does not handle (nothing is written)
bool make_cm_args(const b200_channelmixerrgb_piece_t *pc, cm_args_t *a)
{
  const b200_channelmixerrgb_data_t *d = &pc->data;
  if(d->adaptation < B200_ADAPTATION_LINEAR_BRADFORD || d->adaptation > B200_ADAPTATION_RGB) return false;
  for(int r = 0; r < 3; r++)
  {
    for(int c = 0; c < 3; c++)
    {
      a->mix[3 * r + c] = d->MIX[r][c];
      a->r2x[3 * r + c] = pc->work_profile.matrix_in[r][c];
      a->x2r[3 * r + c] = pc->work_profile.matrix_out[r][c];
    }
    a->saturation[r] = d->saturation[r];
    a->lightness[r] = d->lightness[r];
    a->grey[r] = d->grey[r];
    a->illuminant[r] = d->illuminant[r];
  }
  a->p = d->p;
  a->gamut = d->gamut;
  a->apply_grey = d->apply_grey;
  a->clip = d->clip;
  a->kind = d->adaptation;
  a->version = d->version;
  return true;
}
} // namespace

#ifndef B200_KERNELS_ON_CPU
using namespace b200;

static int cm_check(const b200_piece_t *piece, const void *in, const void *out)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "channelmixerrgb: NULL argument");
  if(!piece->data || piece->data_size < sizeof(b200_channelmixerrgb_piece_t))
    return fail(B200_ERR_ARG, "channelmixerrgb: piece->data is not a b200_channelmixerrgb_piece_t (data block + work profile matrices)");
  if(in == out) return fail(B200_ERR_ARG, "channelmixerrgb: in-place processing is not supported");
  if(piece->roi_out.width < 1 || piece->roi_out.height < 1) return fail(B200_ERR_ARG, "channelmixerrgb: empty roi_out");
  const b200_channelmixerrgb_piece_t *pc = (const b200_channelmixerrgb_piece_t *)piece->data;
  if(pc->data.version < 0 || pc->data.version > 2) return fail(B200_ERR_ARG, "channelmixerrgb: version %d", pc->data.version);
  return B200_OK;
}
extern "C" int b200_channelmixerrgb_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = cm_check(piece, d_in, d_out);
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  cm_args_t a;
  if(!make_cm_args((const b200_channelmixerrgb_piece_t *)piece->data, &a)) return B200_OK; // process() :2060-2065: no case, no write
  const size_t npx = (size_t)piece->roi_out.width * piece->roi_out.height;
  channelmixer_kernel<<<(unsigned)((npx + CNT - 1) / CNT), CNT, 0, (cudaStream_t)stream>>>((const float4 *)d_in, (float4 *)d_out, npx, a);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
extern "C" int b200_channelmixerrgb_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = cm_check(piece, in, out);
  if(rc) return rc;
  const size_t bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 16;
  return through_device(piece, in, bytes, out, bytes, true, b200_channelmixerrgb_process_dev); // an unhandled adaptation leaves the output as found
}
extern "C" void b200_channelmixerrgb_tiling(const b200_piece_t *piece, b200_tiling_t *t) { default_tiling(piece, t, 0, false); } // the module declares no tiling callback
#endif
