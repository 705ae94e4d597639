// Colour balance rgb (colorbalancergb): chroma and hue rotation in Yrg, four-way grading in Filmlight RGB behind the opacity masks,
// luminance power and contrast, then saturation / brilliance with gamut mapping in JzAzBz or darktable UCS.
//
// Reference: iop/colorbalancergb.c process() :585-927 with opacity_masks :509-536, soft_clip :538-544, lookup_gamut :547-581;
// common/colorspaces_inline_conversions.h (dt_XYZ_to_xyY_simd :119-123, dt_xyY_to_XYZ_simd :135-139, dt_XYZ_2_JzAzBz_simd :726-768,
// dt_JzAzBz_2_XYZ_simd :854-891, LMS_to_XYZ_simd :940-952, gradingRGB_to_LMS_simd :977-988, LMS_to_gradingRGB_simd :996-1007,
// LMS_to_Yrg_simd :1034-1042, Yrg_to_LMS_simd :1066-1073, the darktable UCS functions :1261-1466); system/simd.h dt_mat3x4_mul_vec4
// :189-197, dt_simd_max_zero :108-114; math/math.h scalar_product :185-195.
//
// Pointwise, 32 bytes per pixel at the module boundary and 19 powf, 5 expf (JzAzBz: 2 expf + 2 atan2f + sinf / cosf; dt UCS: one
// atan2f, one sinf, one cosf) per pixel: glibc's, restated in flt32_math.cuh.  One thread per pixel, float4 loads and stores.  The
// saturation formula is a template parameter, so each instance carries one branch.  The gamut LUT is indexed by hue, so it is staged
// in shared memory; from parameter space its reads would serialise across a warp.  Every operation in the reference's order, no
// contraction; MIN / MAX are the reference's ternaries (not fminf / fmaxf, which pick differently on NaN); divisions by constants
// that are not powers of two take their divisor from the arguments (cb_args_t).  The powf calls go through one
// out-of-line copy, so the kernel is not nineteen inlined powf bodies (see filmic.cu on code size).
#ifndef B200_KERNELS_ON_CPU // tests/emul/emul_colorbalancergb.cpp compiles the kernel and its host set-up with g++
#include "runtime.h"
#endif
#include "flt32_math.cuh"
#include <math.h>
#include <string.h>

namespace
{
constexpr int CB_CNT = 128;
constexpr int CB_LUT = B200_COLORBALANCE_LUT_ELEM;

// what the pixel loop reads: the host's part of process() (:613-674) flattened, plus the LUT
struct cb_args_t
{
  float in_m[3][3];  // input_matrix: work RGB -> CIE 2006 LMS (XYZ_D65_to_LMS_2006_D65 . XYZ_D50_to_D65_CAT16 . matrix_in)
  float out_m[3][3]; // output_matrix: XYZ D65 -> work RGB (matrix_out . XYZ_D65_to_D50_CAT16)
  float global[3], shadows[3], highlights[3], midtones[3];
  float chroma[3], saturation[3], brilliance[3];
  float chroma_global, vibrance, contrast, saturation_global, brilliance_global, midtones_Y;
  float shadows_weight, highlights_weight, midtones_weight, mask_grey_fulcrum, white_fulcrum, grey_fulcrum;
  float L_white;
  float rot[2][2]; // hue_rotation_matrix :671-674
  // the divisors that are constants of the reference but not powers of two: lookup_gamut's 2 M_PI_F, JzAzBz's 10000, b and g.  As
  // arguments they are IEEE divisions in plain sight; nvcc would rewrite `x / literal` into a product, and ptxas expands div.rn by a
  // literal around a hoisted reciprocal that no MUFU marks
  float two_pi, d10000, b, g;
  float lut[CB_LUT];
};

constexpr float CB_PI = 3.14159265358979324f; // M_PI_F, DT_M_PI_F (math/math.h:50,54)
constexpr float D65_R = 0.21902143f, D65_G = 0.54371398f;

__device__ __forceinline__ float cb_max(float a, float b) { return (a > b) ? a : b; } // MAX, the ternary
__device__ __forceinline__ float cb_min(float a, float b) { return (a < b) ? a : b; } // MIN
__device__ __forceinline__ float sqf(float x) { return x * x; }
// dt_simd_max_zero: non-finite -> 0, else MAX(v, 0)
__device__ __forceinline__ float max_zero(float v) { return ((__float_as_uint(v) & 0x7f800000u) != 0x7f800000u) ? cb_max(v, 0.0f) : 0.0f; }
// scalar_product over the opacities: the reference's `omp simd reduction(+)` is evaluated as 0 + ((p0 + p2) + p1) (channelmixer.cu)
__device__ __forceinline__ float sp3(const float o[3], const float v[3]) { return 0.f + ((o[0] * v[0] + o[2] * v[2]) + o[1] * v[1]); }
// dt_mat3x4_mul_vec4 with the rows of the untransposed matrix: row0 * in0, then row1 * in1 + that, then row2 * in2 + that
__device__ __forceinline__ void mul3(const float (*m)[3], const float in[3], float out[3])
{
  for(int c = 0; c < 3; c++) out[c] = m[c][2] * in[2] + (m[c][1] * in[1] + m[c][0] * in[0]);
}

__device__ const float C_grading_to_LMS[3][3] = { { 0.95f, 0.38f, 0.00f }, { 0.05f, 0.62f, 0.03f }, { 0.00f, 0.00f, 0.97f } };
__device__ const float C_LMS_to_grading[3][3] = { { 1.0877193f, -0.66666667f, 0.02061856f }, { -0.0877193f, 1.66666667f, -0.05154639f }, { 0.f, 0.f, 1.03092784f } };
__device__ const float C_LMS_to_XYZ[3][3] = { { 1.80794659f, -1.29971660f, 0.34785879f }, { 0.61783960f, 0.39595453f, -0.04104687f },
                                              { -0.12546960f, 0.20478038f, 1.74274183f } };
__device__ const float C_Jz_M[3][3] = { { 0.41478972f, 0.579999f, 0.0146480f }, { -0.2015100f, 1.120649f, 0.0531008f }, { -0.0166008f, 0.264800f, 0.6684799f } };
__device__ const float C_Jz_A[3][3] = { { 0.5f, 0.5f, 0.0f }, { 3.524000f, -4.066708f, 0.542708f }, { 0.199076f, 1.096799f, -1.295875f } };
__device__ const float C_Jz_AI[3][3] = { { 1.0f, 0.1386050432715393f, 0.0580473161561189f },
                                         { 1.0f, -0.1386050432715393f, -0.0580473161561189f },
                                         { 1.0f, -0.0960192420263190f, -0.8118918960560390f } };
__device__ const float C_Jz_MI[3][3] = { { 1.9242264357876067f, -1.0047923125953657f, 0.0376514040306180f },
                                         { 0.3503167620949991f, 0.7264811939316552f, -0.0653844229480850f },
                                         { -0.0909828109828475f, -0.3127282905230739f, 1.5227665613052603f } };

// glibc's powf, out of line: one copy for the nineteen calls per pixel
__device__ __noinline__ float cb_pow(float x, float y) { return f32m::powf_(f32m::global_tables(), x, y); }
__device__ __forceinline__ float cb_exp(float x) { return f32m::expf_(f32m::global_tables(), x); }

// LMS_to_Yrg_simd
__device__ __forceinline__ void lms_to_yrg(const float LMS[3], float Yrg[3])
{
  const float Y = 0.68990272f * LMS[0] + 0.34832189f * LMS[1];
  const float a = LMS[0] + LMS[1] + LMS[2];
  const float inv_a = (a == 0.f) ? 0.f : 1.f / a;
  const float lms[3] = { LMS[0] * inv_a, LMS[1] * inv_a, LMS[2] * inv_a };
  float rgb[3];
  mul3(C_LMS_to_grading, lms, rgb);
  Yrg[0] = Y;
  Yrg[1] = rgb[0];
  Yrg[2] = rgb[1];
}
// Yrg_to_LMS_simd
__device__ __forceinline__ void yrg_to_lms(const float Yrg[3], float LMS[3])
{
  const float rgb[3] = { Yrg[1], Yrg[2], 1.f - Yrg[1] - Yrg[2] };
  float lms[3];
  mul3(C_grading_to_LMS, rgb, lms);
  const float denom = 0.68990272f * lms[0] + 0.34832189f * lms[1];
  const float a = (denom == 0.f) ? 0.f : Yrg[0] / denom;
  for(int c = 0; c < 3; c++) LMS[c] = lms[c] * a;
}

// opacity_masks :509-536 -> opacities (shadows, mid-tones, highlights) and their complements
__device__ __forceinline__ void opacity_masks(const float x, const cb_args_t &a, float op[3], float comp[3])
{
  const float x_offset = (x - a.mask_grey_fulcrum);
  const float x_offset_norm = x_offset / a.mask_grey_fulcrum;
  const float alpha = 1.f / (1.f + cb_exp(x_offset_norm * a.shadows_weight));
  const float beta = 1.f / (1.f + cb_exp(-x_offset_norm * a.highlights_weight));
  const float alpha_comp = 1.f - alpha;
  const float beta_comp = 1.f - beta;
  const float gamma = cb_exp(-sqf(x_offset) * a.midtones_weight / 4.f) * sqf(alpha_comp) * sqf(beta_comp) * 8.f;
  op[0] = alpha;
  op[1] = gamma;
  op[2] = beta;
  comp[0] = alpha_comp;
  comp[1] = 1.f - gamma;
  comp[2] = beta_comp;
}
// soft_clip :538-544
__device__ __forceinline__ float soft_clip(const float x, const float soft_threshold, const float hard_threshold)
{
  const float norm = hard_threshold - soft_threshold;
  return (x > soft_threshold) ? soft_threshold + (1.f - cb_exp(-(x - soft_threshold) / norm)) * norm : x;
}
// lookup_gamut :547-581 on the staged LUT; two_pi = 2.f * M_PI_F
__device__ __forceinline__ float lookup_gamut(const float *lut, const float x, const float two_pi)
{
  const float x_test = (float)(CB_LUT - 1) * (x + CB_PI) / two_pi;
  const float x_prev = floorf(x_test);
  const float x_next = ceilf(x_test);
  int xi = (int)x_prev;
  if(xi < 0) xi = CB_LUT - 1;
  else if(xi > CB_LUT - 1) xi = 0;
  int xii = (int)x_next;
  if(xii < 0) xii = CB_LUT - 1;
  else if(xii > CB_LUT - 1) xii = 0;
  const float y_prev = lut[xi];
  const float y_next = lut[xii];
  float out = y_prev;
  if(x_next != x_prev) out += (x_test - x_prev) * (y_next - y_prev) / (x_next - x_prev);
  return out;
}

// the JzAzBz branch :763-842, XYZ D65 in place
__device__ __forceinline__ void saturation_jzazbz(float XYZ[3], const float op[3], const float *lut, const cb_args_t &a)
{
  const float b = 1.15f, g = 0.66f, c1 = 0.8359375f, c2 = 18.8515625f, c3 = 18.6875f, n = 0.159301758f, p = 134.034375f, d = -0.56f;
  const float d0 = 1.6295499532821566e-11f;
  // dt_XYZ_2_JzAzBz_simd
  const float Xp[3] = { b * XYZ[0] - (b - 1.0f) * XYZ[2], g * XYZ[1] - (g - 1.0f) * XYZ[0], XYZ[2] };
  float LMS[3], Jab[3];
  mul3(C_Jz_M, Xp, LMS);
  for(int i = 0; i < 3; i++)
  {
    LMS[i] = cb_pow(fmaxf(LMS[i] / a.d10000, 0.0f), n);
    LMS[i] = cb_pow((c1 + c2 * LMS[i]) / (1.0f + c3 * LMS[i]), p);
  }
  mul3(C_Jz_A, LMS, Jab);
  Jab[0] = fmaxf(((1.0f + d) * Jab[0]) / (1.0f + d * Jab[0]) - d0, 0.f);

  float JC[2] = { Jab[0], sqrtf(Jab[1] * Jab[1] + Jab[2] * Jab[2]) };
  const float h = f32m::atan2f_(Jab[2], Jab[1]);
  const float inv_chroma = (JC[1] > 0.f) ? 1.f / JC[1] : 0.f;
  const float cos_H = Jab[1] * inv_chroma;
  const float sin_H = Jab[2] * inv_chroma;
  const float T = f32m::atan2f_(JC[1], JC[0]);
  const float sin_T = f32m::sinf_(T);
  const float cos_T = f32m::cosf_(T);
  const float boosts[2] = { 1.f + a.brilliance_global + sp3(op, a.brilliance), a.saturation_global + sp3(op, a.saturation) };
  float SO[2];
  SO[0] = JC[0] * cos_T + JC[1] * sin_T;
  SO[1] = SO[0] * cb_min(cb_max(T * boosts[1], -T), CB_PI / 2.f - T);
  SO[0] = cb_max(SO[0] * boosts[0], 0.f);
  JC[0] = cb_max(SO[0] * cos_T + SO[1] * -sin_T, 0.f);
  JC[1] = cb_max(SO[0] * sin_T + SO[1] * cos_T, 0.f);

  const float out_max_sat_h = lookup_gamut(lut, h, a.two_pi);
  const float sat = (JC[0] > 0.f) ? soft_clip(JC[1] / JC[0], 0.8f * out_max_sat_h, out_max_sat_h) : out_max_sat_h;
  const float max_C_at_sat = JC[0] * sat;
  const float max_J_at_sat = (sat > 0.f) ? JC[1] / sat : JC[0];
  JC[0] = (JC[0] + max_J_at_sat) / 2.f;
  JC[1] = (JC[1] + max_C_at_sat) / 2.f;

  float Iz = JC[0] + d0;
  Iz /= (1.f + d - d * Iz);
  Iz = cb_max(Iz, 0.f);
  const float IzAzBz[3] = { Iz, JC[1] * cos_H, JC[1] * sin_H };
  float LMS_test[3];
  mul3(C_Jz_AI, IzAzBz, LMS_test);
  float max_C = JC[1];
  for(int i = 0; i < 3; i++)
    if(LMS_test[i] < 0.f) max_C = cb_min(-Iz / (C_Jz_AI[i][1] * cos_H + C_Jz_AI[i][2] * sin_H), max_C);

  // dt_JzAzBz_2_XYZ_simd on { JC[0], max_C cos_H, max_C sin_H }
  const float p_inv = 1.0f / 134.034375f, n_inv = 1.0f / 0.159301758f;
  float I[3] = { JC[0] + d0, max_C * cos_H, max_C * sin_H };
  I[0] = fmaxf(I[0] / (1.0f + d - d * I[0]), 0.f);
  mul3(C_Jz_AI, I, LMS);
  for(int i = 0; i < 3; i++)
  {
    LMS[i] = cb_pow(fmaxf(LMS[i], 0.0f), p_inv);
    LMS[i] = 10000.f * cb_pow(fmaxf((c1 - LMS[i]) / (c3 * LMS[i] - c2), 0.0f), n_inv);
  }
  float X[3];
  mul3(C_Jz_MI, LMS, X);
  XYZ[0] = (X[0] + (b - 1.0f) * X[2]) / a.b;
  XYZ[1] = (X[1] + (g - 1.0f) * ((X[0] + (b - 1.0f) * X[2]) / a.b)) / a.g;
  XYZ[2] = X[2];
}

// the darktable UCS branch :843-885, XYZ D65 in place
__device__ __forceinline__ void saturation_dt_ucs(float XYZ[3], const float op[3], const float *lut, const cb_args_t &a)
{
  const float L_white = a.L_white;
  // dt_XYZ_to_xyY_simd
  const float sum = XYZ[0] + XYZ[1] + XYZ[2];
  const float x = XYZ[0] / sum, y = XYZ[1] / sum, Y = XYZ[1];
  // xyY_to_dt_UCS_JCH: xyY_to_dt_UCS_UV, Y_to_dt_UCS_L_star, dt_UCS_LUV_to_JCH
  float UVD[3];
  UVD[0] = -0.783941002840055f * x + 0.277512987809202f * y + 0.153836578598858f;
  UVD[1] = 0.745273540913283f * x + -0.205375866083878f * y + -0.165478376301988f;
  UVD[2] = 0.318707282433486f * x + 2.16743692732158f * y + 0.291320554395942f;
  UVD[0] /= UVD[2];
  UVD[1] /= UVD[2];
  const float UV_star0 = 1.39656225667f * UVD[0] / (fabsf(UVD[0]) + 1.49217352929f);
  const float UV_star1 = 1.4513954287f * UVD[1] / (fabsf(UVD[1]) + 1.52488637914f);
  const float Up = -1.124983854323892f * UV_star0 - 0.980483721769325f * UV_star1;
  const float Vp = 1.86323315098672f * UV_star0 + 1.971853092390862f * UV_star1;
  const float Y_hat = cb_pow(Y, 0.631651345306265f);
  const float L_star = 2.098883786377f * Y_hat / (Y_hat + 1.12426773749357f);
  const float M2 = Up * Up + Vp * Vp;
  const float J = L_star / L_white;
  const float C = 15.932993652962535f * cb_pow(L_star, 0.6523997524738018f) * cb_pow(M2, 0.6007557017508491f) / L_white;
  const float H = f32m::atan2f_(Vp, Up);
  // dt_UCS_JCH_to_HCB_simd
  float HCB[3] = { H, C, J * (cb_pow(C, 1.33654221029386f) + 1.f) };

  const float radius = sqrtf(HCB[1] * HCB[1] + HCB[2] * HCB[2]);
  const float sin_T = (radius > 0.f) ? HCB[1] / radius : 0.f;
  const float cos_T = (radius > 0.f) ? HCB[2] / radius : 0.f;
  const float P = cb_max(HCB[1], 1.17549435082228750797e-38f); // FLT_MIN
  const float W = sin_T * HCB[1] + cos_T * HCB[2];
  float sa = max_zero(1.f + a.saturation_global + sp3(op, a.saturation));
  const float b = max_zero(1.f + a.brilliance_global + sp3(op, a.brilliance));
  const float max_a = sqrtf(P * P + W * W) / P;
  sa = soft_clip(sa, 0.5f * max_a, max_a);
  const float P_prime = (sa - 1.f) * P;
  const float W_prime = sqrtf(sqf(P) * (1.f - sqf(sa)) + sqf(W)) * b;
  HCB[1] = cb_max(cos_T * P_prime + sin_T * W_prime, 0.f);
  HCB[2] = cb_max(-sin_T * P_prime + cos_T * W_prime, 0.f);

  // dt_UCS_HCB_to_JCH_simd
  float JCH[3] = { HCB[2] / (cb_pow(HCB[1], 1.33654221029386f) + 1.f), HCB[1], HCB[0] };
  const float max_colorfulness = lookup_gamut(lut, JCH[2], a.two_pi);
  const float max_chroma = 15.932993652962535f * cb_pow(JCH[0] * L_white, 0.6523997524738018f) * cb_pow(max_colorfulness, 0.6007557017508491f) / L_white;
  // dt_UCS_JCH_to_HSB_simd of the gamut boundary: its saturation
  const float brightness = JCH[0] * (cb_pow(max_chroma, 1.33654221029386f) + 1.f);
  const float S_boundary = (brightness > 0.f) ? max_chroma / brightness : 0.f;
  float HSB[3] = { HCB[0], (HCB[2] > 0.f) ? HCB[1] / HCB[2] : 0.f, HCB[2] };
  HSB[1] = soft_clip(HSB[1], 0.8f * S_boundary, S_boundary);
  // dt_UCS_HSB_to_JCH_simd
  const float chroma = HSB[1] * HSB[2];
  JCH[0] = HSB[2] / (cb_pow(chroma, 1.33654221029386f) + 1.f);
  JCH[1] = chroma;
  JCH[2] = HSB[0];
  // dt_UCS_JCH_to_xyY
  const float L_s = JCH[0] * L_white;
  const float M = cb_pow(JCH[1] * L_white / (15.932993652962535f * cb_pow(L_s, 0.6523997524738018f)), 0.8322850678616855f);
  const float U_star_prime = M * f32m::cosf_(JCH[2]);
  const float V_star_prime = M * f32m::sinf_(JCH[2]);
  const float UV_s0 = -5.037522385190711f * U_star_prime - 2.504856328185843f * V_star_prime;
  const float UV_s1 = 4.760029407436461f * U_star_prime + 2.874012963239247f * V_star_prime;
  const float UV0 = -1.49217352929f * UV_s0 / (fabsf(UV_s0) - 1.39656225667f);
  const float UV1 = -1.52488637914f * UV_s1 / (fabsf(UV_s1) - 1.4513954287f);
  const float xyD0 = 0.167171472114775f * UV0 + 0.141299802443708f * UV1 + -0.00801531300850582f;
  const float xyD1 = -0.150959086409163f * UV0 + -0.155185060382272f * UV1 + -0.00843312433578007f;
  const float xyD2 = 0.940254742367256f * UV0 + 1.000000000000000f * UV1 + -0.0256325967652889f;
  const float xo = xyD0 / xyD2, yo = xyD1 / xyD2;
  const float Yo = cb_pow((1.12426773749357f * L_s / (2.098883786377f - L_s)), 1.5831518565279648f); // dt_UCS_L_star_to_Y
  // dt_xyY_to_XYZ_simd
  const float y_over_x = Yo / yo;
  XYZ[0] = y_over_x * xo;
  XYZ[1] = Yo;
  XYZ[2] = y_over_x * (1.f - xo - yo);
}

template <int FORMULA>
__global__ void __launch_bounds__(CB_CNT) colorbalancergb_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, const size_t npixels,
                                                                 const __grid_constant__ cb_args_t a)
{
  __shared__ float lut[CB_LUT];
#ifdef B200_KERNELS_ON_CPU
  for(int k = 0; k < CB_LUT; k++) lut[k] = a.lut[k]; // the emulated threads run one after the other
#else
  for(int k = threadIdx.x; k < CB_LUT; k += CB_CNT) lut[k] = a.lut[k];
  __syncthreads();
#endif
  const size_t k = (size_t)blockIdx.x * CB_CNT + threadIdx.x;
  if(k >= npixels) return;
  const float4 px = in[k];

  const float RGB_in[3] = { max_zero(px.x), max_zero(px.y), max_zero(px.z) };
  float LMS[3], Yrg[3], RGB[3];
  mul3(a.in_m, RGB_in, LMS);
  lms_to_yrg(LMS, Yrg);
  Yrg[0] = cb_max(Yrg[0], 0.f);
  float op[3], comp[3];
  opacity_masks(cb_pow(Yrg[0], 0.4101205819200422f), a, op, comp);

  const float r_centered = Yrg[1] - D65_R;
  const float g_centered = Yrg[2] - D65_G;
  const float r_rotated = a.rot[0][0] * r_centered + a.rot[0][1] * g_centered;
  const float g_rotated = a.rot[1][0] * r_centered + a.rot[1][1] * g_centered;
  const float chroma_in = sqrtf(g_rotated * g_rotated + r_rotated * r_rotated);
  const float inv_chroma_in = (chroma_in > 0.f) ? 1.f / chroma_in : 0.f;
  const float cos_h = r_rotated * inv_chroma_in;
  const float sin_h = g_rotated * inv_chroma_in;
  const float chroma_boost = a.chroma_global + sp3(op, a.chroma);
  const float vibrance = a.vibrance * (1.0f - cb_pow(chroma_in, fabsf(a.vibrance)));
  const float chroma_factor = cb_max(1.f + chroma_boost + vibrance, 0.f);
  float chroma_out = chroma_in * chroma_factor;
  const float r_shifted = chroma_out * cos_h + D65_R;
  const float g_shifted = chroma_out * sin_h + D65_G;
  if(r_shifted < 0.f) chroma_out = cb_min(-D65_R / cos_h, chroma_out);
  if(g_shifted < 0.f) chroma_out = cb_min(-D65_G / sin_h, chroma_out);
  if(r_shifted + g_shifted > 1.f) chroma_out = cb_min((1.f - D65_R - D65_G) / (cos_h + sin_h), chroma_out);
  Yrg[1] = chroma_out * cos_h + D65_R;
  Yrg[2] = chroma_out * sin_h + D65_G;

  yrg_to_lms(Yrg, LMS);
  mul3(C_LMS_to_grading, LMS, RGB);
  for(int c = 0; c < 3; c++)
  {
    RGB[c] += a.global[c];
    RGB[c] *= comp[2] * (comp[0] + op[0] * a.shadows[c]) + op[2] * a.highlights[c];
  }
  for(int c = 0; c < 3; c++) RGB[c] = copysignf(cb_pow(fabsf(RGB[c]) / a.white_fulcrum, a.midtones[c]) * a.white_fulcrum, RGB[c]);

  mul3(C_grading_to_LMS, RGB, LMS);
  lms_to_yrg(LMS, Yrg);
  Yrg[0] = cb_pow(cb_max(Yrg[0] / a.white_fulcrum, 0.f), a.midtones_Y) * a.white_fulcrum;
  Yrg[0] = a.grey_fulcrum * cb_pow(Yrg[0] / a.grey_fulcrum, a.contrast);
  yrg_to_lms(Yrg, LMS);
  float XYZ[3];
  mul3(C_LMS_to_XYZ, LMS, XYZ);

  if(FORMULA == B200_COLORBALANCE_SATURATION_JZAZBZ) saturation_jzazbz(XYZ, op, lut, a);
  else saturation_dt_ucs(XYZ, op, lut, a);

  float o[3];
  mul3(a.out_m, XYZ, o);
  out[k] = make_float4(max_zero(o[0]), max_zero(o[1]), max_zero(o[2]), px.w);
}

// dt_colormatrix_mul (math/matrices.h:167-179): dst = m1 . m2, each sum from 0 in j order
void colormatrix_mul(float dst[3][3], const float m1[3][3], const float m2[3][3])
{
  for(int k = 0; k < 3; k++)
    for(int i = 0; i < 3; i++)
    {
      float sum = 0.0f;
      for(int j = 0; j < 3; j++) sum += m1[k][j] * m2[j][i];
      dst[k][i] = sum;
    }
}

// the part of process() before the pixel loop (:613-674) on the host, as the reference runs it there: the two matrix products,
// Y_to_dt_UCS_L_star(white_fulcrum) (colorspaces_inline_conversions.h:1261-1266) and the hue rotation, on the host's libm
void make_cb_args(const b200_colorbalancergb_piece_t *pc, cb_args_t *a)
{
  static const float XYZ_D50_to_D65_CAT16[3][3] = { { 9.89466254e-01f, -4.00304626e-02f, 4.40530317e-02f },
                                                    { -5.40518733e-03f, 1.00666069e+00f, -1.75551955e-03f },
                                                    { -4.03920992e-04f, 1.50768030e-02f, 1.30210211e+00f } };
  static const float XYZ_D65_to_D50_CAT16[3][3] = { { 1.01085433e+00f, 4.07086103e-02f, -3.41445825e-02f },
                                                    { 5.42814201e-03f, 9.93581926e-01f, 1.15592039e-03f },
                                                    { 2.50722468e-04f, -1.14918759e-02f, 7.67964947e-01f } };
  static const float XYZ_D65_to_LMS_2006_D65[3][3] = { { 0.257085f, 0.859943f, -0.031061f }, { -0.394427f, 1.175800f, 0.106423f },
                                                       { 0.064856f, -0.076250f, 0.559067f } };
  const b200_colorbalancergb_data_t *d = &pc->data;
  float work_in[3][3], work_out[3][3], tmp[3][3];
  for(int r = 0; r < 3; r++)
    for(int c = 0; c < 3; c++)
    {
      work_in[r][c] = pc->work_profile.matrix_in[r][c];
      work_out[r][c] = pc->work_profile.matrix_out[r][c];
    }
  colormatrix_mul(tmp, XYZ_D50_to_D65_CAT16, work_in);
  colormatrix_mul(a->in_m, XYZ_D65_to_LMS_2006_D65, tmp);
  colormatrix_mul(a->out_m, work_out, XYZ_D65_to_D50_CAT16);
  for(int c = 0; c < 3; c++)
  {
    a->global[c] = d->global[c];
    a->shadows[c] = d->shadows[c];
    a->highlights[c] = d->highlights[c];
    a->midtones[c] = d->midtones[c];
    a->chroma[c] = d->chroma[c];
    a->saturation[c] = d->saturation[c];
    a->brilliance[c] = d->brilliance[c];
  }
  a->chroma_global = d->chroma_global;
  a->vibrance = d->vibrance;
  a->contrast = d->contrast;
  a->saturation_global = d->saturation_global;
  a->brilliance_global = d->brilliance_global;
  a->midtones_Y = d->midtones_Y;
  a->shadows_weight = d->shadows_weight;
  a->highlights_weight = d->highlights_weight;
  a->midtones_weight = d->midtones_weight;
  a->mask_grey_fulcrum = d->mask_grey_fulcrum;
  a->white_fulcrum = d->white_fulcrum;
  a->grey_fulcrum = d->grey_fulcrum;
  const float Y_hat = powf(d->white_fulcrum, 0.631651345306265f);
  a->L_white = 2.098883786377f * Y_hat / (Y_hat + 1.12426773749357f);
  a->rot[0][0] = cosf(d->hue_angle);
  a->rot[0][1] = -sinf(d->hue_angle);
  a->rot[1][0] = sinf(d->hue_angle);
  a->rot[1][1] = cosf(d->hue_angle);
  a->two_pi = 2.f * CB_PI;
  a->d10000 = 10000.f;
  a->b = 1.15f;
  a->g = 0.66f;
  memcpy(a->lut, pc->gamut_LUT, sizeof(a->lut));
}
} // namespace

#ifndef B200_KERNELS_ON_CPU
using namespace b200;

static int cb_check(const b200_piece_t *piece, const void *in, const void *out)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "colorbalancergb: NULL argument");
  if(!piece->data || piece->data_size < sizeof(b200_colorbalancergb_piece_t))
    return fail(B200_ERR_ARG, "colorbalancergb: piece->data is not a b200_colorbalancergb_piece_t (data block + work profile matrices + gamut LUT)");
  if(in == out) return fail(B200_ERR_ARG, "colorbalancergb: in-place processing is not supported");
  if(piece->roi_out.width < 1 || piece->roi_out.height < 1) return fail(B200_ERR_ARG, "colorbalancergb: empty roi_out");
  if(((const b200_colorbalancergb_piece_t *)piece->data)->data.mask_display)
    return fail(B200_ERR_UNSUPPORTED, "colorbalancergb: the mask display is not built (a darkroom preview; its checkerboard is sized by the GUI's DPI)");
  return B200_OK;
}
extern "C" int b200_colorbalancergb_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = cb_check(piece, d_in, d_out);
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  const b200_colorbalancergb_piece_t *pc = (const b200_colorbalancergb_piece_t *)piece->data;
  cb_args_t a;
  make_cb_args(pc, &a);
  const size_t npx = (size_t)piece->roi_out.width * piece->roi_out.height;
  const unsigned grid = (unsigned)((npx + CB_CNT - 1) / CB_CNT);
  if(pc->data.saturation_formula == B200_COLORBALANCE_SATURATION_JZAZBZ)
    colorbalancergb_kernel<B200_COLORBALANCE_SATURATION_JZAZBZ><<<grid, CB_CNT, 0, (cudaStream_t)stream>>>((const float4 *)d_in, (float4 *)d_out, npx, a);
  else
    colorbalancergb_kernel<B200_COLORBALANCE_SATURATION_DTUCS><<<grid, CB_CNT, 0, (cudaStream_t)stream>>>((const float4 *)d_in, (float4 *)d_out, npx, a);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
extern "C" int b200_colorbalancergb_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = cb_check(piece, in, out);
  if(rc) return rc;
  const size_t bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 16;
  return through_device(piece, in, bytes, out, bytes, false, b200_colorbalancergb_process_dev); // lane 3 comes from the input (:920)
}
extern "C" void b200_colorbalancergb_tiling(const b200_piece_t *piece, b200_tiling_t *t) { default_tiling(piece, t, 0, false); } // the module declares no tiling callback
#endif
