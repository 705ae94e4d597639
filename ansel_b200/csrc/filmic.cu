// filmic rgb, AgX colour sciences (the v8 family, default = medium bleach): pointwise RGBA -> RGBA.
//
// Reference: src/iop/filmicrgb.c  process() :2707-2895 (AgX branch :2843-2856), filmic_agx :2495-2587,
// filmic_agx_compress_negatives :2461-2492, filmic_agx_prepare_bracket :2390-2459,
// _filmic_agx_build_displaced :2344-2388, filmic_v4_prepare_matrices :2033-2063, pipe_RGB_to_Ych_simd
// :1740-1760, Ych_to_pipe_RGB_simd :1763-1777, RGB_tone_mapping_v4_simd :2133-2149, log_tonemapping
// :1046-1051, filmic_spline :1062-1160, gamut_mapping_simd :1986-2030, gamut_check_RGB_simd :1949-1983,
// gamut_check_Yrg_filmic_simd :1928-1946, clip_chroma* :1826-1925, filmic_desaturate_v4 :1779-1816;
// common/colorspaces_inline_conversions.h :902-1075; pixel/chromatic_adaptation.h :248-261;
// math/matrices.h :37-65,167-206; system/simd.h :188-197.
//
// Parity contract: C-standard float semantics of that source (no contraction, IEEE division and sqrt,
// FTZ), glibc's powf/log2f on the device (flt32_math.cuh).  Bit-identical to the oracle, which is
// bit-identical to the reference functions cut verbatim from filmicrgb.c.
//
// Roofline: 32 B/px of HBM traffic against ~3 log2f + up to 9 powf (each a double-precision
// polynomial) + 5 sqrtf + ~30 IEEE divisions per pixel: FP64/XU-issue bound by an order of magnitude,
// not HBM bound (SURVEY.md 8d); reported as such.
//
// Code shape of filmic_agx_kernel.  Every helper was already inlined; what cost time was the size of the code and two arrays in
// local memory.  Steps, each on top of the previous one, timed by tools/time_filmic.py (the bench frame, v8 defaults with the export
// profile, median of 3 alternating rounds of 15 calls, outputs byte-identical) on an H100 80GB HBM3 at 700 W, 1980 MHz; SASS of the
// export instance (sm_90a, CUDA 12.9):
//
//   step                                                       instr  stack  LDL/STL  CALL  BSSY  regs   time
//   parent                                                      6512   32 B   41/20    158   272    38   4.37 ms
//   A  powf_special() returns by value; the tone loop rotates   6376    0      0/0     158   270    52   4.54 ms
//      its three channels through registers
//   B  + use_output_profile a template parameter                4288    0      0/0      96   173    46   4.45 ms
//   C  + one rolled copy of the three clip_white / clip_black,  2520    0      0/0      40    90    45   3.22 ms
//      one clip_white_raw per clip_white
//   D  + __launch_bounds__(128, 12): 40 registers, 48 warps     2520    0      0/0      40    90    38   3.14 ms
//
// A and B alone were slower: they raised the register count (36 resident warps per SM instead of 48) and saved little issue.  C
// paid: the three clip rows had been six inlined clip_white_raw and three clip_black, 41 % of B's code, and the kernel's code
// fell from 104 KB (parent) to 40 KB.  D gave back the occupancy.  All four are kept: D needs A's registers freed
// and C's smaller body.  What remains is divergence across the spline segments and the clip branches, which a pointwise kernel
// has no other pixel map to avoid, and the issue of the divisions and the FP64 libm cores.
#include "runtime.h"
#include <stddef.h>
#include "flt32_math.cuh"
#include <float.h>
#include <math.h>
#include <string.h>

namespace
{
typedef float m34[3][4];
#define CLAMPF(a, mn, mx) ((a) >= (mn) ? ((a) <= (mx) ? (a) : (mx)) : (mn))
#define CLAMPG(x, lo, hi) (((x) > (hi)) ? (hi) : (((x) < (lo)) ? (lo) : (x)))
#define MINF(a, b) (((a) < (b)) ? (a) : (b))
#define MAXF(a, b) (((a) > (b)) ? (a) : (b))
#define Y31_TO_Y06(x) (1.05785528f * (x))

struct filmic_args_t
{
  m34 input, output, export_input, export_output, inset, outset;
  float luma[4];
  int use_output_profile;
  b200_filmic_spline_t spline;
  float grey_source, black_source, dynamic_range, output_power, agx_beta_hue;
  float black, white;
  int copy_alpha;
  // colour sciences before AgX
  int version, preserve_color;
  float saturation, sigma_toe, sigma_shoulder, norm_min, norm_max;
  float work_lum[4]; // row 1 of the work profile's RGB -> XYZ matrix
};

// ---- host-side set-up: plain C float arithmetic + the host libm (cosf, sinf, powf) --------------
const m34 XYZ_D50_to_D65_CAT16 = { { 9.89466254e-01f, -4.00304626e-02f, 4.40530317e-02f, 0.f },
                                   { -5.40518733e-03f, 1.00666069e+00f, -1.75551955e-03f, 0.f },
                                   { -4.03920992e-04f, 1.50768030e-02f, 1.30210211e+00f, 0.f } };
const m34 XYZ_D65_to_D50_CAT16 = { { 1.01085433e+00f, 4.07086103e-02f, -3.41445825e-02f, 0.f },
                                   { 5.42814201e-03f, 9.93581926e-01f, 1.15592039e-03f, 0.f },
                                   { 2.50722468e-04f, -1.14918759e-02f, 7.67964947e-01f, 0.f } };
const m34 XYZ_D65_to_LMS = { { 0.257085f, 0.859943f, -0.031061f, 0.f }, { -0.394427f, 1.175800f, 0.106423f, 0.f }, { 0.064856f, -0.076250f, 0.559067f, 0.f } };
const m34 LMS_to_XYZ_D65 = { { 1.80794659f, -1.29971660f, 0.34785879f, 0.f },
                             { 0.61783960f, 0.39595453f, -0.04104687f, 0.f },
                             { -0.12546960f, 0.20478038f, 1.74274183f, 0.f } };
const m34 H_filmlightRGB_to_LMS = { { 0.95f, 0.38f, 0.00f, 0.f }, { 0.05f, 0.62f, 0.03f, 0.f }, { 0.00f, 0.00f, 0.97f, 0.f } };
const m34 H_LMS_to_filmlightRGB = { { 1.0877193f, -0.66666667f, 0.02061856f, 0.f }, { -0.0877193f, 1.66666667f, -0.05154639f, 0.f }, { 0.f, 0.f, 1.03092784f, 0.f } };

// scalar_product() (math/math.h:185-195) is an `omp simd reduction` loop; gcc reduces its 4-lane vector
// pairwise: (p0 + p2) + (p1 + 0).  Pinned against the compiled reference (tests/test_cpu_oracle_pin.py).
void dot3(const float v[4], const m34 M, float out[4])
{
  for(int i = 0; i < 3; i++)
  {
    const float p0 = v[0] * M[i][0], p1 = v[1] * M[i][1], p2 = v[2] * M[i][2];
    out[i] = (p0 + p2) + p1;
  }
}
void mmul(m34 dst, const m34 m1, const m34 m2) // dt_colormatrix_mul, matrices.h:167-179
{
  m34 r;
  for(int k = 0; k < 3; k++)
    for(int i = 0; i < 4; i++)
    {
      float sum = 0.0f;
      for(int j = 0; j < 3; j++) sum += m1[k][j] * m2[j][i];
      r[k][i] = sum;
    }
  memcpy(dst, r, sizeof(r));
}
int minv(m34 dst, const m34 src) // mat3SSEinv, matrices.h:37-65
{
#define A(y, x) src[(y - 1)][(x - 1)]
#define B(y, x) dst[(y - 1)][(x - 1)]
  const float det = A(1, 1) * (A(3, 3) * A(2, 2) - A(3, 2) * A(2, 3)) - A(2, 1) * (A(3, 3) * A(1, 2) - A(3, 2) * A(1, 3))
                    + A(3, 1) * (A(2, 3) * A(1, 2) - A(2, 2) * A(1, 3));
  if(fabsf(det) < 1e-7f) return 1;
  const float invDet = 1.f / det;
  B(1, 1) = invDet * (A(3, 3) * A(2, 2) - A(3, 2) * A(2, 3));
  B(1, 2) = -invDet * (A(3, 3) * A(1, 2) - A(3, 2) * A(1, 3));
  B(1, 3) = invDet * (A(2, 3) * A(1, 2) - A(2, 2) * A(1, 3));
  B(2, 1) = -invDet * (A(3, 3) * A(2, 1) - A(3, 1) * A(2, 3));
  B(2, 2) = invDet * (A(3, 3) * A(1, 1) - A(3, 1) * A(1, 3));
  B(2, 3) = -invDet * (A(2, 3) * A(1, 1) - A(2, 1) * A(1, 3));
  B(3, 1) = invDet * (A(3, 2) * A(2, 1) - A(3, 1) * A(2, 2));
  B(3, 2) = -invDet * (A(3, 2) * A(1, 1) - A(3, 1) * A(1, 2));
  B(3, 3) = invDet * (A(2, 2) * A(1, 1) - A(2, 1) * A(1, 2));
#undef A
#undef B
  return 0;
}
void ident(m34 M)
{
  memset(M, 0, sizeof(m34));
  M[0][0] = M[1][1] = M[2][2] = 1.f;
}
void h_lms_to_yrg(const float LMS[4], float Yrg[4]) // colorspaces_inline_conversions.h:1014-1031
{
  const float Y = 0.68990272f * LMS[0] + 0.34832189f * LMS[1];
  const float a = LMS[0] + LMS[1] + LMS[2];
  float lms[4] = { 0 }, rgb[4] = { 0 };
  for(int c = 0; c < 4; c++) lms[c] = (a == 0.f) ? 0.f : LMS[c] / a;
  dot3(lms, H_LMS_to_filmlightRGB, rgb);
  Yrg[0] = Y;
  Yrg[1] = rgb[0];
  Yrg[2] = rgb[1];
}
void h_yrg_to_lms(const float Yrg[4], float LMS[4]) // :1045-1063
{
  const float Y = Yrg[0], r = Yrg[1], g = Yrg[2], b = 1.f - r - g;
  const float rgb[4] = { r, g, b, 0.f };
  float lms[4] = { 0 };
  dot3(rgb, H_filmlightRGB_to_LMS, lms);
  const float denom = (0.68990272f * lms[0] + 0.34832189f * lms[1]);
  const float a = (denom == 0.f) ? 0.f : Y / denom;
  for(int c = 0; c < 4; c++) LMS[c] = lms[c] * a;
}
void xyz50_to_yrg(const float xyz[4], float Yrg[4]) // filmicrgb.c:2314-2321
{
  float d65[4] = { 0 }, lms[4] = { 0 };
  dot3(xyz, XYZ_D50_to_D65_CAT16, d65);
  dot3(d65, XYZ_D65_to_LMS, lms);
  h_lms_to_yrg(lms, Yrg);
}
void yrg_to_xyz50(const float Yrg[4], float xyz[4]) // :2323-2330
{
  float lms[4] = { 0 }, d65[4] = { 0 };
  h_yrg_to_lms(Yrg, lms);
  dot3(lms, LMS_to_XYZ_D65, d65);
  dot3(d65, XYZ_D65_to_D50_CAT16, xyz);
}
bool build_displaced(const m34 work_in, const m34 work_out, const float inset[3], const float rotation[3], m34 M) // :2344-2388
{
  float white_xyz[4] = { 0 }, white_Yrg[4] = { 0 };
  for(int r = 0; r < 3; r++)
    for(int c = 0; c < 3; c++) white_xyz[r] += work_in[r][c];
  xyz50_to_yrg(white_xyz, white_Yrg);
  m34 P = { { 0 } };
  for(int i = 0; i < 3; i++)
  {
    const float pxyz[4] = { work_in[0][i], work_in[1][i], work_in[2][i], 0.f };
    float pY[4] = { 0 };
    xyz50_to_yrg(pxyz, pY);
    const float dr = pY[1] - white_Yrg[1], dg = pY[2] - white_Yrg[2];
    const float scale = 1.f - CLAMPF(inset[i], 0.f, 0.9f);
    const float cos_a = cosf(rotation[i]), sin_a = sinf(rotation[i]);
    const float dY[4] = { pY[0], white_Yrg[1] + scale * (cos_a * dr - sin_a * dg), white_Yrg[2] + scale * (sin_a * dr + cos_a * dg), 0.f };
    float dxyz[4] = { 0 };
    yrg_to_xyz50(dY, dxyz);
    for(int r = 0; r < 3; r++) P[r][i] = dxyz[r];
  }
  m34 Pinv = { { 0 } };
  if(minv(Pinv, P)) return false;
  float s[4] = { 0 };
  dot3(white_xyz, Pinv, s);
  for(int r = 0; r < 3; r++)
    for(int c = 0; c < 3; c++) P[r][c] *= s[c];
  mmul(M, work_out, P);
  return true;
}

// filmic_v4_prepare_matrices :2033-2063 + filmic_agx_prepare_bracket :2390-2459
void prepare(filmic_args_t *m, int version, const m34 work_in, const m34 work_out, const m34 *exp_in, const m34 *exp_out)
{
  m34 tmp;
  mmul(tmp, XYZ_D50_to_D65_CAT16, work_in);
  mmul(m->input, XYZ_D65_to_LMS, tmp);
  mmul(tmp, XYZ_D65_to_D50_CAT16, LMS_to_XYZ_D65);
  mmul(m->output, work_out, tmp);
  m->use_output_profile = exp_in != nullptr;
  if(exp_in)
  {
    mmul(tmp, XYZ_D65_to_D50_CAT16, LMS_to_XYZ_D65);
    mmul(m->export_output, *exp_out, tmp);
    mmul(tmp, XYZ_D50_to_D65_CAT16, *exp_in);
    mmul(m->export_input, XYZ_D65_to_LMS, tmp);
  }
  // inset anchor, inset rotation, outset anchor, outset rotation per variant (filmicrgb.c:2408-2445)
  static const float K[5][12] = {
    { 0.5991055f, 0.6000000f, 0.3300009f, 0.0571015f, 0.1999891f, 0.0886110f, 0.761433f, 0.752267f, 0.465293f, -0.0034297f, 0.1952448f, -0.0480109f },
    { 0.6410825f, 0.6898110f, 0.3194529f, 0.0405734f, 0.1631286f, 0.0350584f, 0.784757f, 0.789387f, 0.445403f, -0.0057845f, 0.1593207f, -0.0592955f },
    { 0.6509540f, 0.7488775f, 0.3517703f, 0.0278602f, 0.1214671f, -0.0228829f, 0.793082f, 0.815169f, 0.460318f, -0.0053781f, 0.1187604f, -0.0794801f },
    { 0.6379749f, 0.7878689f, 0.3753822f, 0.0106096f, 0.0582598f, -0.0696729f, 0.790237f, 0.831376f, 0.465406f, -0.0080070f, 0.0571100f, -0.0912220f },
    { 0.5770235f, 0.8102094f, 0.4000390f, -0.0081060f, -0.0034008f, -0.1035236f, 0.766420f, 0.838020f, 0.465130f, -0.0122011f, -0.0021732f, -0.0971215f },
  };
  const int row = (version >= 5 && version <= 9) ? version - 5 : 0;
  m34 rec = { { 0 } };
  if(!build_displaced(work_in, work_out, K[row], K[row] + 3, m->inset) || !build_displaced(work_in, work_out, K[row] + 6, K[row] + 9, rec)
     || minv(m->outset, rec))
  {
    ident(m->inset);
    ident(m->outset);
  }
  m->luma[0] = work_in[1][0];
  m->luma[1] = work_in[1][1];
  m->luma[2] = work_in[1][2];
  m->luma[3] = 0.f;
}

// ---- device ------------------------------------------------------------------------------------
__device__ const float D_filmlightRGB_to_LMS[3][4] = { { 0.95f, 0.38f, 0.00f, 0.f }, { 0.05f, 0.62f, 0.03f, 0.f }, { 0.00f, 0.00f, 0.97f, 0.f } };
__device__ const float D_LMS_to_filmlightRGB[3][4] = { { 1.0877193f, -0.66666667f, 0.02061856f, 0.f },
                                                       { -0.0877193f, 1.66666667f, -0.05154639f, 0.f },
                                                       { 0.f, 0.f, 1.03092784f, 0.f } };

// dt_mat3x4_mul_vec4 on the transposed rows of M: lane i = (M[i][0]*x + M[i][1]*y) + M[i][2]*z
__device__ __forceinline__ void mat4(const float (*M)[4], const float in[4], float out[4])
{
  float r[4];
#pragma unroll
  for(int i = 0; i < 4; i++)
  {
    const float a = i < 3 ? M[i][0] : 0.f, b = i < 3 ? M[i][1] : 0.f, c = i < 3 ? M[i][2] : 0.f;
    float acc = a * in[0];
    acc = b * in[1] + acc;
    r[i] = c * in[2] + acc;
  }
#pragma unroll
  for(int i = 0; i < 4; i++) out[i] = r[i];
}
__device__ __forceinline__ void lms_to_yrg(const float LMS[4], float Yrg[4])
{
  const float Y = 0.68990272f * LMS[0] + 0.34832189f * LMS[1];
  const float a = LMS[0] + LMS[1] + LMS[2];
  const float inv_a = (a == 0.f) ? 0.f : 1.f / a;
  const float lms[4] = { LMS[0] * inv_a, LMS[1] * inv_a, LMS[2] * inv_a, 0.f };
  float rgb[4];
  mat4(D_LMS_to_filmlightRGB, lms, rgb);
  Yrg[0] = Y;
  Yrg[1] = rgb[0];
  Yrg[2] = rgb[1];
  Yrg[3] = 0.f;
}
__device__ __forceinline__ void yrg_to_lms(const float Yrg[4], float LMS[4])
{
  const float rgb[4] = { Yrg[1], Yrg[2], 1.f - Yrg[1] - Yrg[2], 0.f };
  float lms[4];
  mat4(D_filmlightRGB_to_LMS, rgb, lms);
  const float denom = 0.68990272f * lms[0] + 0.34832189f * lms[1];
  const float a = (denom == 0.f) ? 0.f : Yrg[0] / denom;
  LMS[0] = lms[0] * a;
  LMS[1] = lms[1] * a;
  LMS[2] = lms[2] * a;
  LMS[3] = 0.f;
}
__device__ __forceinline__ void rgb_to_ych(const float in[4], const float (*M)[4], float Ych[4])
{
  float lms[4], Yrg[4];
  mat4(M, in, lms);
  lms_to_yrg(lms, Yrg);
  const float r = Yrg[1] - 0.21902143f, g = Yrg[2] - 0.54371398f;
  const float c = sqrtf(g * g + r * r);
  Ych[0] = Yrg[0];
  Ych[1] = c;
  Ych[2] = c != 0.f ? r / c : 1.f;
  Ych[3] = c != 0.f ? g / c : 0.f;
}
__device__ __forceinline__ void ych_to_rgb(const float in[4], const float (*M)[4], float out[4])
{
  const float Yrg[4] = { in[0], in[1] * in[2] + 0.21902143f, in[1] * in[3] + 0.54371398f, 0.f };
  float lms[4];
  yrg_to_lms(Yrg, lms);
  mat4(M, lms, out);
}

// filmic_spline(), :1062-1160
__device__ float spline_eval(const f32m::tables_t &tb, float x, const b200_filmic_spline_t &s)
{
  const float *M1 = s.M1, *M2 = s.M2, *M3 = s.M3, *M4 = s.M4, *M5 = s.M5;
  float result;
  if(x < s.latitude_min)
  {
    if(s.type[0] == 3)
    {
      if(M5[0] != 0.f)
        result = M3[2] + fmaxf(0.f, M3[0] * f32m::powf_(tb, fmaxf(x, 0.f), M4[0]));
      else
      {
        const float ty = s.latitude_min * M2[2] + M1[2];
        const float u = M2[2] * (x - s.latitude_min) / M1[0];
        result = M1[0] * (u / f32m::powf_(tb, 1.f + f32m::powf_(tb, u, M2[0]), 1.f / M2[0])) + ty;
      }
    }
    else if(s.type[0] == 0)
      result = M1[0] + x * (M2[0] + x * (M3[0] + x * (M4[0] + x * M5[0])));
    else if(s.type[0] == 1)
      result = M1[0] + x * (M2[0] + x * (M3[0] + x * M4[0]));
    else
    {
      const float xi = s.latitude_min - x;
      const float rat = xi * (xi * M2[0] + 1.f);
      result = M4[0] - M1[0] * rat / (rat + M3[0]);
    }
  }
  else if(x > s.latitude_max)
  {
    if(s.type[1] == 3)
    {
      if(M5[1] != 0.f)
        result = M4[2] - fmaxf(0.f, M3[1] * f32m::powf_(tb, fmaxf(1.f - x, 0.f), M4[1]));
      else
      {
        const float ty = s.latitude_max * M2[2] + M1[2];
        const float u = M2[2] * (x - s.latitude_max) / M1[1];
        result = M1[1] * (u / f32m::powf_(tb, 1.f + f32m::powf_(tb, u, M2[1]), 1.f / M2[1])) + ty;
      }
    }
    else if(s.type[1] == 0)
      result = M1[1] + x * (M2[1] + x * (M3[1] + x * (M4[1] + x * M5[1])));
    else if(s.type[1] == 1)
      result = M1[1] + x * (M2[1] + x * (M3[1] + x * M4[1]));
    else
    {
      const float xi = x - s.latitude_max;
      const float rat = xi * (xi * M2[1] + 1.f);
      result = M4[1] + M1[1] * rat / (rat + M3[1]);
    }
  }
  else
    result = M1[2] + x * M2[2];
  return result;
}

__device__ __forceinline__ float clip_white_raw(const float co[4], float tw, float Y, float ch, float sh)
{
  const float dY = co[0] * (0.979381443298969f * ch + 0.391752577319588f * sh) + co[1] * (0.0206185567010309f * ch + 0.608247422680412f * sh)
                   - co[2] * (ch + sh);
  const float dt = tw * (0.68285981628866f * ch + 0.482137060515464f * sh);
  if(dY == 0.f) return FLT_MAX;
  const float Ya = dt / dY;
  if(Y <= Ya) return FLT_MAX;
  const float den = Y * dY - dt;
  const float num = -0.427506877216495f * (Y * (co[0] + 0.856492345150334f * co[1] + 0.554995960637719f * co[2]) - 0.988237752433297f * tw);
  return num / den;
}
__device__ __forceinline__ float clip_white(const float co[4], float tw, float Y, float ch, float sh)
{
  const float eps = 1e-3f;
  const float max_Y = Y31_TO_Y06(tw);
  const float delta_Y = MAXF(max_Y - Y, 0.f);
  // both branches of the reference evaluate clip_white_raw(), at different Y: one inlined copy serves them
  const bool near_white = delta_Y < eps;
  const float raw = clip_white_raw(co, tw, near_white ? (1.f - eps) * max_Y : Y, ch, sh);
  const float mc = near_white ? delta_Y / (eps * max_Y) * raw : raw;
  return mc >= 0.f ? mc : FLT_MAX;
}
__device__ __forceinline__ float clip_black(const float co[4], float ch, float sh)
{
  const float den = co[0] * (0.979381443298969f * ch + 0.391752577319588f * sh) + co[1] * (0.0206185567010309f * ch + 0.608247422680412f * sh)
                    - co[2] * (ch + sh);
  if(den == 0.f) return FLT_MAX;
  const float num = -0.427506877216495f * (co[0] + 0.856492345150334f * co[1] + 0.554995960637719f * co[2]);
  const float mc = num / den;
  return mc >= 0.f ? mc : FLT_MAX;
}
__device__ __forceinline__ float clip_chroma(const float (*out_m)[4], float tw, float Y, float ch, float sh, float chroma)
{
  // one rolled copy of the clips serves the three rows of out_m; the folds keep the reference's order, MINF(MINF(r0, r1), r2)
  float w = 0.f, b = 0.f;
#pragma unroll 1
  for(int i = 0; i < 3; i++)
  {
    const float wi = clip_white(out_m[i], tw, Y, ch, sh), bi = clip_black(out_m[i], ch, sh);
    w = i == 0 ? wi : MINF(w, wi);
    b = i == 0 ? bi : MINF(b, bi);
  }
  return MINF(MINF(chroma, b), w);
}
__device__ void gamut_check_rgb(const float (*m_out)[4], const float (*m_in)[4], float black, float white, const float Ych[4], float out[4])
{
  float bright[4];
  ych_to_rgb(Ych, m_out, bright);
  const float min_pix = MINF(MINF(bright[0], bright[1]), bright[2]);
  const float off = MAXF(-min_pix, 0.f);
#pragma unroll
  for(int c = 0; c < 4; c++) bright[c] += off;
  float Yb[4];
  rgb_to_ych(bright, m_in, Yb);
  const float Ym = (Ych[0] + Yb[0]) / 2.f;
  const float Y = CLAMPG(Ym, Y31_TO_Y06(black), Y31_TO_Y06(white));
  const float nc = clip_chroma(m_out, white, Y, Ych[2], Ych[3], Ych[1]);
  const float t[4] = { Y, nc, Ych[2], Ych[3] };
  ych_to_rgb(t, m_out, out);
#pragma unroll
  for(int c = 0; c < 4; c++) out[c] = CLAMPG(out[c], 0.f, white);
}

// gamut_mapping_simd(), :1986-2030 (filmic_desaturate_v4 :1779-1816, gamut_check_Yrg_filmic_simd :1928-1946).
// EXPORT = a.use_output_profile, the same for every pixel of a launch: each kernel instance compiles one of the two
// gamut checks.
template <bool EXPORT>
__device__ __forceinline__ void gamut_map(const filmic_args_t &a, float Yf[4], const float Yr[4], float saturation, float res[4])
{
  Yf[2] = Yr[2];
  Yf[3] = Yr[3];
  Yf[0] = CLAMPG(Yf[0], Y31_TO_Y06(a.black), Y31_TO_Y06(a.white));
  {
    const float c_o = Yr[1] * Yr[0];
    float c_f = Yf[1] * Yf[0];
    const float delta = saturation * (c_o - c_f);
    const bool brightens = (Yf[0] > Yr[0]), resat = (c_o < c_f), desat = (c_o > c_f);
    const bool u_resat = (saturation > 0.f), u_desat = (saturation < 0.f);
    c_f = (brightens && resat) ? (c_o + c_f) / 2.f : (((u_resat && desat) || u_desat) ? c_f + delta : c_f);
    Yf[1] = fmaxf(c_f / Yf[0], 0.f);
  }
  {
    const float y1 = Yf[1] * Yf[2] + 0.21902143f, y2 = Yf[1] * Yf[3] + 0.54371398f;
    float max_c = Yf[1];
    if(y1 < 0.f) max_c = fminf(-0.21902143f / Yf[2], max_c);
    if(y2 < 0.f) max_c = fminf(-0.54371398f / Yf[3], max_c);
    if(y1 + y2 > 1.f) max_c = fminf((1.f - 0.21902143f - 0.54371398f) / (Yf[2] + Yf[3]), max_c);
    Yf[1] = max_c;
  }
  if(!EXPORT)
    gamut_check_rgb(a.output, a.input, a.black, a.white, Yf, res);
  else
  {
    float px[4], lms[4];
    gamut_check_rgb(a.export_output, a.export_input, a.black, a.white, Yf, px);
    mat4(a.export_input, px, lms);
    mat4(a.output, lms, res);
  }
}

// 12 blocks per SM hold the kernel at 40 registers and 48 resident warps; left free, ptxas takes 45 and 36 warps fit (step D above)
template <bool EXPORT>
__global__ void __launch_bounds__(128, 12) filmic_agx_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, size_t npx,
                                                         const __grid_constant__ filmic_args_t a)
{
  __shared__ double tabs[f32m::SMEM_DOUBLES];
  const f32m::tables_t tb = f32m::stage_tables(tabs, threadIdx.x, 128);
  __syncthreads();
  const size_t k = (size_t)blockIdx.x * 128 + threadIdx.x;
  if(k >= npx) return;
  const float4 p = __ldcs(in + k);
  float pix[4] = { p.x, p.y, p.z, p.w };
#pragma unroll
  for(int c = 0; c < 3; c++) pix[c] = (pix[c] != pix[c]) ? 0.f : CLAMPF(pix[c], -1e6f, 1e6f);

  // filmic_agx_compress_negatives(), :2461-2492
  float cmp[4];
  {
    const float *lc = a.luma;
    const float input_y = pix[0] * lc[0] + pix[1] * lc[1] + pix[2] * lc[2];
    const float max_rgb = fmaxf(fmaxf(pix[0], pix[1]), pix[2]);
    const float min_rgb = fminf(fminf(pix[0], pix[1]), pix[2]);
    float opp[4];
#pragma unroll
    for(int c = 0; c < 4; c++) opp[c] = max_rgb - pix[c];
    const float opp_y = opp[0] * lc[0] + opp[1] * lc[1] + opp[2] * lc[2];
    const float max_opp = fmaxf(fmaxf(opp[0], opp[1]), opp[2]);
    const float y_comp = max_opp - opp_y + input_y;
    const float offset = fmaxf(-min_rgb, 0.f);
    float sh[4];
#pragma unroll
    for(int c = 0; c < 4; c++) sh[c] = pix[c] + offset;
    const float max_sh = fmaxf(fmaxf(sh[0], sh[1]), sh[2]);
    float os[4];
#pragma unroll
    for(int c = 0; c < 4; c++) os[c] = max_sh - sh[c];
    const float max_os = fmaxf(fmaxf(os[0], os[1]), os[2]);
    const float y_os = os[0] * lc[0] + os[1] * lc[1] + os[2] * lc[2];
    float y_new = sh[0] * lc[0] + sh[1] * lc[1] + sh[2] * lc[2];
    y_new += max_os - y_os;
    const float ratio = (y_new > y_comp && y_new > 1e-6f) ? y_comp / y_new : 1.f;
#pragma unroll
    for(int c = 0; c < 4; c++) cmp[c] = sh[c] * ratio;
  }

  float Yo[4];
  rgb_to_ych(cmp, a.input, Yo);
  float ren[4];
  mat4(a.inset, cmp, ren);
  // RGB_tone_mapping_v4_simd(), :2133-2149.  One rolled copy of the curve serves the three channels; they rotate
  // through ren[0..2] so that no array is indexed at run time (that would place it in local memory).
#pragma unroll 1
  for(int c = 0; c < 3; c++)
  {
    const float lg = fminf(fmaxf((f32m::log2f_(tb, ren[0] / a.grey_source) - a.black_source) / a.dynamic_range, 0.0f), 1.0f);
    const float sp = spline_eval(tb, lg, a.spline);
    ren[0] = ren[1];
    ren[1] = ren[2];
    ren[2] = f32m::powf_(tb, CLAMPF(sp, 0.f, a.spline.y[4]), a.output_power);
  }
  float po[4];
  mat4(a.outset, ren, po);
  float Yf[4];
  rgb_to_ych(po, a.input, Yf);
  const float chroma_final = fminf(Yo[1], Yf[1]);
  const float beta = a.agx_beta_hue;
  const float r_mix = beta * Yo[1] * Yo[2] + (1.f - beta) * chroma_final * Yf[2];
  const float g_mix = beta * Yo[1] * Yo[3] + (1.f - beta) * chroma_final * Yf[3];
  const float norm_mix = sqrtf(g_mix * g_mix + r_mix * r_mix);
  const float Yr[4] = { Yo[0], Yo[1], (norm_mix > 1e-9f) ? r_mix / norm_mix : Yo[2], (norm_mix > 1e-9f) ? g_mix / norm_mix : Yo[3] };
  Yf[1] = chroma_final;

  float res[4];
  gamut_map<EXPORT>(a, Yf, Yr, 0.f, res);
  if(a.copy_alpha) res[3] = p.w; // dt_iop_alpha_copy when the pipe displays a mask (:2893-2894)
  __stcs(out + k, make_float4(res[0], res[1], res[2], res[3]));
}

// ---- the colour sciences before AgX (filmicrgb.c:2857-2887): "v3 (2019)" .. "v7 (2023)" ------------------------
#define NORM_MIN 1.52587890625e-05f // math/math.h:37
__device__ __forceinline__ float clamp01(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); } // clamp_simd
__device__ __forceinline__ float log_tm(const f32m::tables_t &tb, const filmic_args_t &a, float x)
{ // log_tonemapping(), :1047-1051
  return clamp01((f32m::log2f_(tb, x / a.grey_source) - a.black_source) / a.dynamic_range);
}
__device__ __forceinline__ float lum_work(const filmic_args_t &a, const float p[4]) { return a.work_lum[0] * p[0] + a.work_lum[1] * p[1] + a.work_lum[2] * p[2]; }
__device__ float pixel_norm(const filmic_args_t &a, const float p[4], int variant)
{ // get_pixel_norm_simd(), :976-1038
  switch(variant)
  {
    case 1: return fmaxf(fmaxf(p[0], p[1]), p[2]);
    case 3:
    { // pixel_rgb_norm_power_simd(), :949-967
      float num = 0.0f, den = 0.0f;
#pragma unroll
      for(int c = 0; c < 3; c++)
      {
        const float v = fabsf(p[c]);
        const float sq = v * v;
        const float cu = sq * v;
        num += cu;
        den += sq;
      }
      return num / fmaxf(den, 1e-12f);
    }
    case 4: return sqrtf(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    case 5: return sqrtf(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]) * 0.5773502691896258f;
    default: return lum_work(a, p);
  }
}
__device__ float desat_v1(const f32m::tables_t &tb, const filmic_args_t &a, float x)
{ // filmic_desaturate_v1(), :1164-1175
  const float rt = x, rs = 1.0f - x;
  const float kt = f32m::expf_(tb, -0.5f * rt * rt / a.sigma_toe), ks = f32m::expf_(tb, -0.5f * rs * rs / a.sigma_shoulder);
  return 1.0f - clamp01((kt + ks) / a.saturation);
}
__device__ float desat_v2(const f32m::tables_t &tb, const filmic_args_t &a, float x)
{ // filmic_desaturate_v2(), :1178-1189
  const float rt = x, rs = 1.0f - x;
  const float sat2 = 0.5f / sqrtf(a.saturation);
  const float kt = f32m::expf_(tb, -rt * rt / a.sigma_toe * sat2), ks = f32m::expf_(tb, -rs * rs / a.sigma_shoulder * sat2);
  return (a.saturation - (kt + ks) * (a.saturation));
}
__device__ float curve_out(const f32m::tables_t &tb, const filmic_args_t &a, float x, float lo)
{
  return f32m::powf_(tb, CLAMPF(spline_eval(tb, x, a.spline), lo, a.spline.y[4]), a.output_power);
}
__device__ void norm_tm_v4(const f32m::tables_t &tb, const filmic_args_t &a, const float in[4], int variant, float o[4])
{ // norm_tone_mapping_v4_simd(), :2106-2131
  float norm = CLAMPF(pixel_norm(a, in, variant), a.norm_min, a.norm_max);
  float ratios[4];
#pragma unroll
  for(int c = 0; c < 4; c++) ratios[c] = in[c] / norm;
  norm = log_tm(tb, a, norm);
  norm = curve_out(tb, a, norm, a.spline.y[0]);
#pragma unroll
  for(int c = 0; c < 4; c++) o[c] = ratios[c] * norm;
}
__device__ void rgb_tm_v4(const f32m::tables_t &tb, const filmic_args_t &a, const float in[4], float o[4])
{ // RGB_tone_mapping_v4_simd(), :2133-2149
#pragma unroll
  for(int c = 0; c < 3; c++) o[c] = curve_out(tb, a, log_tm(tb, a, in[c]), 0.f);
  o[3] = in[3];
}

__global__ void __launch_bounds__(128) filmic_legacy_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, size_t npx, const filmic_args_t a)
{
  __shared__ double tabs[f32m::SMEM_DOUBLES];
  const f32m::tables_t tb = f32m::stage_tables(tabs, threadIdx.x, 128);
  __syncthreads();
  const size_t k = (size_t)blockIdx.x * 128 + threadIdx.x;
  if(k >= npx) return;
  const float4 p = __ldcs(in + k);
  const float pix[4] = { p.x, p.y, p.z, p.w };
  float res[4] = { 0.f, 0.f, 0.f, p.w };
  if(a.version >= 3)
  { // filmic_chroma_v4 :2153-2198, filmic_split_v4 :2201-2243, filmic_v5 :2247-2299
    float po[4], Yo[4], Yf[4];
    float saturation = a.saturation;
    bool clamp_chroma = false;
    if(a.version == 4)
    {
      float naive[4], maxrgb[4];
      rgb_tm_v4(tb, a, pix, naive);
      norm_tm_v4(tb, a, pix, 1, maxrgb);
#pragma unroll
      for(int c = 0; c < 4; c++) po[c] = (0.5f + a.saturation) * maxrgb[c];
#pragma unroll
      for(int c = 0; c < 4; c++) po[c] = (0.5f - a.saturation) * naive[c] + po[c];
      saturation = 0.f;
      clamp_chroma = true;
    }
    else if(a.preserve_color == 0)
    {
      rgb_tm_v4(tb, a, pix, po);
      clamp_chroma = true;
    }
    else
      norm_tm_v4(tb, a, pix, a.preserve_color, po);
    rgb_to_ych(pix, a.input, Yo);
    rgb_to_ych(po, a.input, Yf);
    if(clamp_chroma) Yf[1] = fminf(Yo[1], Yf[1]);
    if(a.use_output_profile)
      gamut_map<true>(a, Yf, Yo, saturation, res);
    else
      gamut_map<false>(a, Yf, Yo, saturation, res);
  }
  else if(a.preserve_color == 0)
  { // filmic_split_v1 :1534-1571, filmic_split_v2_v3 :1575-1612; lane 3 is not written by the reference: the input's is kept
    float temp[4];
#pragma unroll
    for(int c = 0; c < 3; c++) temp[c] = log_tm(tb, a, fmaxf(pix[c], NORM_MIN));
    const float lum = lum_work(a, temp);
    const float desat = a.version == 0 ? desat_v1(tb, a, lum) : desat_v2(tb, a, lum);
#pragma unroll
    for(int c = 0; c < 3; c++) res[c] = curve_out(tb, a, lum + desat * (temp[c] - lum), a.spline.y[0]); // linear_saturation :1193-1196
  }
  else
  { // filmic_chroma_v1 :1616-1666, filmic_chroma_v2_v3 :1670-1737
    float norm = fmaxf(pixel_norm(a, pix, a.preserve_color), NORM_MIN);
    float ratios[4];
#pragma unroll
    for(int c = 0; c < 4; c++) ratios[c] = pix[c] / norm;
    const float min_ratios = fminf(fminf(ratios[0], ratios[1]), ratios[2]);
    if(min_ratios < 0.0f)
    {
#pragma unroll
      for(int c = 0; c < 4; c++) ratios[c] -= min_ratios;
    }
    norm = log_tm(tb, a, norm);
    if(a.version == 0)
    {
      const float desat = desat_v1(tb, a, norm);
#pragma unroll
      for(int c = 0; c < 4; c++) ratios[c] *= norm;
      const float lum = lum_work(a, ratios);
#pragma unroll
      for(int c = 0; c < 3; c++) ratios[c] = (lum + desat * (ratios[c] - lum)) / norm;
      norm = curve_out(tb, a, norm, a.spline.y[0]);
#pragma unroll
      for(int c = 0; c < 4; c++) res[c] = ratios[c] * norm;
    }
    else
    {
      const float desat = desat_v2(tb, a, norm);
      norm = curve_out(tb, a, norm, a.spline.y[0]);
#pragma unroll
      for(int c = 0; c < 3; c++) ratios[c] = fmaxf(ratios[c] + (1.0f - ratios[c]) * (1.0f - desat), 0.0f);
      if(a.version == 2) norm /= fmaxf(pixel_norm(a, ratios, a.preserve_color), NORM_MIN);
#pragma unroll
      for(int c = 0; c < 4; c++) res[c] = ratios[c] * norm;
      const float max_pix = fmaxf(fmaxf(res[0], res[1]), res[2]);
      if(max_pix > 1.0f)
      {
#pragma unroll
        for(int c = 0; c < 4; c++)
        {
          ratios[c] = fmaxf(ratios[c] + (1.0f - max_pix), 0.0f);
          res[c] = ratios[c] * norm;
        }
      }
    }
  }
  if(a.copy_alpha) res[3] = p.w;
  __stcs(out + k, make_float4(res[0], res[1], res[2], res[3]));
}

void to_m34(m34 dst, const float src[3][4])
{
  memset(dst, 0, sizeof(m34));
  for(int i = 0; i < 3; i++)
    for(int j = 0; j < 3; j++) dst[i][j] = src[i][j];
}
} // namespace

using namespace b200;

static int check_fl(const b200_piece_t *piece, const void *in, void *out)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "filmicrgb: NULL argument");
  if(!piece->data || piece->data_size < sizeof(b200_filmicrgb_piece_t))
    return fail(B200_ERR_ARG, "filmicrgb: piece->data is not a b200_filmicrgb_piece_t");
  const b200_filmicrgb_data_t *d = &((const b200_filmicrgb_piece_t *)piece->data)->data;
  if(d->version < 0 || d->version > 9) return fail(B200_ERR_ARG, "filmicrgb: colour science %d", d->version);
  return B200_OK;
}

namespace b200
{
int filmic_reconstruct_dev(const b200_piece_t *piece, const b200_filmicrgb_data_t *d, const float *d_in, const float **d_use, cudaStream_t st);
int filmic_reconstruct_scales(const b200_piece_t *piece);
}

extern "C" int b200_filmicrgb_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = check_fl(piece, d_in, d_out);
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  const b200_filmicrgb_piece_t *fp = (const b200_filmicrgb_piece_t *)piece->data;
  const b200_filmicrgb_data_t *d = &fp->data;
  filmic_args_t a;
  memset(&a, 0, sizeof(a));
  m34 wi, wo, ei, eo;
  to_m34(wi, fp->work_profile.matrix_in);
  to_m34(wo, fp->work_profile.matrix_out);
  if(fp->has_export_profile)
  {
    to_m34(ei, fp->export_profile.matrix_in);
    to_m34(eo, fp->export_profile.matrix_out);
  }
  prepare(&a, d->version, wi, wo, fp->has_export_profile ? &ei : nullptr, fp->has_export_profile ? &eo : nullptr);
  a.spline = d->spline;
  a.grey_source = d->grey_source;
  a.black_source = d->black_source;
  a.dynamic_range = d->dynamic_range;
  a.output_power = d->output_power;
  a.agx_beta_hue = d->agx_beta_hue;
  a.white = powf(d->spline.y[4], d->output_power); // :2840-2841
  a.black = powf(d->spline.y[0], d->output_power);
  a.copy_alpha = (piece->mask_display & B200_DISPLAY_MASK) ? 1 : 0;
  const size_t npx = (size_t)piece->roi_out.width * piece->roi_out.height;
  if(!npx) return B200_OK;
  if(!d->hl_deprecated)
  { // :2729-2838: edits that still carry a reconstruction threshold get their clipped highlights inpainted first
    const float *use = (const float *)d_in;
    if((rc = filmic_reconstruct_dev(piece, d, (const float *)d_in, &use, (cudaStream_t)stream))) return rc;
    d_in = use;
  }
  a.version = d->version;
  a.preserve_color = d->preserve_color;
  a.saturation = d->saturation;
  a.sigma_toe = d->sigma_toe;
  a.sigma_shoulder = d->sigma_shoulder;
  a.norm_min = d->grey_source * exp2f(d->dynamic_range * 0.f + d->black_source); // exp_tonemapping_v2(), :1054-1059, at 0 and 1
  a.norm_max = d->grey_source * exp2f(d->dynamic_range * 1.f + d->black_source);
  for(int c = 0; c < 3; c++) a.work_lum[c] = fp->work_profile.matrix_in[1][c];
  if(d->version >= 5)
    (a.use_output_profile ? filmic_agx_kernel<true> : filmic_agx_kernel<false>)<<<(unsigned)((npx + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      (const float4 *)d_in, (float4 *)d_out, npx, a);
  else
    filmic_legacy_kernel<<<(unsigned)((npx + 127) / 128), 128, 0, (cudaStream_t)stream>>>((const float4 *)d_in, (float4 *)d_out, npx, a);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}

extern "C" int b200_filmicrgb_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_fl(piece, in, out);
  if(rc) return rc;
  const size_t bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 16;
  return through_device(piece, in, bytes, out, bytes, false, b200_filmicrgb_process_dev);
}

// tiling_callback(), filmicrgb.c:2668-2704
extern "C" void b200_filmicrgb_tiling(const b200_piece_t *piece, b200_tiling_t *tiling)
{
  if(!piece || !tiling) return;
  tiling->factor = 2.0f; // reconstruction deprecated (every new edit): in + out, pointwise
  tiling->factor_cl = 2.0f;
  tiling->maxbuf = 1.0f;
  tiling->maxbuf_cl = 1.0f;
  tiling->overhead = 0;
  tiling->overlap = 0;
  tiling->xalign = 1;
  tiling->yalign = 1;
  // the data block is the first member of b200_filmicrgb_piece_t and the only one read here: the module adapter passes
  // the reference's own piece->data (sizeof(dt_iop_filmicrgb_data_t)), library callers the flattened piece
  static_assert(offsetof(b200_filmicrgb_piece_t, data) == 0, "data must lead b200_filmicrgb_piece_t");
  if(!piece->data || piece->data_size < sizeof(b200_filmicrgb_data_t)) return;
  const b200_filmicrgb_data_t *d = (const b200_filmicrgb_data_t *)piece->data;
  if(d->hl_deprecated) return;
  tiling->factor = 9.0f; // in + out + 2 * tmp + 2 * LF + 2 * temp + ratios
  tiling->factor_cl = 9.0f;
  tiling->overlap = 1u << filmic_reconstruct_scales(piece);
}
