/* CPU restatement of colour balance rgb's process().  TEST INFRASTRUCTURE ONLY.
 *
 * Follows /root/reference/src/iop/colorbalancergb.c process() :585-927, opacity_masks :509-536, soft_clip :538-544, lookup_gamut
 * :547-581; common/colorspaces_inline_conversions.h (xyY :119-139, JzAzBz :726-891, LMS / Filmlight RGB / Yrg :940-1073, darktable UCS
 * :1261-1466); system/simd.h dt_mat3x4_mul_vec4 :189-197, dt_simd_max_zero :108-114; math/matrices.h dt_colormatrix_mul :167-179;
 * math/math.h scalar_product :185-195 (evaluated as 0 + ((p0 + p2) + p1)), dt_fast_hypotf :246-249.  MIN / MAX are the reference's
 * ternaries.  glibc's powf, expf, atan2f, sinf, cosf: flt32_math.h.  Pinned bit for bit against those lines cut verbatim
 * (oracle/colorbalancergb.mk). */
#include "oracle_common.h"
#include "b200iop.h"
#include "flt32_math.h"
#include <float.h>

#define CB_MAX(a, b) (((a) > (b)) ? (a) : (b))
#define CB_MIN(a, b) (((a) < (b)) ? (a) : (b))
#define CB_PI 3.14159265358979324f
#define LUT_ELEM B200_COLORBALANCE_LUT_ELEM

static const float XYZ_D50_to_D65_CAT16[3][3] = { { 9.89466254e-01f, -4.00304626e-02f, 4.40530317e-02f },
                                                  { -5.40518733e-03f, 1.00666069e+00f, -1.75551955e-03f },
                                                  { -4.03920992e-04f, 1.50768030e-02f, 1.30210211e+00f } };
static const float XYZ_D65_to_D50_CAT16[3][3] = { { 1.01085433e+00f, 4.07086103e-02f, -3.41445825e-02f },
                                                  { 5.42814201e-03f, 9.93581926e-01f, 1.15592039e-03f },
                                                  { 2.50722468e-04f, -1.14918759e-02f, 7.67964947e-01f } };
static const float XYZ_D65_to_LMS_2006[3][3] = { { 0.257085f, 0.859943f, -0.031061f }, { -0.394427f, 1.175800f, 0.106423f },
                                                 { 0.064856f, -0.076250f, 0.559067f } };
static const float LMS_2006_to_XYZ_D65[3][3] = { { 1.80794659f, -1.29971660f, 0.34785879f }, { 0.61783960f, 0.39595453f, -0.04104687f },
                                                 { -0.12546960f, 0.20478038f, 1.74274183f } };
static const float filmlight_to_LMS[3][3] = { { 0.95f, 0.38f, 0.00f }, { 0.05f, 0.62f, 0.03f }, { 0.00f, 0.00f, 0.97f } };
static const float LMS_to_filmlight[3][3] = { { 1.0877193f, -0.66666667f, 0.02061856f }, { -0.0877193f, 1.66666667f, -0.05154639f },
                                              { 0.f, 0.f, 1.03092784f } };
static const float JZ_M[3][3] = { { 0.41478972f, 0.579999f, 0.0146480f }, { -0.2015100f, 1.120649f, 0.0531008f }, { -0.0166008f, 0.264800f, 0.6684799f } };
static const float JZ_A[3][3] = { { 0.5f, 0.5f, 0.0f }, { 3.524000f, -4.066708f, 0.542708f }, { 0.199076f, 1.096799f, -1.295875f } };
static const float JZ_AI[3][3] = { { 1.0f, 0.1386050432715393f, 0.0580473161561189f },
                                   { 1.0f, -0.1386050432715393f, -0.0580473161561189f },
                                   { 1.0f, -0.0960192420263190f, -0.8118918960560390f } };
static const float JZ_MI[3][3] = { { 1.9242264357876067f, -1.0047923125953657f, 0.0376514040306180f },
                                   { 0.3503167620949991f, 0.7264811939316552f, -0.0653844229480850f },
                                   { -0.0909828109828475f, -0.3127282905230739f, 1.5227665613052603f } };

/* dt_mat3x4_mul_vec4 over the transposed rows: out = row0 * in0; out = row1 * in1 + out; out = row2 * in2 + out */
static void mat3(const float M[3][3], const float in[3], float out[3])
{
  for(int r = 0; r < 3; r++)
  {
    float acc = M[r][0] * in[0];
    acc = M[r][1] * in[1] + acc;
    out[r] = M[r][2] * in[2] + acc;
  }
}
static void colormatrix_mul(float dst[3][3], const float m1[3][3], const float m2[3][3])
{
  for(int k = 0; k < 3; k++)
    for(int i = 0; i < 3; i++)
    {
      float sum = 0.0f;
      for(int j = 0; j < 3; j++) sum += m1[k][j] * m2[j][i];
      dst[k][i] = sum;
    }
}
static float sqf(float x) { return x * x; }
static float max_zero(float v) { return isfinite(v) ? CB_MAX(v, 0.0f) : 0.f; }
static float scalar3(const float o[3], const float v[3]) { return 0.f + ((o[0] * v[0] + o[2] * v[2]) + o[1] * v[1]); }

static void lms_to_yrg(const float LMS[3], float Yrg[3])
{
  const float Y = 0.68990272f * LMS[0] + 0.34832189f * LMS[1];
  const float a = LMS[0] + LMS[1] + LMS[2];
  const float inv_a = (a == 0.f) ? 0.f : 1.f / a;
  const float lms[3] = { LMS[0] * inv_a, LMS[1] * inv_a, LMS[2] * inv_a };
  float rgb[3];
  mat3(LMS_to_filmlight, lms, rgb);
  Yrg[0] = Y;
  Yrg[1] = rgb[0];
  Yrg[2] = rgb[1];
}
static void yrg_to_lms(const float Yrg[3], float LMS[3])
{
  const float rgb[3] = { Yrg[1], Yrg[2], 1.f - Yrg[1] - Yrg[2] };
  float lms[3];
  mat3(filmlight_to_LMS, rgb, lms);
  const float denom = 0.68990272f * lms[0] + 0.34832189f * lms[1];
  const float a = (denom == 0.f) ? 0.f : Yrg[0] / denom;
  for(int c = 0; c < 3; c++) LMS[c] = lms[c] * a;
}
static float soft_clip(float x, float soft, float hard)
{
  const float norm = hard - soft;
  return (x > soft) ? soft + (1.f - f32m_expf(-(x - soft) / norm)) * norm : x;
}
static float lookup_gamut(const float *lut, float x)
{
  const float x_test = (LUT_ELEM - 1) * (x + CB_PI) / (2.f * CB_PI);
  const float x_prev = floorf(x_test), x_next = ceilf(x_test);
  int xi = (int)x_prev;
  if(xi < 0) xi = LUT_ELEM - 1;
  else if(xi > LUT_ELEM - 1) xi = 0;
  int xii = (int)x_next;
  if(xii < 0) xii = LUT_ELEM - 1;
  else if(xii > LUT_ELEM - 1) xii = 0;
  float out = lut[xi];
  if(x_next != x_prev) out += (x_test - x_prev) * (lut[xii] - lut[xi]) / (x_next - x_prev);
  return out;
}

typedef struct
{
  float in_m[3][3], out_m[3][3], L_white, rot[2][2];
} cb_plan_t;

static void jzazbz(float XYZ[3], const float op[3], const float *lut, const b200_colorbalancergb_data_t *d)
{
  const float b = 1.15f, g = 0.66f, c1 = 0.8359375f, c2 = 18.8515625f, c3 = 18.6875f, n = 0.159301758f, p = 134.034375f, dd = -0.56f;
  const float d0 = 1.6295499532821566e-11f, n_inv = 1.0f / 0.159301758f, p_inv = 1.0f / 134.034375f;
  const float Xp[3] = { b * XYZ[0] - (b - 1.0f) * XYZ[2], g * XYZ[1] - (g - 1.0f) * XYZ[0], XYZ[2] };
  float LMS[3], Jab[3];
  mat3(JZ_M, Xp, LMS);
  for(int i = 0; i < 3; i++)
  {
    LMS[i] = f32m_powf(fmaxf(LMS[i] / 10000.f, 0.0f), n);
    LMS[i] = f32m_powf((c1 + c2 * LMS[i]) / (1.0f + c3 * LMS[i]), p);
  }
  mat3(JZ_A, LMS, Jab);
  Jab[0] = fmaxf(((1.0f + dd) * Jab[0]) / (1.0f + dd * Jab[0]) - d0, 0.f);
  float JC[2] = { Jab[0], sqrtf(Jab[1] * Jab[1] + Jab[2] * Jab[2]) };
  const float h = f32m_atan2f(Jab[2], Jab[1]);
  const float inv_chroma = (JC[1] > 0.f) ? 1.f / JC[1] : 0.f;
  const float cos_H = Jab[1] * inv_chroma, sin_H = Jab[2] * inv_chroma;
  const float T = f32m_atan2f(JC[1], JC[0]);
  const float sin_T = f32m_sinf(T), cos_T = f32m_cosf(T);
  const float boosts[2] = { 1.f + d->brilliance_global + scalar3(op, d->brilliance), d->saturation_global + scalar3(op, d->saturation) };
  float SO[2];
  SO[0] = JC[0] * cos_T + JC[1] * sin_T;
  SO[1] = SO[0] * CB_MIN(CB_MAX(T * boosts[1], -T), CB_PI / 2.f - T);
  SO[0] = CB_MAX(SO[0] * boosts[0], 0.f);
  JC[0] = CB_MAX(SO[0] * cos_T + SO[1] * -sin_T, 0.f);
  JC[1] = CB_MAX(SO[0] * sin_T + SO[1] * cos_T, 0.f);
  const float out_max_sat_h = lookup_gamut(lut, h);
  const float sat = (JC[0] > 0.f) ? soft_clip(JC[1] / JC[0], 0.8f * out_max_sat_h, out_max_sat_h) : out_max_sat_h;
  const float max_C_at_sat = JC[0] * sat;
  const float max_J_at_sat = (sat > 0.f) ? JC[1] / sat : JC[0];
  JC[0] = (JC[0] + max_J_at_sat) / 2.f;
  JC[1] = (JC[1] + max_C_at_sat) / 2.f;
  float Iz = JC[0] + d0;
  Iz /= (1.f + dd - dd * Iz);
  Iz = CB_MAX(Iz, 0.f);
  const float IzAzBz[3] = { Iz, JC[1] * cos_H, JC[1] * sin_H };
  float test[3];
  mat3(JZ_AI, IzAzBz, test);
  float max_C = JC[1];
  for(int i = 0; i < 3; i++)
    if(test[i] < 0.f) max_C = CB_MIN(-Iz / (JZ_AI[i][1] * cos_H + JZ_AI[i][2] * sin_H), max_C);
  /* dt_JzAzBz_2_XYZ_simd */
  float I[3] = { JC[0] + d0, max_C * cos_H, max_C * sin_H };
  I[0] = fmaxf(I[0] / (1.0f + dd - dd * I[0]), 0.f);
  mat3(JZ_AI, I, LMS);
  for(int i = 0; i < 3; i++)
  {
    LMS[i] = f32m_powf(fmaxf(LMS[i], 0.0f), p_inv);
    LMS[i] = 10000.f * f32m_powf(fmaxf((c1 - LMS[i]) / (c3 * LMS[i] - c2), 0.0f), n_inv);
  }
  float X[3];
  mat3(JZ_MI, LMS, X);
  XYZ[0] = (X[0] + (b - 1.0f) * X[2]) / b;
  XYZ[1] = (X[1] + (g - 1.0f) * ((X[0] + (b - 1.0f) * X[2]) / b)) / g;
  XYZ[2] = X[2];
}

static void dt_ucs(float XYZ[3], const float op[3], const float *lut, const b200_colorbalancergb_data_t *d, const float L_white)
{
  const float sum = XYZ[0] + XYZ[1] + XYZ[2];
  const float xyY[3] = { XYZ[0] / sum, XYZ[1] / sum, XYZ[1] };
  /* xyY_to_dt_UCS_UV */
  static const float xf[3] = { -0.783941002840055f, 0.745273540913283f, 0.318707282433486f };
  static const float yf[3] = { 0.277512987809202f, -0.205375866083878f, 2.16743692732158f };
  static const float of[3] = { 0.153836578598858f, -0.165478376301988f, 0.291320554395942f };
  static const float factors[2] = { 1.39656225667f, 1.4513954287f }, half_values[2] = { 1.49217352929f, 1.52488637914f };
  float UVD[3];
  for(int c = 0; c < 3; c++) UVD[c] = xf[c] * xyY[0] + yf[c] * xyY[1] + of[c];
  UVD[0] /= UVD[2];
  UVD[1] /= UVD[2];
  float UV_star[2];
  for(int c = 0; c < 2; c++) UV_star[c] = factors[c] * UVD[c] / (fabsf(UVD[c]) + half_values[c]);
  const float Up = -1.124983854323892f * UV_star[0] - 0.980483721769325f * UV_star[1];
  const float Vp = 1.86323315098672f * UV_star[0] + 1.971853092390862f * UV_star[1];
  /* Y_to_dt_UCS_L_star, dt_UCS_LUV_to_JCH */
  const float Y_hat = f32m_powf(xyY[2], 0.631651345306265f);
  const float L_star = 2.098883786377f * Y_hat / (Y_hat + 1.12426773749357f);
  const float M2 = Up * Up + Vp * Vp;
  float JCH[3] = { L_star / L_white, 15.932993652962535f * f32m_powf(L_star, 0.6523997524738018f) * f32m_powf(M2, 0.6007557017508491f) / L_white,
                   f32m_atan2f(Vp, Up) };
  float HCB[3] = { JCH[2], JCH[1], JCH[0] * (f32m_powf(JCH[1], 1.33654221029386f) + 1.f) };
  const float radius = sqrtf(HCB[1] * HCB[1] + HCB[2] * HCB[2]);
  const float sin_T = (radius > 0.f) ? HCB[1] / radius : 0.f;
  const float cos_T = (radius > 0.f) ? HCB[2] / radius : 0.f;
  const float P = CB_MAX(HCB[1], FLT_MIN);
  const float W = sin_T * HCB[1] + cos_T * HCB[2];
  float a = max_zero(1.f + d->saturation_global + scalar3(op, d->saturation));
  const float b = max_zero(1.f + d->brilliance_global + scalar3(op, d->brilliance));
  const float max_a = sqrtf(P * P + W * W) / P;
  a = soft_clip(a, 0.5f * max_a, max_a);
  const float P_prime = (a - 1.f) * P;
  const float W_prime = sqrtf(sqf(P) * (1.f - sqf(a)) + sqf(W)) * b;
  HCB[1] = CB_MAX(cos_T * P_prime + sin_T * W_prime, 0.f);
  HCB[2] = CB_MAX(-sin_T * P_prime + cos_T * W_prime, 0.f);
  JCH[0] = HCB[2] / (f32m_powf(HCB[1], 1.33654221029386f) + 1.f);
  JCH[1] = HCB[1];
  JCH[2] = HCB[0];
  const float max_colorfulness = lookup_gamut(lut, JCH[2]);
  const float max_chroma = 15.932993652962535f * f32m_powf(JCH[0] * L_white, 0.6523997524738018f) * f32m_powf(max_colorfulness, 0.6007557017508491f) / L_white;
  const float brightness = JCH[0] * (f32m_powf(max_chroma, 1.33654221029386f) + 1.f);
  const float S_boundary = (brightness > 0.f) ? max_chroma / brightness : 0.f;
  float HSB[3] = { HCB[0], (HCB[2] > 0.f) ? HCB[1] / HCB[2] : 0.f, HCB[2] };
  HSB[1] = soft_clip(HSB[1], 0.8f * S_boundary, S_boundary);
  const float chroma = HSB[1] * HSB[2];
  JCH[0] = HSB[2] / (f32m_powf(chroma, 1.33654221029386f) + 1.f);
  JCH[1] = chroma;
  JCH[2] = HSB[0];
  /* dt_UCS_JCH_to_xyY */
  const float L_s = JCH[0] * L_white;
  const float M = f32m_powf(JCH[1] * L_white / (15.932993652962535f * f32m_powf(L_s, 0.6523997524738018f)), 0.8322850678616855f);
  const float U_sp = M * f32m_cosf(JCH[2]), V_sp = M * f32m_sinf(JCH[2]);
  const float UVs[2] = { -5.037522385190711f * U_sp - 2.504856328185843f * V_sp, 4.760029407436461f * U_sp + 2.874012963239247f * V_sp };
  float UV[2];
  for(int c = 0; c < 2; c++) UV[c] = -half_values[c] * UVs[c] / (fabsf(UVs[c]) - factors[c]);
  static const float Uf[3] = { 0.167171472114775f, -0.150959086409163f, 0.940254742367256f };
  static const float Vf[3] = { 0.141299802443708f, -0.155185060382272f, 1.000000000000000f };
  static const float off[3] = { -0.00801531300850582f, -0.00843312433578007f, -0.0256325967652889f };
  float xyD[3];
  for(int c = 0; c < 3; c++) xyD[c] = Uf[c] * UV[0] + Vf[c] * UV[1] + off[c];
  const float x = xyD[0] / xyD[2], y = xyD[1] / xyD[2];
  const float Y = f32m_powf((1.12426773749357f * L_s / (2.098883786377f - L_s)), 1.5831518565279648f);
  const float y_over_x = Y / y;
  XYZ[0] = y_over_x * x;
  XYZ[1] = Y;
  XYZ[2] = y_over_x * (1.f - x - y);
}

/* process() on npixels RGBA floats.  Returns B200_ERR_UNSUPPORTED (output untouched) for the mask display. */
int orc_colorbalancergb(const float *in, float *out, size_t npixels, const b200_colorbalancergb_piece_t *pc)
{
  const b200_colorbalancergb_data_t *d = &pc->data;
  if(d->mask_display) return B200_ERR_UNSUPPORTED;
  orc_fp_fast_mode(); /* the pipe's threads run with FTZ|DAZ (darktable.c:877, common/dtpthread.c:54) */
  float work_in[3][3], work_out[3][3], tmp[3][3], in_m[3][3], out_m[3][3];
  for(int r = 0; r < 3; r++)
    for(int c = 0; c < 3; c++)
    {
      work_in[r][c] = pc->work_profile.matrix_in[r][c];
      work_out[r][c] = pc->work_profile.matrix_out[r][c];
    }
  colormatrix_mul(tmp, XYZ_D50_to_D65_CAT16, work_in);
  colormatrix_mul(in_m, XYZ_D65_to_LMS_2006, tmp);
  colormatrix_mul(out_m, work_out, XYZ_D65_to_D50_CAT16);
  const float Y_hat = f32m_powf(d->white_fulcrum, 0.631651345306265f);
  const float L_white = 2.098883786377f * Y_hat / (Y_hat + 1.12426773749357f);
  const float rot[2][2] = { { f32m_cosf(d->hue_angle), -f32m_sinf(d->hue_angle) }, { f32m_sinf(d->hue_angle), f32m_cosf(d->hue_angle) } };
  const float *lut = pc->gamut_LUT;
  for(size_t k = 0; k < npixels; k++)
  {
    const float *px = in + 4 * k;
    const float RGB_in[3] = { max_zero(px[0]), max_zero(px[1]), max_zero(px[2]) };
    float LMS[3], Yrg[3], RGB[3], XYZ[3], o[3];
    mat3(in_m, RGB_in, LMS);
    lms_to_yrg(LMS, Yrg);
    Yrg[0] = CB_MAX(Yrg[0], 0.f);
    /* opacity_masks */
    const float x = f32m_powf(Yrg[0], 0.4101205819200422f);
    const float x_offset = (x - d->mask_grey_fulcrum);
    const float x_offset_norm = x_offset / d->mask_grey_fulcrum;
    const float alpha = 1.f / (1.f + f32m_expf(x_offset_norm * d->shadows_weight));
    const float beta = 1.f / (1.f + f32m_expf(-x_offset_norm * d->highlights_weight));
    const float alpha_comp = 1.f - alpha, beta_comp = 1.f - beta;
    const float gamma = f32m_expf(-sqf(x_offset) * d->midtones_weight / 4.f) * sqf(alpha_comp) * sqf(beta_comp) * 8.f;
    const float op[3] = { alpha, gamma, beta }, comp[3] = { alpha_comp, 1.f - gamma, beta_comp };

    const float r_centered = Yrg[1] - 0.21902143f, g_centered = Yrg[2] - 0.54371398f;
    const float r_rotated = rot[0][0] * r_centered + rot[0][1] * g_centered;
    const float g_rotated = rot[1][0] * r_centered + rot[1][1] * g_centered;
    const float chroma_in = sqrtf(g_rotated * g_rotated + r_rotated * r_rotated);
    const float inv_chroma_in = (chroma_in > 0.f) ? 1.f / chroma_in : 0.f;
    const float cos_h = r_rotated * inv_chroma_in, sin_h = g_rotated * inv_chroma_in;
    const float chroma_boost = d->chroma_global + scalar3(op, d->chroma);
    const float vibrance = d->vibrance * (1.0f - f32m_powf(chroma_in, fabsf(d->vibrance)));
    const float chroma_factor = CB_MAX(1.f + chroma_boost + vibrance, 0.f);
    float chroma_out = chroma_in * chroma_factor;
    const float r_shifted = chroma_out * cos_h + 0.21902143f, g_shifted = chroma_out * sin_h + 0.54371398f;
    if(r_shifted < 0.f) chroma_out = CB_MIN(-0.21902143f / cos_h, chroma_out);
    if(g_shifted < 0.f) chroma_out = CB_MIN(-0.54371398f / sin_h, chroma_out);
    if(r_shifted + g_shifted > 1.f) chroma_out = CB_MIN((1.f - 0.21902143f - 0.54371398f) / (cos_h + sin_h), chroma_out);
    Yrg[1] = chroma_out * cos_h + 0.21902143f;
    Yrg[2] = chroma_out * sin_h + 0.54371398f;

    yrg_to_lms(Yrg, LMS);
    mat3(LMS_to_filmlight, LMS, RGB);
    for(int c = 0; c < 3; c++)
    {
      RGB[c] += d->global[c];
      RGB[c] *= comp[2] * (comp[0] + op[0] * d->shadows[c]) + op[2] * d->highlights[c];
    }
    for(int c = 0; c < 3; c++) RGB[c] = copysignf(f32m_powf(fabsf(RGB[c]) / d->white_fulcrum, d->midtones[c]) * d->white_fulcrum, RGB[c]);
    mat3(filmlight_to_LMS, RGB, LMS);
    lms_to_yrg(LMS, Yrg);
    Yrg[0] = f32m_powf(CB_MAX(Yrg[0] / d->white_fulcrum, 0.f), d->midtones_Y) * d->white_fulcrum;
    Yrg[0] = d->grey_fulcrum * f32m_powf(Yrg[0] / d->grey_fulcrum, d->contrast);
    yrg_to_lms(Yrg, LMS);
    mat3(LMS_2006_to_XYZ_D65, LMS, XYZ);
    if(d->saturation_formula == B200_COLORBALANCE_SATURATION_JZAZBZ) jzazbz(XYZ, op, lut, d);
    else dt_ucs(XYZ, op, lut, d, L_white);
    mat3(out_m, XYZ, o);
    float *po = out + 4 * k;
    for(int c = 0; c < 3; c++) po[c] = max_zero(o[c]);
    po[3] = px[3];
  }
  return 0;
}
