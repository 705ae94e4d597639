// Single-precision libm for the device, bit-compatible with what the reference's CPU path calls:
// glibc 2.39 sysdeps/ieee754/flt-32/{e_powf,e_log2f,e_logf,e_expf,e_exp2f}.c in the FMA build that
// glibc's ifunc selects on every FMA-capable x86-64 (double-precision core, 16-entry log tables,
// 32-entry exp2 table; each a*b+c below is one fused operation there and here).
// Reference call sites: colorprofiles/iop_profile.h:561 (powf), iop/denoiseprofile.c:938,1020,1041,1086,
// iop/filmicrgb.c:1050,1089-1132,2124,2143, pixel/locallaplacian.c:323 (expf).
// CUDA's own powf/log2f/expf are NOT used: they are up to 2-4 ulp off and would break the
// <= 1 ulp contract.  tests/test_flt32_math.py pins these against the system libm on the GPU box.
//
// Tables live in global memory (L1/L2 resident, 16+16+16+32 doubles); kernels that evaluate many
// transcendentals per pixel copy them to shared memory and pass that pointer set instead.
#pragma once
#include <stdint.h>
#include <math_constants.h>

namespace f32m
{
struct tables_t
{
  const double *invc;    // 1/c of the 16 sub-intervals of [0x3f330000, 2*0x3f330000)
  const double *lnc;     // ln c      (__logf_data)
  const double *log2c;   // log2 c    (__log2f_data, __powf_log2_data with POWF_SCALE = 1)
  const uint64_t *exp2;  // bits(2^(i/32)) - (i << 47)   (__exp2f_data)
};

__device__ const uint64_t g_exp2[32] = {
  0x3ff0000000000000ULL, 0x3fefd9b0d3158574ULL, 0x3fefb5586cf9890fULL, 0x3fef9301d0125b51ULL,
  0x3fef72b83c7d517bULL, 0x3fef54873168b9aaULL, 0x3fef387a6e756238ULL, 0x3fef1e9df51fdee1ULL,
  0x3fef06fe0a31b715ULL, 0x3feef1a7373aa9cbULL, 0x3feedea64c123422ULL, 0x3feece086061892dULL,
  0x3feebfdad5362a27ULL, 0x3feeb42b569d4f82ULL, 0x3feeab07dd485429ULL, 0x3feea47eb03a5585ULL,
  0x3feea09e667f3bcdULL, 0x3fee9f75e8ec5f74ULL, 0x3feea11473eb0187ULL, 0x3feea589994cce13ULL,
  0x3feeace5422aa0dbULL, 0x3feeb737b0cdc5e5ULL, 0x3feec49182a3f090ULL, 0x3feed503b23e255dULL,
  0x3feee89f995ad3adULL, 0x3feeff76f2fb5e47ULL, 0x3fef199bdd85529cULL, 0x3fef3720dcef9069ULL,
  0x3fef5818dcfba487ULL, 0x3fef7c97337b9b5fULL, 0x3fefa4afa2a490daULL, 0x3fefd0765b6e4540ULL
};
__device__ const double g_invc[16] = {
  0x1.661ec79f8f3bep+0, 0x1.571ed4aaf883dp+0, 0x1.49539f0f010b0p+0, 0x1.3c995b0b80385p+0,
  0x1.30d190c8864a5p+0, 0x1.25e227b0b8ea0p+0, 0x1.1bb4a4a1a343fp+0, 0x1.12358f08ae5bap+0,
  0x1.0953f419900a7p+0, 0x1.0000000000000p+0, 0x1.e608cfd9a47acp-1, 0x1.ca4b31f026aa0p-1,
  0x1.b2036576afce6p-1, 0x1.9c2d163a1aa2dp-1, 0x1.886e6037841edp-1, 0x1.767dcf5534862p-1
};
__device__ const double g_lnc[16] = {
  -0x1.57bf7808caadep-2, -0x1.2bef0a7c06ddbp-2, -0x1.01eae7f513a67p-2, -0x1.b31d8a68224e9p-3,
  -0x1.6574f0ac07758p-3, -0x1.1aa2bc79c8100p-3, -0x1.a4e76ce8c0e5ep-4, -0x1.1973c5a611cccp-4,
  -0x1.252f438e10c1ep-5, 0x0.0p+0,              0x1.aa5aa5df25984p-5,  0x1.c5e53aa362eb4p-4,
  0x1.526e57720db08p-3,  0x1.bc2860d224770p-3,  0x1.1058bc8a07ee1p-2,  0x1.4043057b6ee09p-2
};
__device__ const double g_log2c[16] = {
  -0x1.efec65b963019p-2, -0x1.b0b6832d4fca4p-2, -0x1.7418b0a1fb77bp-2, -0x1.39de91a6dcf7bp-2,
  -0x1.01d9bf3f2b631p-2, -0x1.97c1d1b3b7af0p-3, -0x1.2f9e393af3c9fp-3, -0x1.960cbbf788d5cp-4,
  -0x1.a6f9db6475fcep-5, 0x0.0p+0,              0x1.338ca9f24f53dp-4,  0x1.476a9543891bap-3,
  0x1.e840b4ac4e4d2p-3,  0x1.40645f0c6651cp-2,  0x1.88e9c2c1b9ff8p-2,  0x1.ce0a44eb17bccp-2
};

__device__ __forceinline__ tables_t global_tables()
{
  tables_t t;
  t.invc = g_invc;
  t.lnc = g_lnc;
  t.log2c = g_log2c;
  t.exp2 = g_exp2;
  return t;
}
// 80 doubles = 640 bytes of shared memory; call from all threads of the block, then __syncthreads()
constexpr int SMEM_DOUBLES = 16 + 16 + 16 + 32;
__device__ __forceinline__ tables_t stage_tables(double *smem, int tid, int nthreads)
{
  for(int k = tid; k < 16; k += nthreads)
  {
    smem[k] = g_invc[k];
    smem[16 + k] = g_lnc[k];
    smem[32 + k] = g_log2c[k];
  }
  uint64_t *e = reinterpret_cast<uint64_t *>(smem + 48);
  for(int k = tid; k < 32; k += nthreads) e[k] = g_exp2[k];
  tables_t t;
  t.invc = smem;
  t.lnc = smem + 16;
  t.log2c = smem + 32;
  t.exp2 = e;
  return t;
}

constexpr double EXP2_C0 = 0x1.c6af84b912394p-5, EXP2_C1 = 0x1.ebfce50fac4f3p-3, EXP2_C2 = 0x1.62e42ff0c52d6p-1;
constexpr double EXP2_SHIFT_SCALED = 0x1.8p+47, EXP_SHIFT = 0x1.8p+52, INVLN2_SCALED = 0x1.71547652b82fep+5;
constexpr double EXP_C0S = 0x1.c6af84b912394p-20, EXP_C1S = 0x1.ebfce50fac4f3p-13, EXP_C2S = 0x1.62e42ff0c52d6p-6;
constexpr double LN2 = 0x1.62e42fefa39efp-1;
constexpr double LOGF_A0 = -0x1.00ea348b88334p-2, LOGF_A1 = 0x1.5575b0be00b6ap-2, LOGF_A2 = -0x1.ffffef20a4123p-2;
constexpr double LOG2F_A0 = -0x1.712b6f70a7e4dp-2, LOG2F_A1 = 0x1.ecabf496832e0p-2, LOG2F_A2 = -0x1.715479ffae3dep-1,
                 LOG2F_A3 = 0x1.715475f35c8b8p+0;
constexpr double POWF_A0 = 0x1.27616c9496e0bp-2, POWF_A1 = -0x1.71969a075c67ap-2, POWF_A2 = 0x1.ec70a6ca7baddp-2,
                 POWF_A3 = -0x1.7154748bef6c8p-1, POWF_A4 = 0x1.71547652ab82bp+0;
constexpr uint32_t OFF = 0x3f330000u;

__device__ __forceinline__ uint32_t top12(float x) { return __float_as_uint(x) >> 20; }

// 2^(k/32) * poly(r): the tail shared by expf, exp2f and powf (exp2_inline, e_powf.c)
__device__ __forceinline__ double exp2_tail(const tables_t &tb, uint64_t ki, uint64_t ski, double r, double c0, double c1, double c2)
{
  uint64_t t = tb.exp2[ki & 31];
  t += ski << (52 - 5);
  const double s = __longlong_as_double((long long)t);
  const double z = fma(c0, r, c1);
  const double r2 = r * r;
  double y = fma(c2, r, 1.0);
  y = fma(z, r2, y);
  return y * s;
}

// e_expf.c
__device__ __forceinline__ float expf_(const tables_t &tb, float x)
{
  const uint32_t abstop = top12(x) & 0x7ff;
  if(abstop >= (0x42b00000u >> 20)) // |x| >= 88 or NaN
  {
    if(__float_as_uint(x) == 0xff800000u) return 0.0f;
    if(abstop >= (0x7f800000u >> 20)) return x + x;
    if(x > 0x1.62e42ep6f) return CUDART_INF_F;
    if(x < -0x1.9fe368p6f) return 0.0f;
  }
  const double z = INVLN2_SCALED * (double)x;
  double kd = z + EXP_SHIFT;
  const uint64_t ki = (uint64_t)__double_as_longlong(kd);
  kd -= EXP_SHIFT;
  return (float)exp2_tail(tb, ki, ki, z - kd, EXP_C0S, EXP_C1S, EXP_C2S);
}

// e_exp2f.c
__device__ __forceinline__ float exp2f_(const tables_t &tb, float x)
{
  const uint32_t abstop = top12(x) & 0x7ff;
  if(abstop >= (0x43000000u >> 20)) // |x| >= 128 or NaN
  {
    if(__float_as_uint(x) == 0xff800000u) return 0.0f;
    if(abstop >= (0x7f800000u >> 20)) return x + x;
    if(x > 0.0f) return CUDART_INF_F;
    if(x <= -150.0f) return 0.0f;
  }
  const double xd = (double)x;
  double kd = xd + EXP2_SHIFT_SCALED;
  const uint64_t ki = (uint64_t)__double_as_longlong(kd);
  kd -= EXP2_SHIFT_SCALED;
  return (float)exp2_tail(tb, ki, ki, xd - kd, EXP2_C0, EXP2_C1, EXP2_C2);
}

// x < 0x1p-126, inf or nan: what e_logf.c / e_log2f.c return before the main path; `ix` is
// rewritten for subnormals.  Returns true when `out` is final.
__device__ __forceinline__ bool log_special(float x, uint32_t &ix, float &out)
{
  if(ix * 2 == 0)
  {
    out = -CUDART_INF_F;
    return true;
  }
  if(ix == 0x7f800000u)
  {
    out = x;
    return true;
  }
  if((ix & 0x80000000u) || ix * 2 >= 0xff000000u)
  {
    out = CUDART_NAN_F;
    return true;
  }
  ix = __float_as_uint(x * 0x1p23f); // flushed to zero under FTZ exactly as DAZ does on the CPU
  ix -= 23u << 23;
  return false;
}

// e_logf.c
__device__ __forceinline__ float logf_(const tables_t &tb, float x)
{
  uint32_t ix = __float_as_uint(x);
  if(ix == 0x3f800000u) return 0.0f;
  if(ix - 0x00800000u >= 0x7f800000u - 0x00800000u)
  {
    float out;
    if(log_special(x, ix, out)) return out;
  }
  const uint32_t tmp = ix - OFF;
  const int i = (tmp >> (23 - 4)) & 15;
  const int k = (int32_t)tmp >> 23;
  const uint32_t iz = ix - (tmp & (0x1ffu << 23));
  const double z = (double)__uint_as_float(iz);
  const double r = fma(z, tb.invc[i], -1.0);
  const double y0 = fma((double)k, LN2, tb.lnc[i]);
  const double r2 = r * r;
  double y = fma(LOGF_A1, r, LOGF_A2);
  y = fma(LOGF_A0, r2, y);
  y = fma(y, r2, y0 + r);
  return (float)y;
}

// e_log2f.c
__device__ __forceinline__ float log2f_(const tables_t &tb, float x)
{
  uint32_t ix = __float_as_uint(x);
  if(ix == 0x3f800000u) return 0.0f;
  if(ix - 0x00800000u >= 0x7f800000u - 0x00800000u)
  {
    float out;
    if(log_special(x, ix, out)) return out;
  }
  const uint32_t tmp = ix - OFF;
  const int i = (tmp >> (23 - 4)) & 15;
  const uint32_t iz = ix - (tmp & 0xff800000u);
  const int k = (int32_t)tmp >> 23;
  const double z = (double)__uint_as_float(iz);
  const double r = fma(z, tb.invc[i], -1.0);
  const double y0 = tb.log2c[i] + (double)k;
  const double r2 = r * r;
  double y = fma(LOG2F_A1, r, LOG2F_A2);
  y = fma(LOG2F_A0, r2, y);
  const double p = fma(LOG2F_A3, r, y0);
  y = fma(y, r2, p);
  return (float)y;
}

// checkint(): 0 = not an integer, 1 = odd, 2 = even (e_powf.c)
__device__ __forceinline__ int checkint(uint32_t iy)
{
  const int e = iy >> 23 & 0xff;
  if(e < 0x7f) return 0;
  if(e > 0x7f + 23) return 2;
  if(iy & ((1u << (0x7f + 23 - e)) - 1)) return 0;
  if(iy & (1u << (0x7f + 23 - e))) return 1;
  return 2;
}
__device__ __forceinline__ bool zeroinfnan(uint32_t ix) { return 2 * ix - 1 >= 2u * 0x7f800000u - 1; }

// the rare inputs of powf: x < 0x1p-126, x inf/nan, y zero/inf/nan.  `done` says `out` is final;
// otherwise ix / sign_bias are prepared for the main path.  Everything travels by value: the call
// is out of line, and an argument passed by reference would put ix and sign_bias on the stack, with
// a store and three loads of local memory on every powf_ call, special or not.
struct powf_pre_t
{
  float out;
  uint32_t ix, sign_bias;
  bool done;
};
static __device__ __noinline__ powf_pre_t powf_special(float x, float y, uint32_t ix, uint32_t iy)
{
  powf_pre_t r = { 0.0f, ix, 0u, true };
  if(zeroinfnan(iy))
  {
    if(2 * iy == 0 || ix == 0x3f800000u) r.out = 1.0f;
    else if(2 * ix > 2u * 0x7f800000u || 2 * iy > 2u * 0x7f800000u) r.out = x + y;
    else if(2 * ix == 2 * 0x3f800000u) r.out = 1.0f;
    else if((2 * ix < 2 * 0x3f800000u) == !(iy & 0x80000000u)) r.out = 0.0f;
    else r.out = y * y;
    return r;
  }
  if(zeroinfnan(ix))
  {
    float x2 = x * x;
    bool neg = false;
    if((ix & 0x80000000u) && checkint(iy) == 1)
    {
      x2 = -x2;
      neg = true;
    }
    if(2 * ix == 0 && (iy & 0x80000000u)) r.out = neg ? -CUDART_INF_F : CUDART_INF_F;
    else r.out = (iy & 0x80000000u) ? 1.0f / x2 : x2;
    return r;
  }
  if(ix & 0x80000000u)
  {
    const int yint = checkint(iy);
    if(yint == 0)
    {
      r.out = CUDART_NAN_F;
      return r;
    }
    if(yint == 1) r.sign_bias = 1u << (5 + 11);
    r.ix &= 0x7fffffffu;
  }
  if(r.ix < 0x00800000u)
  {
    r.ix = __float_as_uint(x * 0x1p23f);
    r.ix &= 0x7fffffffu;
    r.ix -= 23u << 23;
  }
  r.done = false;
  return r;
}

// e_powf.c
__device__ __forceinline__ float powf_(const tables_t &tb, float x, float y)
{
  uint32_t sign_bias = 0;
  uint32_t ix = __float_as_uint(x);
  const uint32_t iy = __float_as_uint(y);
  if(ix - 0x00800000u >= 0x7f800000u - 0x00800000u || zeroinfnan(iy))
  {
    const powf_pre_t pre = powf_special(x, y, ix, iy);
    if(pre.done) return pre.out;
    ix = pre.ix;
    sign_bias = pre.sign_bias;
  }
  // log2_inline
  const uint32_t tmp = ix - OFF;
  const int i = (tmp >> (23 - 4)) & 15;
  const uint32_t top = tmp & 0xff800000u;
  const uint32_t iz = ix - top;
  const int k = (int32_t)top >> 23;
  const double z = (double)__uint_as_float(iz);
  const double r = fma(z, tb.invc[i], -1.0);
  const double y0 = tb.log2c[i] + (double)k;
  const double r2 = r * r;
  double yy = fma(POWF_A0, r, POWF_A1);
  const double p = fma(POWF_A2, r, POWF_A3);
  const double r4 = r2 * r2;
  double q = fma(POWF_A4, r, y0);
  q = fma(p, r2, q);
  yy = fma(yy, r4, q);
  const double ylogx = (double)y * yy;
  if((((uint64_t)__double_as_longlong(ylogx)) >> 47 & 0xffff) >= (0x405f800000000000ULL >> 47)) // |y log2 x| >= 126
  {
    if(ylogx > 0x1.fffffffd1d571p+6) return sign_bias ? -CUDART_INF_F : CUDART_INF_F;
    if(ylogx <= -150.0) return sign_bias ? -0.0f : 0.0f;
  }
  // exp2_inline
  double kd = ylogx + EXP2_SHIFT_SCALED;
  const uint64_t ki = (uint64_t)__double_as_longlong(kd);
  kd -= EXP2_SHIFT_SCALED;
  return (float)exp2_tail(tb, ki, ki + sign_bias, ylogx - kd, EXP2_C0, EXP2_C1, EXP2_C2);
}
// ---- s_sinf.c / s_cosf.c / sincosf.h (reached through iop/noise_generator.h:93-96 with arguments 2*pi*u) ------
// |x| < 120: the pi/4 polynomial and the single multiply-subtract reduction.  Larger arguments need glibc's
// table-driven reduction, which nothing on this path calls: NaN, so a misuse shows.
constexpr double SC_HPI_INV = 0x1.45F306DC9C883p+23, SC_HPI = 0x1.921FB54442D18p0;
constexpr double SC_C1 = -0x1.ffffffd0c621cp-2, SC_C2 = 0x1.55553e1068f19p-5, SC_C3 = -0x1.6c087e89a359dp-10, SC_C4 = 0x1.99343027bf8c3p-16;
constexpr double SC_S1 = -0x1.555545995a603p-3, SC_S2 = 0x1.1107605230bc4p-7, SC_S3 = -0x1.994eb3774cf24p-13;

__device__ __forceinline__ uint32_t abstop12(float x) { return (__float_as_uint(x) >> 20) & 0x7ffu; }
// sinf_poly(): sine polynomial for even n, cosine for odd; neg selects __sincosf_table[1]
__device__ __forceinline__ float sinf_poly(double x, double x2, bool neg, int n)
{
  if((n & 1) == 0)
  {
    const double x3 = x * x2;
    const double s1 = fma(x2, SC_S3, SC_S2);
    const double x7 = x3 * x2;
    const double s = fma(x3, SC_S1, x);
    return (float)fma(x7, s1, s);
  }
  const double sg = neg ? -1.0 : 1.0;
  const double x4 = x2 * x2;
  const double c2 = fma(x2, sg * SC_C4, sg * SC_C3);
  const double c1 = fma(x2, sg * SC_C1, sg);
  const double x6 = x4 * x2;
  const double c = fma(x4, sg * SC_C2, c1);
  return (float)fma(x6, c2, c);
}
template <bool COS> __device__ __forceinline__ float sincosf_(float y)
{
  double x = (double)y;
  if(abstop12(y) < abstop12(0x1.921FB6p-1f))
  {
    if(abstop12(y) < abstop12(0x1p-12f)) return COS ? 1.0f : y;
    return sinf_poly(x, x * x, false, COS ? 1 : 0);
  }
  if(abstop12(y) < abstop12(120.0f))
  {
    const double r = x * SC_HPI_INV;
    const int n = (__double2int_rz(r) + 0x800000) >> 24;
    x = fma(-(double)n, SC_HPI, x);
    const double s = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
    return sinf_poly(x * s, x * x, (n & 2) != 0, COS ? (n ^ 1) : n);
  }
  return CUDART_NAN_F;
}
__device__ __forceinline__ float sinf_(float y) { return sincosf_<false>(y); }
__device__ __forceinline__ float cosf_(float y) { return sincosf_<true>(y); }

// ---- atanf, atan2f, hypotf: glibc 2.39 sysdeps/ieee754/flt-32/{s_atanf,e_atan2f,e_hypotf}.c ----------------------------------------
// The first two are the fdlibm float routines: reduction to four breakpoints, an 11-term odd polynomial split in two, head / tail
// constants of the breakpoints; no FMA build exists, every operation is a float operation in source order (the library is compiled
// with --fmad=false).  hypotf is one square root of the exact double sum of the squares.  What the reference calls them for:
// dt_Lab_2_LCH and dt_JzAzBz_2_JzCzhz (common/colorspaces_inline_conversions.h:594-606, :775-781).
__device__ __forceinline__ float atan_hi(int id) { return id == 0 ? 4.6364760399e-01f : (id == 1 ? 7.8539812565e-01f : (id == 2 ? 9.8279368877e-01f : 1.5707962513e+00f)); }
__device__ __forceinline__ float atan_lo(int id) { return id == 0 ? 5.0121582440e-09f : (id == 1 ? 3.7748947079e-08f : (id == 2 ? 3.4473217170e-08f : 7.5497894159e-08f)); }
__device__ __forceinline__ float atanf_(float x)
{
  const int hx = (int)__float_as_uint(x), ix = hx & 0x7fffffff;
  int id;
  if(ix >= 0x4c000000)
  { // |x| >= 2^25
    if(ix > 0x7f800000) return x + x;
    return hx > 0 ? atan_hi(3) + atan_lo(3) : -atan_hi(3) - atan_lo(3);
  }
  if(ix < 0x3ee00000)
  { // |x| < 0.4375
    if(ix < 0x31000000) return x; // |x| < 2^-29
    id = -1;
  }
  else
  {
    x = fabsf(x);
    if(ix < 0x3f980000)
    {
      if(ix < 0x3f300000)
      {
        id = 0;
        x = (2.0f * x - 1.0f) / (2.0f + x);
      }
      else
      {
        id = 1;
        x = (x - 1.0f) / (x + 1.0f);
      }
    }
    else if(ix < 0x401c0000)
    {
      id = 2;
      x = (x - 1.5f) / (1.0f + 1.5f * x);
    }
    else
    {
      id = 3;
      x = -1.0f / x;
    }
  }
  const float z = x * x, w = z * z;
  const float s1 = z * (3.3333334327e-01f + w * (1.4285714924e-01f + w * (9.0908870101e-02f + w * (6.6610731184e-02f + w * (4.9768779427e-02f + w * 1.6285819933e-02f)))));
  const float s2 = w * (-2.0000000298e-01f + w * (-1.1111110449e-01f + w * (-7.6918758452e-02f + w * (-5.8335702866e-02f + w * -3.6531571299e-02f))));
  if(id < 0) return x - x * (s1 + s2);
  const float r = atan_hi(id) - ((x * (s1 + s2) - atan_lo(id)) - x);
  return hx < 0 ? -r : r;
}
__device__ __forceinline__ float atan2f_(float y, float x)
{
  const float tiny = 1.0e-30f, pi_o_4 = 7.8539818525e-01f, pi_o_2 = 1.5707963705e+00f, pi = 3.1415927410e+00f, pi_lo = -8.7422776573e-08f;
  const int hx = (int)__float_as_uint(x), ix = hx & 0x7fffffff, hy = (int)__float_as_uint(y), iy = hy & 0x7fffffff;
  if(ix > 0x7f800000 || iy > 0x7f800000) return x + y;
  if(hx == 0x3f800000) return atanf_(y);
  const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2); // 2 * sign(x) + sign(y)
  if(iy == 0) return m < 2 ? y : (m == 2 ? pi + tiny : -pi - tiny);
  if(ix == 0) return hy < 0 ? -pi_o_2 - tiny : pi_o_2 + tiny;
  if(ix == 0x7f800000)
  {
    if(iy == 0x7f800000) return m == 0 ? pi_o_4 + tiny : (m == 1 ? -pi_o_4 - tiny : (m == 2 ? 3.0f * pi_o_4 + tiny : -3.0f * pi_o_4 - tiny));
    return m == 0 ? 0.0f : (m == 1 ? -0.0f : (m == 2 ? pi + tiny : -pi - tiny));
  }
  if(iy == 0x7f800000) return hy < 0 ? -pi_o_2 - tiny : pi_o_2 + tiny;
  const int k = (iy - ix) >> 23;
  float z;
  if(k > 60)
    z = pi_o_2 + 0.5f * pi_lo;
  else if(hx < 0 && k < -60)
    z = 0.0f;
  else
    z = atanf_(fabsf(y / x));
  if(m == 0) return z;
  if(m == 1) return __uint_as_float(__float_as_uint(z) ^ 0x80000000u);
  if(m == 2) return pi - (z - pi_lo);
  return (z - pi_lo) - pi;
}
__device__ __forceinline__ float hypotf_(float x, float y)
{
  const uint32_t ax = __float_as_uint(x) & 0x7fffffffu, ay = __float_as_uint(y) & 0x7fffffffu;
  if(ax >= 0x7f800000u || ay >= 0x7f800000u) return (ax == 0x7f800000u || ay == 0x7f800000u) ? __int_as_float(0x7f800000) : x + y;
  return (float)sqrt((double)x * (double)x + (double)y * (double)y);
}
} // namespace f32m
