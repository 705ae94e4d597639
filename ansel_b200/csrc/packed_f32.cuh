// Pairs of floats: two lanes of the same IEEE operation, written once for both.  sm_90 has no packed FP32 instructions, so
// every pair is two scalar FADD / FMUL / FFMA, each round-to-nearest, flush-to-zero, identical to the scalar instruction the
// library's flags (--fmad=false -ftz=true) give.  The operations go through the _rn intrinsics, which ptxas never contracts
// into an FFMA whatever feeds them.
// tests/test_cpu_nlm_sass.py checks the built SASS: every FFMA of the NLM kernels is Markstein's division or part of an IEEE division.
// With B200_KERNELS_ON_CPU (tests/emul) the same names are plain scalar code.
#pragma once
#ifdef B200_KERNELS_ON_CPU
struct f2
{
  float x, y;
};
static inline f2 mk2(float x, float y) { return f2{ x, y }; }
static inline f2 add2(f2 a, f2 b) { return f2{ a.x + b.x, a.y + b.y }; }
static inline f2 sub2(f2 a, f2 b) { return f2{ a.x - b.x, a.y - b.y }; }
static inline f2 mul2(f2 a, f2 b) { return f2{ a.x * b.x, a.y * b.y }; }
static inline f2 fma2(f2 a, f2 b, f2 c) { return f2{ fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y) }; }
static inline f2 neg2(f2 a) { return f2{ -a.x, -a.y }; }
static inline float min_nan(float a, float b) { return (a != a) ? a : ((b != b) ? b : (a < b ? a : b)); }
static inline int __float2int_rz(float x) { return (int)x; } // cvttss2si: INT_MIN beyond the range, where the device saturates (same below -2^31)
#else
typedef float2 f2;
__device__ __forceinline__ f2 mk2(float x, float y) { return make_float2(x, y); }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f2 sub2(f2 a, f2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ f2 neg2(f2 a) { return make_float2(-a.x, -a.y); }
__device__ __forceinline__ float min_nan(float a, float b) // a NaN stays a NaN (fminf drops it)
{
  float r;
  asm("min.NaN.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
#endif

