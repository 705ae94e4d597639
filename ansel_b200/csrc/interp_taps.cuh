// The tap weights of the three interpolators of pixel/interpolation.c (_maketaps_bilinear :186, _maketaps_bicubic :219-228,
// _maketaps_mitchell :272-282), shared by the resampler of finalscale/initialscale (resample.cu) and lens correction (lens.cu).
// Each kernel's norm is 1 by construction (partition of unity), which both callers rely on.
#pragma once
#include <math.h>

// one tap weight at position t
static __host__ __device__ __forceinline__ float tap_weight(int interpolator, float t)
{
  const float a = fabsf(t);
  if(interpolator == B200_INTERPOLATION_BILINEAR) return 1.0f - a;
  if(interpolator == B200_INTERPOLATION_BICUBIC)
  {
    const float t2 = t * t, t5 = 5.0f * a;
    return a <= 1.0f ? ((3.0f * t2 - t5) * a + 2.0f) * 0.5f : (a * (t5 - 8.0f - t2) + 4.0f) * 0.5f;
  }
  const float a2 = a * a, a3 = a2 * a;
  return a <= 1.0f ? (7.0f / 6.0f) * a3 - 2.0f * a2 + (8.0f / 9.0f) : 2.0f * a2 - (7.0f / 18.0f) * a3 - (10.0f / 3.0f) * a + (16.0f / 9.0f);
}
