// diffuse or sharpen: iterations x ( a-trous B-spline decomposition into `scales` bands, then the anisotropic
// heat PDE solved band by band from coarse to fine ).
//
// Reference: src/iop/diffuse.c process :1155-1259, wavelets_process :978-1107, heat_PDE_diffusion :760-953,
// compute_kernel :727-758, tiling_callback :585-610; src/pixel/bspline.h decompose_2D_Bspline :351-377 with
// _bspline_vertical_pass :118-133 / _bspline_horizontal :136-151 (clip at zero after EACH pass).
//
// Layout: RGBA float, all four lanes processed like the reference's 4-wide vectors.  One thread per FLOAT
// (flat index = 4*pixel + lane): every tap of every stencil is then a fully coalesced 128-byte warp access,
// including the dilated ones (offset 4*mult floats), and the lane count is 4x the pixel count, which hides the
// latency of the 18-tap PDE gather without shared memory.  The stencil taps re-hit L2 (5 taps x mult rows of
// 132 KB stay far below 50 MB), so DRAM sees ~1 read + 1 write per pass.
// Per band and per pixel: vertical pass 16 B in + 16 B out, horizontal pass 32 B in + 32 B out, PDE 48 B in +
// 32 B out = 176 B; module boundary (SURVEY.md 8d) 32 B/px.  Compute-heavy part is the PDE (~110 flops + 2
// sqrt + 4 div per float).
//
// Arithmetic contract: the reference source under C float semantics (no contraction, IEEE div/sqrt), as
// restated in oracle/restate/diffuse_oracle.c, which is bit-identical to diffuse.c's own process().
#include "runtime.h"
#include "flt32_math.cuh"
#include "bspline.cuh"
#include <math.h>

namespace
{
constexpr int MAX_SCALES = B200_DIFFUSE_MAX_SCALES;
constexpr float B_SPLINE_SIGMA = 1.0553651328015339f; // bspline.h:38
constexpr float KAPPA = 0.25f;                        // diffuse.c:624
using namespace bsp; // NT, clip0, max_zero, the two B-spline kernels, splitmix32, xoshiro128plus

// (int) of a float the way x86 cvttss2si does it: out of range and NaN give INT_MIN
__device__ __forceinline__ int cvtt(float v) { return (v >= -2147483648.0f && v < 2147483648.0f) ? __float2int_rz(v) : (int)0x80000000; }
__device__ __forceinline__ float fast_expf(float x)
{ // dt_fast_expf, math/math.h:254-267
  const int k0 = cvtt(1065353216.0f + x * 11401300.0f); // i1 + x * (i2 - i1), evaluated in float
  return __int_as_float(k0 > 0 ? k0 : 0);
}

struct pde_t
{
  float anisotropy[4];
  int isotropy[4]; // dt_isotropy_t per order
  float variance_threshold, normalized_regularization, ABCD[4], strength;
};

// compute_kernel(), diffuse.c:727-758
__device__ __forceinline__ void make_kernel(float c2, float cs, float cos2, float sin2, int type, float k[9])
{
  if(type == 0)
  { // isotrope_laplacian :709-725
    k[0] = k[2] = k[6] = k[8] = 0.25f;
    k[1] = k[3] = k[5] = k[7] = 0.5f;
    k[4] = -3.f;
    return;
  }
  float a00, a11, a01;
  if(type == 1)
  { // rotation_matrix_isophote :648-661
    a00 = cos2 + c2 * sin2;
    a11 = c2 * cos2 + sin2;
    a01 = (c2 - 1.f) * cs;
  }
  else
  { // rotation_matrix_gradient :663-677
    a00 = c2 * cos2 + sin2;
    a11 = cos2 + c2 * sin2;
    a01 = (1.f - c2) * cs;
  }
  const float b11 = a01 * 0.5f, b13 = -b11, b22 = -2.f * (a00 + a11); // build_matrix :679-707
  k[0] = b11;
  k[1] = a11;
  k[2] = b13;
  k[3] = a00;
  k[4] = b22;
  k[5] = a00;
  k[6] = b13;
  k[7] = a11;
  k[8] = b11;
}

// ---- luminance mask (threshold > 0): build_mask :1109-1119, inpaint_mask :1122-1152 -----------------------------
// iop/noise_generator.h: splitmix32 :36-43, xoshiro128plus :54-70, gaussian_noise :82-96 (Box-Muller on glibc
// logf / sinf / cosf -> flt32_math.cuh).
__device__ __forceinline__ float gaussian_noise(const f32m::tables_t &tb, float mu, float sigma, bool flip, uint32_t (&st)[4])
{
  const float u1 = fmaxf(xoshiro128plus(st), 1.17549435e-38f);
  const float u2 = xoshiro128plus(st);
  const float radius = sqrtf(-2.0f * f32m::logf_(tb, u1));
  const float angle = (float)(6.283185307179586 * (double)u2); // 2.f * M_PI * u2 is a double product in the source
  const float noise = flip ? radius * f32m::cosf_(angle) : radius * f32m::sinf_(angle);
  return noise * sigma + mu;
}
// one thread per pixel: the mask byte, and the start image -- the input outside the mask, |noise around the input| inside
__global__ void __launch_bounds__(NT) mask_inpaint_kernel(const float4 *__restrict__ in, float4 *__restrict__ inpainted, unsigned char *__restrict__ mask,
                                                          size_t npx, unsigned width, float threshold)
{
  const size_t px = (size_t)blockIdx.x * NT + threadIdx.x;
  if(px >= npx) return;
  const float4 v = __ldg(in + px);
  const bool m = v.x > threshold || v.y > threshold || v.z > threshold;
  mask[px] = m ? 1 : 0;
  if(!m)
  {
    inpainted[px] = v;
    return;
  }
  const f32m::tables_t tb = f32m::global_tables();
  // the reference seeds from the FLOAT index k = 4*px and k / width (:1132-1136)
  const size_t k = 4 * px;
  const uint32_t i = (uint32_t)(k / width);
  const uint32_t j = (uint32_t)(k - i);
  uint32_t st[4] = { splitmix32((uint64_t)(uint32_t)(j + 1u)), splitmix32((uint64_t)(uint32_t)(j + 1u) * (uint64_t)(uint32_t)(i + 3u)), splitmix32(1337), splitmix32(666) };
  xoshiro128plus(st);
  xoshiro128plus(st);
  xoshiro128plus(st);
  xoshiro128plus(st);
  const bool flip = (i % 2u) || (j % 2u);
  float4 o;
  o.x = fabsf(gaussian_noise(tb, v.x, v.x, flip, st));
  o.y = fabsf(gaussian_noise(tb, v.y, v.y, flip, st));
  o.z = fabsf(gaussian_noise(tb, v.z, v.z, flip, st));
  o.w = fabsf(gaussian_noise(tb, v.w, v.w, flip, st));
  inpainted[px] = o;
}

// heat_PDE_diffusion(), :760-953; mask == nullptr is has_mask == 0
// R holds (HF/safe(LF))^2 of this band per float -- every pixel's term is needed by its nine neighbours, so it is
// computed once where LF is produced (the previous, coarser PDE step or the last B-spline pass) instead of nine
// times here: one IEEE division per float instead of nine.  HFnext/Rnext: the next finer band, whose LF is `out`.
__global__ void __launch_bounds__(NT) heat_pde_kernel(const float *__restrict__ HF, const float *__restrict__ LF, const float *__restrict__ R,
                                                      float *__restrict__ out, const float *__restrict__ HFnext, float *__restrict__ Rnext,
                                                      const unsigned char *__restrict__ mask, int w4, int width, int height, int mult, const pde_t p)
{
  const int x = blockIdx.x * NT + threadIdx.x, i = blockIdx.y;
  if(x >= w4) return;
  const int j = x >> 2, c = x & 3;
  const size_t rn[3] = { (size_t)w4 * max(i - mult, 0), (size_t)w4 * i, (size_t)w4 * min(i + mult, height - 1) };
  if(mask && !mask[(size_t)i * width + j])
  { // :938-947: outside the mask the band is only added back
    const float o = max_zero(__ldg(HF + rn[1] + x) + __ldg(LF + rn[1] + x));
    out[rn[1] + x] = o;
    if(Rnext) Rnext[rn[1] + x] = ratio_sq(__ldg(HFnext + rn[1] + x), o);
    return;
  }
  const int cn[3] = { 4 * max(j - mult, 0) + c, x, 4 * min(j + mult, width - 1) + c };
  float hf[9], lf[9];
#pragma unroll
  for(int ii = 0; ii < 3; ii++)
#pragma unroll
    for(int jj = 0; jj < 3; jj++)
    {
      hf[3 * ii + jj] = __ldg(HF + rn[ii] + cn[jj]);
      lf[3 * ii + jj] = __ldg(LF + rn[ii] + cn[jj]);
    }
  float energy = 0.f;
#pragma unroll
  for(int ii = 0; ii < 3; ii++)
#pragma unroll
    for(int jj = 0; jj < 3; jj++) energy += __ldg(R + rn[ii] + cn[jj]);
  energy = max_zero(p.variance_threshold + energy * p.normalized_regularization - 1e-8f) + 1e-8f;

  float cs[2], cos2[2], sin2[2], mag[2];
#pragma unroll
  for(int g = 0; g < 2; g++)
  { // g = 0: gradient of LF, g = 1: gradient of HF (the reference's "lapl")
    const float *px = g ? hf : lf;
    float gx = (px[7] - px[1]) * 0.5f, gy = (px[5] - px[3]) * 0.5f; // find_gradients :627-635
    const float m = sqrtf(gx * gx + gy * gy);
    const float nonzero = (m != 0.f) ? 1.0f : 0.0f;
    const float inv_mag = 1.f / (m + (1.f - nonzero));
    gx = gx * inv_mag + (1.f - nonzero);
    gy = gy * inv_mag;
    mag[g] = m;
    cos2[g] = gx * gx;
    sin2[g] = gy * gy;
    cs[g] = gx * gy;
  }
  float d[4] = { 0.f, 0.f, 0.f, 0.f };
#pragma unroll
  for(int o = 0; o < 4; o++)
  { // orders 1,3 follow the LF gradient, 2,4 the HF gradient; orders 1,2 act on LF, 3,4 on HF
    const int g = o & 1;
    float k[9];
    make_kernel(fast_expf(-mag[g] * p.anisotropy[o]), cs[g], cos2[g], sin2[g], p.isotropy[o], k);
    const float *px = (o < 2) ? lf : hf;
#pragma unroll
    for(int t = 0; t < 9; t++) d[o] = k[t] * px[t] + d[o];
  }
  float update = d[0] * p.ABCD[0];
  update = d[1] * p.ABCD[1] + update;
  update = d[2] * p.ABCD[2] + update;
  update = d[3] * p.ABCD[3] + update;
  const float acc = hf[4] * p.strength + update / energy;
  const float o = max_zero(acc + lf[4]);
  out[rn[1] + x] = o;
  if(Rnext) Rnext[rn[1] + x] = ratio_sq(__ldg(HFnext + rn[1] + x), o);
}

float sigma_at_step(unsigned s)
{ // equivalent_sigma_at_step, bspline.h:52-63
  if(s == 0) return B_SPLINE_SIGMA;
  const float prev = sigma_at_step(s - 1), e = exp2f((float)s) * B_SPLINE_SIGMA;
  return sqrtf(prev * prev + e * e);
}
int scale_count(const b200_diffuse_data_t *d, float zoom)
{ // diffuse.c:1175-1183, num_steps_to_reach_equivalent_sigma bspline.h:65-77
  const float final_radius = (d->radius + d->radius_center) * 2.f / zoom;
  unsigned s = 0;
  float radius = B_SPLINE_SIGMA;
  while(radius < final_radius)
  {
    ++s;
    const float e = (float)(1 << s) * B_SPLINE_SIGMA;
    radius = sqrtf(radius * radius + e * e);
  }
  const int n = (int)(s + 1);
  return n < 1 ? 1 : (n > MAX_SCALES ? MAX_SCALES : n);
}
} // namespace

using namespace b200;

static int check_df(const b200_piece_t *piece, const void *in, void *out)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "diffuse: NULL argument");
  if(!piece->data || piece->data_size < sizeof(b200_diffuse_data_t)) return fail(B200_ERR_ARG, "diffuse: piece->data is not a b200_diffuse_data_t");
  const b200_diffuse_data_t *d = (const b200_diffuse_data_t *)piece->data;
  if(in == out) return fail(B200_ERR_ARG, "diffuse: in-place processing is not supported");
  if(piece->roi_in.width != piece->roi_out.width || piece->roi_in.height != piece->roi_out.height)
    return fail(B200_ERR_ARG, "diffuse: roi_in and roi_out differ in size");
  return B200_OK;
}

extern "C" int b200_diffuse_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = check_df(piece, d_in, d_out);
  if(rc) return rc;
  if((rc = bind_device(piece->devid))) return rc;
  const b200_diffuse_data_t *d = (const b200_diffuse_data_t *)piece->data;
  cudaStream_t st = (cudaStream_t)stream;
  const int width = piece->roi_out.width, height = piece->roi_out.height;
  if(width <= 0 || height <= 0) return B200_OK;
  const size_t n = (size_t)width * height * 4;
  const float zoom = (float)((double)piece->iscale / piece->roi_in.scale); // dt_dev_get_module_scale, develop/imageop.c:134-137 (double division)
  const int it_f = (int)ceilf((float)d->iterations);
  const int iterations = it_f > 1 ? it_f : 1;
  const int scales = scale_count(d, zoom);

  void *base = nullptr;
  if((rc = scratch(SLOT_TMP0, (size_t)(scales + 7) * n * sizeof(float) + n / 4, &base))) return rc;
  float *p = (float *)base;
  float *HF[MAX_SCALES];
  for(int s = 0; s < scales; s++, p += n) HF[s] = p;
  float *const LF_odd = p, *const LF_even = p + n, *const temp1 = p + 2 * n, *const temp2 = p + 3 * n, *const vtmp = p + 4 * n;
  float *Rbuf[2] = { p + 5 * n, p + 6 * n }; // energy terms of the band being solved / of the next one
  unsigned char *mask = nullptr;            // one byte per pixel, behind the float planes

  // wavelets_process() :985-1000, :1057-1075: per-call constants
  pde_t pde;
  const float an[4] = { d->anisotropy_first, d->anisotropy_second, d->anisotropy_third, d->anisotropy_fourth };
  for(int k = 0; k < 4; k++)
  {
    pde.anisotropy[k] = an[k] * an[k];                                  // compute_anisotropy_factor :955-962
    pde.isotropy[k] = an[k] == 0.f ? 0 : (an[k] > 0.f ? 1 : 2);         // check_isotropy_mode :151-162
  }
  const float regularization = powf(10.f, d->regularization) - 1.f;
  pde.variance_threshold = powf(10.f, d->variance_threshold);

  const int w4 = 4 * width;
  const dim3 grid((w4 + NT - 1) / NT, height);        // PDE: one thread per float
  const dim3 grid_px((width + NT - 1) / NT, height);  // B-spline passes: one thread per pixel
  if(d->threshold > 0.f)
  { // :1207-1218: mask of the pixels above the threshold, noise-seeded start image in temp1
    mask = (unsigned char *)(p + 7 * n);
    const size_t npx = n / 4;
    mask_inpaint_kernel<<<(unsigned)((npx + NT - 1) / NT), NT, 0, st>>>((const float4 *)d_in, (float4 *)temp1, mask, npx, (unsigned)width, d->threshold);
    B200_CUDA_TRY(cudaGetLastError());
    d_in = temp1;
  }
  for(int it = 0; it < iterations; it++)
  {
    const float *temp_in = it == 0 ? (const float *)d_in : (it % 2 == 0 ? temp1 : temp2);
    float *temp_out = it == 0 ? temp2 : (it % 2 == 0 ? temp2 : temp1);
    if(it == iterations - 1) temp_out = (float *)d_out;

    float *residual = nullptr;
    for(int s = 0; s < scales; s++)
    {
      const float *bin = s == 0 ? temp_in : (s % 2 != 0 ? LF_odd : LF_even);
      float *bout = s == 0 ? LF_odd : (s % 2 != 0 ? LF_even : LF_odd);
      bspline_vertical_kernel<<<grid_px, NT, 0, st>>>((const float4 *)bin, (float4 *)vtmp, width, height, 1 << s);
      bspline_horizontal_kernel<<<grid_px, NT, 0, st>>>((const float4 *)vtmp, (const float4 *)bin, (float4 *)bout, (float4 *)HF[s],
                                                      s == scales - 1 ? (float4 *)Rbuf[0] : nullptr, width, 1 << s);
      residual = bout;
    }
    B200_CUDA_TRY(cudaGetLastError());
    float *temp = residual == LF_even ? LF_odd : LF_even;
    int count = 0;
    for(int s = scales - 1; s > -1; --s)
    {
      const float real_radius = sigma_at_step(s) * zoom;
      pde.normalized_regularization = regularization / 9.f * (real_radius * real_radius);
      const float dr = real_radius - (float)d->radius_center, rad = (float)d->radius;
      const float norm = expf(-(dr * dr) / (rad * rad));
      pde.ABCD[0] = d->first * KAPPA * norm;
      pde.ABCD[1] = d->second * KAPPA * norm;
      pde.ABCD[2] = d->third * KAPPA * norm;
      pde.ABCD[3] = d->fourth * KAPPA * norm;
      pde.strength = d->sharpness * norm + 1.f;
      const float *bin = count == 0 ? residual : (count % 2 != 0 ? temp : residual);
      float *bout = count == 0 ? temp : (count % 2 != 0 ? residual : temp);
      if(s == 0) bout = temp_out;
      heat_pde_kernel<<<grid, NT, 0, st>>>(HF[s], bin, Rbuf[count & 1], bout, s > 0 ? HF[s - 1] : nullptr, s > 0 ? Rbuf[(count + 1) & 1] : nullptr, mask, w4,
                                           width, height, 1 << s, pde);
      count++;
    }
    B200_CUDA_TRY(cudaGetLastError());
  }
  return B200_OK;
}

extern "C" int b200_diffuse_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_df(piece, in, out);
  if(rc) return rc;
  const size_t bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 16;
  return through_device(piece, in, bytes, out, bytes, false, b200_diffuse_process_dev);
}

// tiling_callback(), diffuse.c:585-610
extern "C" void b200_diffuse_tiling(const b200_piece_t *piece, b200_tiling_t *tiling)
{
  if(!piece || !tiling || !piece->data) return;
  const b200_diffuse_data_t *d = (const b200_diffuse_data_t *)piece->data;
  const float zoom = (float)((double)piece->iscale / piece->roi_in.scale);
  const int scales = scale_count(d, zoom);
  tiling->factor = 6.0625f + scales;
  tiling->factor_cl = 6.0625f + scales;
  tiling->maxbuf = 1.0f;
  tiling->maxbuf_cl = 1.0f;
  tiling->overhead = 0;
  tiling->overlap = 1 << scales;
  tiling->xalign = 1;
  tiling->yalign = 1;
}
