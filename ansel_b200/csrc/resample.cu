// finalscale: the export's final resampling (and the darkroom's final upscale).
//
// Reference: iop/finalscale.c process() :117-131 -> develop/imageop_math.c dt_iop_clip_and_zoom_roi :146-152 ->
// pixel/interpolation.c _interpolation_resample_plain :897-1027 with the per-axis plans of _prepare_resampling_plan
// :710-893 (tap generators :175-287, _compute_upsampling_kernel :320-342, _compute_downsampling_kernel :354-387).
//
// The plans are a few thousand floats and are built on the host exactly as the reference builds them (same float
// operations in the same order: the tap positions advance by 4 * interval per group of four, the norm is a sequential
// sum).  The pixel loop is the device's: one thread per output pixel accumulates rows, and columns within a row, in the
// reference's order, so the result is bit-identical; a separable two-pass resampler would be cheaper in flops but rounds
// differently.  A block is 128 consecutive pixels of one output row: the vertical taps are uniform across the block, the
// horizontal taps of neighbouring threads overlap (L1).  Downscaling 45 MP by s reads (4/s)^2 float4 per output pixel
// out of L1/L2 and writes 16 s^2 * 45 M bytes: bounded by L1/L2 gather throughput, not by HBM.
#ifndef B200_KERNELS_ON_CPU // tests/emul compiles the kernels and the plan builder of this file with g++
#include "runtime.h"
#endif
#include <math.h>
#include <string.h>
#include <vector>
#include "interp_taps.cuh"

namespace
{
constexpr int RNT = 128;

struct axis_plan_t
{
  std::vector<int> length, offset, index; // per output sample: number of taps, where they start; per tap: input sample
  std::vector<float> kernel;              // per tap: normalised weight
};

inline float ceil_fast(float x) { return x <= 0.f ? (float)(int)x : -((float)(int)-x) + 1.f; } // math/math.h:324-334
inline int half_width(int interpolator) { return interpolator == B200_INTERPOLATION_BILINEAR ? 1 : 2; }
// the reference generates taps four at a time: lane k starts at first + k * interval and every lane advances by
// 4 * interval per group, so tap n sits at (((first + (n % 4) * interval) + 4 interval) + 4 interval) ...  (n / 4 times)
inline void make_taps(int interpolator, float *taps, int num_taps, float first_tap, float interval)
{
  const float iter = 4.0f * interval;
  for(int k = 0; k < 4 && k < num_taps; k++)
  {
    float t = first_tap + (float)k * interval;
    for(int n = k; n < num_taps; n += 4)
    {
      taps[n] = tap_weight(interpolator, t);
      t += iter;
    }
  }
}

// _prepare_resampling_plan :710-893 for one axis (RESAMPLING_BORDER_MODE = replicate: every tap kept, indexes clipped).
// false when scale == 1 (nothing to resample).
bool build_axis_plan(int interpolator, int in, int in_x0, int out, int out_x0, float scale, axis_plan_t &P)
{
  P.length.clear(), P.offset.clear(), P.index.clear(), P.kernel.clear();
  if(scale == 1.f) return false;
  const int width = half_width(interpolator);
  const int maxtaps = scale > 1.f ? 2 * width : (int)ceil_fast((float)2 * (float)width / scale);
  std::vector<float> scratch((size_t)maxtaps + 8);
  P.length.reserve(out), P.offset.reserve(out);
  P.kernel.reserve((size_t)out * maxtaps), P.index.reserve((size_t)out * maxtaps);
  for(int x = 0; x < out; x++)
  {
    int first, taps;
    if(scale > 1.f)
    { // _compute_upsampling_kernel
      const float fx = (float)(out_x0 + x) / scale - (float)in_x0;
      first = (int)floorf(fx) - width + 1;
      taps = 2 * width;
      make_taps(interpolator, scratch.data(), taps, fx - (float)first, -1.0f);
    }
    else
    { // _compute_downsampling_kernel
      const float w = (float)width;
      const float xin = ceil_fast(((float)(out_x0 + x) - w) / scale);
      first = (int)xin;
      const float t = xin * scale - (float)(out_x0 + x);
      taps = (int)((w - t) / scale);
      if(taps < 0) taps = 0;
      if((size_t)taps + 4 > scratch.size()) scratch.resize((size_t)taps + 8);
      make_taps(interpolator, scratch.data(), taps, t, scale);
    }
    P.length.push_back(taps);
    P.offset.push_back((int)P.kernel.size());
    float norm = 0.f;
    for(int k = 0; k < taps; k++) norm += scratch[k];
    norm = 1.f / norm;
    for(int k = 0; k < taps; k++)
    {
      P.kernel.push_back(scratch[k] * norm);
      const int i = first + k;
      P.index.push_back(i < 0 ? 0 : (i > in - 1 ? in - 1 : i));
    }
  }
  return true;
}

struct plan_view_t
{ // device (or, under emulation, host) arrays of the two axes
  const int *hlen, *hoff, *hidx, *vlen, *voff, *vidx;
  const float *hker, *vker;
};

__device__ __forceinline__ float max_zero(float v)
{ // dt_simd_max_zero, system/simd.h:108-114: finite ? MAX(v, 0) : 0
  return ((__float_as_uint(v) & 0x7f800000u) != 0x7f800000u && v > 0.0f) ? v : 0.0f;
}

__global__ void __launch_bounds__(RNT) resample_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, int in_w, int out_w, plan_view_t P)
{
  const int ox = blockIdx.x * RNT + threadIdx.x, oy = blockIdx.y;
  if(ox >= out_w) return;
  const int hl = P.hlen[ox], vl = P.vlen[oy];
  const int *hidx = P.hidx + P.hoff[ox], *vidx = P.vidx + P.voff[oy];
  const float *hker = P.hker + P.hoff[ox], *vker = P.vker + P.voff[oy];
  float4 vs = make_float4(0.f, 0.f, 0.f, 0.f);
  for(int iy = 0; iy < vl; iy++)
  {
    const float4 *line = in + (size_t)vidx[iy] * in_w;
    float4 vhs = make_float4(0.f, 0.f, 0.f, 0.f);
    for(int ix = 0; ix < hl; ix++)
    {
      const float4 p = line[hidx[ix]];
      const float t = hker[ix];
      vhs.x += p.x * t;
      vhs.y += p.y * t;
      vhs.z += p.z * t;
      vhs.w += p.w * t;
    }
    const float t = vker[iy];
    vs.x += vhs.x * t;
    vs.y += vhs.y * t;
    vs.z += vhs.z * t;
    vs.w += vhs.w * t;
  }
  out[(size_t)oy * out_w + ox] = make_float4(max_zero(vs.x), max_zero(vs.y), max_zero(vs.z), max_zero(vs.w));
}

// the 1:1 path :916-932: rows of the output copied from the top-left corner of the input
__global__ void __launch_bounds__(RNT) copy_rows_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, int in_w, int out_w)
{
  const int ox = blockIdx.x * RNT + threadIdx.x, oy = blockIdx.y;
  if(ox < out_w) out[(size_t)oy * out_w + ox] = in[(size_t)oy * in_w + ox];
}
// the 1:1 path with ROI origins :916-932: the output is a crop of the input at (dx, dy) = roi_out - roi_in
__global__ void __launch_bounds__(RNT) crop_rows_kernel(const float4 *__restrict__ in, float4 *__restrict__ out, int in_w, int out_w, int dx, int dy)
{
  const int ox = blockIdx.x * RNT + threadIdx.x, oy = blockIdx.y;
  if(ox < out_w) out[(size_t)oy * out_w + ox] = in[(size_t)(oy + dy) * in_w + ox + dx];
}
// dt_imageio_flip_buffers, imageio/imageio_core.c:258-297: pixel (i, j) of the input lands at |sj| jj + |si| ii + sj j + si i
// (in pixels here; `ch` floats per pixel)
__global__ void __launch_bounds__(RNT) flip_kernel(const float *__restrict__ in, float *__restrict__ out, int width, int height, int ch, int orientation)
{
  const int i = blockIdx.x * RNT + threadIdx.x, j = blockIdx.y;
  if(i >= width) return;
  long ii = 0, jj = 0, si = 1, sj = width;
  if(orientation & 4)
  {
    sj = 1;
    si = height;
  }
  if(orientation & 1)
  {
    jj = height - 1;
    sj = -sj;
  }
  if(orientation & 2)
  {
    ii = width - 1;
    si = -si;
  }
  const long o = (sj < 0 ? -sj : sj) * jj + (si < 0 ? -si : si) * ii + sj * j + si * i;
  const size_t p = (size_t)j * width + i;
  if(ch == 4)
    ((float4 *)out)[o] = ((const float4 *)in)[p];
  else
    for(int c = 0; c < ch; c++) out[(size_t)o * ch + c] = in[p * ch + c];
}
} // namespace

#ifndef B200_KERNELS_ON_CPU
using namespace b200;

extern "C" int b200_resampling_plan(int interpolator, int in, int in_x0, int out, int out_x0, float scale, int *lengths, float *kernel, int *index,
                                    int max_taps)
{
  if(interpolator < B200_INTERPOLATION_BILINEAR || interpolator > B200_INTERPOLATION_MITCHELL || in < 1 || out < 1 || !(scale > 0.f) || !lengths || !kernel
     || !index)
    return -2;
  axis_plan_t P;
  if(!build_axis_plan(interpolator, in, in_x0, out, out_x0, scale, P)) return -1;
  if((int)P.kernel.size() > max_taps) return -3;
  memcpy(lengths, P.length.data(), sizeof(int) * out);
  memcpy(kernel, P.kernel.data(), sizeof(float) * P.kernel.size());
  memcpy(index, P.index.data(), sizeof(int) * P.index.size());
  return (int)P.kernel.size();
}

static int clip_and_zoom_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream, bool keep_origins);
extern "C" int b200_finalscale_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  return clip_and_zoom_dev(piece, d_in, d_out, stream, false); // process() :117-131 zeroes the origins of both ROIs
}
extern "C" int b200_initialscale_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  return clip_and_zoom_dev(piece, d_in, d_out, stream, true); // iop/initialscale.c:122-129: the ROIs as they are
}
// dt_iop_clip_and_zoom_roi (develop/imageop_math.c:146-152) -> _interpolation_resample_plain
static int clip_and_zoom_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream, bool keep_origins)
{
  if(!piece || !d_in || !d_out) return fail(B200_ERR_ARG, "finalscale: NULL argument");
  if(!piece->data || piece->data_size < sizeof(b200_finalscale_data_t)) return fail(B200_ERR_ARG, "finalscale: piece->data is not a b200_finalscale_data_t");
  if(d_in == d_out) return fail(B200_ERR_ARG, "finalscale: in-place processing is not supported");
  const int itor = ((const b200_finalscale_data_t *)piece->data)->interpolator;
  if(itor < B200_INTERPOLATION_BILINEAR || itor > B200_INTERPOLATION_MITCHELL) return fail(B200_ERR_ARG, "finalscale: interpolator %d", itor);
  const int in_w = piece->roi_in.width, in_h = piece->roi_in.height, out_w = piece->roi_out.width, out_h = piece->roi_out.height;
  if(in_w < 1 || in_h < 1 || out_w < 1 || out_h < 1 || out_h > 65535) return fail(B200_ERR_ARG, "finalscale: %dx%d -> %dx%d", in_w, in_h, out_w, out_h);
  if(!(piece->roi_in.scale > 0.0) || !(piece->roi_out.scale > 0.0)) return fail(B200_ERR_ARG, "finalscale: roi scales %g -> %g", piece->roi_in.scale, piece->roi_out.scale);
  int rc = bind_device(piece->devid);
  if(rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid((unsigned)((out_w + RNT - 1) / RNT), (unsigned)out_h);
  const int in_x = keep_origins ? piece->roi_in.x : 0, in_y = keep_origins ? piece->roi_in.y : 0;
  const int out_x = keep_origins ? piece->roi_out.x : 0, out_y = keep_origins ? piece->roi_out.y : 0;
  if(piece->roi_out.scale == 1.f || piece->roi_out.scale == piece->roi_in.scale)
  {
    const int dx = out_x - in_x, dy = out_y - in_y;
    if(dx < 0 || dy < 0 || dx + out_w > in_w || dy + out_h > in_h)
      return fail(B200_ERR_ARG, "finalscale: 1:1 copy of %dx%d at %d,%d out of %dx%d", out_w, out_h, dx, dy, in_w, in_h);
    if(dx == 0 && dy == 0)
      copy_rows_kernel<<<grid, RNT, 0, s>>>((const float4 *)d_in, (float4 *)d_out, in_w, out_w);
    else
      crop_rows_kernel<<<grid, RNT, 0, s>>>((const float4 *)d_in, (float4 *)d_out, in_w, out_w, dx, dy);
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
  }
  const float resample_scale = (float)(piece->roi_out.scale / piece->roi_in.scale); // :939, a double division stored in a float
  axis_plan_t H, V;
  if(!build_axis_plan(itor, in_w, in_x, out_w, out_x, resample_scale, H) || !build_axis_plan(itor, in_h, in_y, out_h, out_y, resample_scale, V))
    return fail(B200_ERR_ARG, "finalscale: resampling scale rounds to 1 between different ROI scales");
  // one upload: [hlen | hoff | hidx | vlen | voff | vidx | hker | vker]
  const size_t nh = H.kernel.size(), nv = V.kernel.size();
  const size_t words = 2 * (size_t)out_w + 2 * (size_t)out_h + 2 * nh + 2 * nv;
  std::vector<int> blob(words);
  int *w = blob.data();
  const size_t o_hlen = 0, o_hoff = o_hlen + out_w, o_hidx = o_hoff + out_w, o_vlen = o_hidx + nh, o_voff = o_vlen + out_h, o_vidx = o_voff + out_h,
               o_hker = o_vidx + nv, o_vker = o_hker + nh;
  memcpy(w + o_hlen, H.length.data(), sizeof(int) * out_w);
  memcpy(w + o_hoff, H.offset.data(), sizeof(int) * out_w);
  memcpy(w + o_hidx, H.index.data(), sizeof(int) * nh);
  memcpy(w + o_vlen, V.length.data(), sizeof(int) * out_h);
  memcpy(w + o_voff, V.offset.data(), sizeof(int) * out_h);
  memcpy(w + o_vidx, V.index.data(), sizeof(int) * nv);
  memcpy(w + o_hker, H.kernel.data(), sizeof(float) * nh);
  memcpy(w + o_vker, V.kernel.data(), sizeof(float) * nv);
  void *dp = nullptr;
  if((rc = scratch(SLOT_SMALL + 4, words * sizeof(int), &dp))) return rc;
  // pageable source: the runtime stages it before returning, so the vector may go out of scope
  B200_CUDA_TRY(cudaMemcpyAsync(dp, blob.data(), words * sizeof(int), cudaMemcpyHostToDevice, s));
  const int *d = (const int *)dp;
  const plan_view_t P = { d + o_hlen, d + o_hoff, d + o_hidx, d + o_vlen, d + o_voff, d + o_vidx, (const float *)(d + o_hker), (const float *)(d + o_vker) };
  resample_kernel<<<grid, RNT, 0, s>>>((const float4 *)d_in, (float4 *)d_out, in_w, out_w, P);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}

static int check_zoom(const b200_piece_t *piece, const void *in, const void *out)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "finalscale: NULL argument");
  if(piece->roi_in.width < 1 || piece->roi_in.height < 1 || piece->roi_out.width < 1 || piece->roi_out.height < 1)
    return fail(B200_ERR_ARG, "finalscale: empty ROI");
  return B200_OK;
}
extern "C" int b200_finalscale_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_zoom(piece, in, out);
  if(rc) return rc;
  const size_t in_bytes = (size_t)piece->roi_in.width * piece->roi_in.height * 16, out_bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 16;
  return through_device(piece, in, in_bytes, out, out_bytes, false, b200_finalscale_process_dev);
}
extern "C" int b200_initialscale_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = check_zoom(piece, in, out);
  if(rc) return rc;
  const size_t in_bytes = (size_t)piece->roi_in.width * piece->roi_in.height * 16, out_bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 16;
  return through_device(piece, in, in_bytes, out, out_bytes, false, b200_initialscale_process_dev);
}

// neither module declares a tiling callback; both have IOP_FLAGS_TILING_FULL_ROI
extern "C" void b200_finalscale_tiling(const b200_piece_t *piece, b200_tiling_t *t) { default_tiling(piece, t, 4, false); }
#endif // B200_KERNELS_ON_CPU

#ifndef B200_KERNELS_ON_CPU
extern "C" void b200_initialscale_tiling(const b200_piece_t *piece, b200_tiling_t *t) { default_tiling(piece, t, 4, false); }

// ---- flip -------------------------------------------------------------------------------------------------------------------------
extern "C" int b200_flip_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  if(!piece || !d_in || !d_out) return fail(B200_ERR_ARG, "flip: NULL argument");
  if(!piece->data || piece->data_size < sizeof(b200_flip_data_t)) return fail(B200_ERR_ARG, "flip: piece->data is not a b200_flip_data_t");
  if(d_in == d_out) return fail(B200_ERR_ARG, "flip: in-place processing is not supported");
  const int w = piece->roi_in.width, h = piece->roi_in.height, ch = (int)piece->channels;
  const int orientation = ((const b200_flip_data_t *)piece->data)->orientation;
  if(w < 1 || h < 1 || h > 65535 || ch < 1) return fail(B200_ERR_ARG, "flip: %d x %d x %d", w, h, ch);
  if(orientation < 0 || orientation > 7) return fail(B200_ERR_ARG, "flip: orientation %d", orientation);
  int rc = bind_device(piece->devid);
  if(rc) return rc;
  flip_kernel<<<dim3((unsigned)((w + RNT - 1) / RNT), (unsigned)h), RNT, 0, (cudaStream_t)stream>>>((const float *)d_in, (float *)d_out, w, h, ch, orientation);
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}
extern "C" int b200_flip_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "flip: NULL argument");
  if(piece->roi_in.width < 1 || piece->roi_in.height < 1 || piece->channels < 1) return fail(B200_ERR_ARG, "flip: empty ROI");
  const size_t bytes = (size_t)piece->roi_in.width * piece->roi_in.height * piece->channels * sizeof(float);
  return through_device(piece, in, bytes, out, bytes, false, b200_flip_process_dev);
}
extern "C" void b200_flip_tiling(const b200_piece_t *piece, b200_tiling_t *t)
{ // flip.c tiling_callback: in + out, no overlap; the module does not define alignment
  if(!piece || !t) return;
  t->factor = 2.0f;
  t->factor_cl = 2.0f;
  t->maxbuf = 1.0f;
  t->maxbuf_cl = 1.0f;
  t->overhead = 0;
  t->overlap = 0;
  t->xalign = 1;
  t->yalign = 1;
}
#endif

#ifndef B200_KERNELS_ON_CPU
// ---- basebuffer: the crop of the sensor buffer is the upload -------------------------------------------------------------------------
extern "C" int b200_basebuffer_upload_dev(const b200_piece_t *piece, const void *host_full, int iwidth, int iheight, size_t bpp, void *d_out, void *stream)
{
  if(!piece || !host_full || !d_out) return fail(B200_ERR_ARG, "basebuffer: NULL argument");
  if(iwidth < 1 || iheight < 1 || bpp < 1 || piece->roi_out.width < 1 || piece->roi_out.height < 1) return fail(B200_ERR_ARG, "basebuffer: empty buffer or ROI");
  int rc = bind_device(piece->devid);
  if(rc) return rc;
  // basebuffer.c:127-139: the crop origin clamped at 0, its size clamped to what the buffer holds from there
  const size_t x = piece->roi_out.x > 0 ? (size_t)piece->roi_out.x : 0, y = piece->roi_out.y > 0 ? (size_t)piece->roi_out.y : 0;
  if(x >= (size_t)iwidth || y >= (size_t)iheight) return fail(B200_ERR_ARG, "basebuffer: roi_out origin %zu,%zu outside the %dx%d buffer", x, y, iwidth, iheight);
  const size_t in_width = (size_t)piece->roi_out.width < (size_t)iwidth - x ? (size_t)piece->roi_out.width : (size_t)iwidth - x;
  const size_t in_height = (size_t)piece->roi_out.height < (size_t)iheight - y ? (size_t)piece->roi_out.height : (size_t)iheight - y;
  const size_t in_stride = (size_t)iwidth * bpp, out_stride = (size_t)piece->roi_out.width * bpp;
  B200_CUDA_TRY(cudaMemcpy2DAsync(d_out, out_stride, (const char *)host_full + y * in_stride + x * bpp, in_stride, in_width * bpp, in_height, cudaMemcpyHostToDevice,
                                  (cudaStream_t)stream));
  return B200_OK;
}
#endif
