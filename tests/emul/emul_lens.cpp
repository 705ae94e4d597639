/* Test infrastructure: the host plan and the kernels of ansel_b200/csrc/lens.cu compiled with g++ and run thread by thread on the CPU
 * (FTZ|DAZ, as the pipe's threads), driven the way b200_lens_process_dev() drives them.  Not part of the product. */
#define B200_KERNELS_ON_CPU
#include "cuda_on_cpu.h"
#include "../../include/b200iop.h"
#include "../../ansel_b200/csrc/lens.cu"

using namespace b200;

template <typename K, typename... A> static void emulate2d(dim3 grid, dim3 block, K kernel, A... args)
{
  _mm_setcsr(_mm_getcsr() | 0x8040u);
  blockDim = block;
  gridDim = grid;
  for(unsigned by = 0; by < grid.y; by++)
    for(unsigned bx = 0; bx < grid.x; bx++)
      for(unsigned ty = 0; ty < block.y; ty++)
        for(unsigned tx = 0; tx < block.x; tx++)
        {
          blockIdx = dim3(bx, by);
          threadIdx = dim3(tx, ty);
          kernel(args...);
        }
}

extern "C" int emul_lens_plan(const b200_lens_data_t *d, int w, int h, int monochrome, int *modflags, b200_lens_eval_t *eval)
{
  *modflags = lens_plan(d, w, h, monochrome, eval);
  return 0;
}

/* the decisions of b200_lens_process_dev with the refusals' return codes; out must hold the caller's lane 3 */
extern "C" int emul_lens(const float *in, float *out, const b200_lens_data_t *d, int itor, int monochrome, int mask_display, int in_x, int in_y, int in_w,
                         int in_h, double in_scale, int out_x, int out_y, int out_w, int out_h, int buf_in_w, int buf_in_h)
{
  const bool same_shape = in_w == out_w && in_h == out_h;
  const size_t out_bytes = (size_t)out_w * out_h * 16;
  if(!d->ls_have || d->crop <= 0.0f)
  {
    if(!same_shape) return B200_ERR_UNSUPPORTED;
    memcpy(out, in, out_bytes);
    return 0;
  }
  const float orig_w = in_scale * buf_in_w, orig_h = in_scale * buf_in_h;
  b200_lens_eval_t p;
  const int modflags = lens_plan(d, (int)orig_w, (int)orig_h, monochrome, &p);
  if((p.enabled & B200_LS_ENABLE_GEOMETRY) || p.dist_model == B200_LS_DIST_KNOTS || p.vig_model == B200_LS_VIG_KNOTS) return B200_ERR_UNSUPPORTED;
  const bool vignette = (modflags & B200_LENS_MODIFY_VIGNETTING) != 0;
  const bool geometry = (modflags & (B200_LENS_MODIFY_TCA | B200_LENS_MODIFY_DISTORTION | B200_LENS_MODIFY_GEOMETRY | B200_LENS_MODIFY_SCALE)) != 0;
  if(geometry && (in_w < 3 || in_h < 3)) return B200_ERR_UNSUPPORTED;
  if(!geometry && !same_shape) return B200_ERR_UNSUPPORTED;
  const dim3 block(LBX, LBY), grid((unsigned)((out_w + LBX - 1) / LBX), (unsigned)((out_h + LBY - 1) / LBY));
  if(!geometry)
  {
    memcpy(out, in, out_bytes);
    if(vignette) emulate2d(grid, block, lens_vignette_kernel, out, p, out_w, out_h, d->inverse ? out_x : in_x, d->inverse ? out_y : in_y);
    return 0;
  }
  const lens_geom_t g = { in_w, in_h, in_x, in_y, out_w, out_h, out_x, out_y, d->do_nan_checks ? 1 : 0, monochrome, (mask_display & B200_DISPLAY_MASK) ? 1 : 0,
                          vignette ? 1 : 0 };
  switch(itor)
  {
    case B200_INTERPOLATION_BILINEAR: emulate2d(grid, block, lens_kernel<B200_INTERPOLATION_BILINEAR>, in, out, p, g); break;
    case B200_INTERPOLATION_BICUBIC: emulate2d(grid, block, lens_kernel<B200_INTERPOLATION_BICUBIC>, in, out, p, g); break;
    default: emulate2d(grid, block, lens_kernel<B200_INTERPOLATION_MITCHELL>, in, out, p, g); break;
  }
  return 0;
}
