/* Test infrastructure: the kernel and the host set-up of ansel_b200/csrc/colorbalancergb.cu compiled with g++ and run thread by thread
 * on the CPU (FTZ|DAZ, as the device's -ftz=true), driven the way b200_colorbalancergb_process_dev() drives them.  Not part of the
 * product. */
#define B200_KERNELS_ON_CPU
#define __shared__ static
#include "cuda_on_cpu.h"
#include "../../include/b200iop.h"
#include "../../ansel_b200/csrc/colorbalancergb.cu"

extern "C" int emul_colorbalancergb(const float *in, float *out, size_t npixels, const b200_colorbalancergb_piece_t *pc)
{
  if(pc->data.mask_display) return B200_ERR_UNSUPPORTED;
  static cb_args_t a;
  make_cb_args(pc, &a);
  const dim3 grid((unsigned)((npixels + CB_CNT - 1) / CB_CNT));
  if(pc->data.saturation_formula == B200_COLORBALANCE_SATURATION_JZAZBZ)
    emulate(grid, CB_CNT, colorbalancergb_kernel<B200_COLORBALANCE_SATURATION_JZAZBZ>, (const float4 *)in, (float4 *)out, npixels, a);
  else
    emulate(grid, CB_CNT, colorbalancergb_kernel<B200_COLORBALANCE_SATURATION_DTUCS>, (const float4 *)in, (float4 *)out, npixels, a);
  return 0;
}
