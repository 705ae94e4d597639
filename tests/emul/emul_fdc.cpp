/* Test infrastructure: the FDC stages of ansel_b200/csrc/markesteijn.cu compiled with g++ and run thread by thread on the CPU, tile after
 * tile, in the order fdc_tiles_kernel runs them -- the threads of every stage in descending (or ascending) order, so that a stage whose
 * pixels read what the same stage writes elsewhere shows up as a difference to the oracle.  Not part of the product. */
#define B200_KERNELS_ON_CPU
#include "cuda_on_cpu.h"
#include "../../include/b200iop.h"
#include "../../ansel_b200/csrc/markesteijn.cu"
#include <vector>

extern "C" int emul_fdc(float *out, const float *in, int width, int height, int x0, int y0, const unsigned char *xtrans36, int pure, int nthreads, int ascending)
{
  _mm_setcsr(_mm_getcsr() | 0x8040u);
  mk_args_t a;
  memset(&a, 0, sizeof(a));
  a.width = width;
  a.height = height;
  a.pad = fdc_geo::PAD;
  a.step = fdc_geo::STEP;
  for(int r = 0; r < 6; r++)
    for(int c = 0; c < 6; c++) a.xt[r * 6 + c] = xtrans36[((r + y0 + 600) % 6) * 6 + (c + x0 + 600) % 6];
  mk_hexagons(a);
  fdc_offsets(a);
  a.hybrid[0] = pure ? 0.0f : 1.0f;
  a.hybrid[1] = pure ? 1.0f : 0.0f;
  a.ntx = (width + fdc_geo::STEP - 1) / fdc_geo::STEP;
  a.ntiles = a.ntx * ((height + fdc_geo::STEP - 1) / fdc_geo::STEP);
  a.in = in;
  a.out = (float4 *)out;
  std::vector<float> P((size_t)fdc_geo::PLANES * NPX, __builtin_nanf("")), isrc(NPX, __builtin_nanf(""));
  std::vector<uint8_t> homo(4 * NPX, 0xff);
  std::vector<short> start(NPX);
  a.start = start.data();
  for(int t = 0; t < a.ntiles; t++)
  {
    mk_tile_t T = mk_tile_of(a, t);
    T.cls = 0; /* one record, rebuilt per tile: the classes are checked by test_cpu_markesteijn's class test and the GPU tests */
    mk_walk(start.data(), a.xt, a.sgrow, T.top, T.left, T.nrow, T.ncol);
#define STAGE(call)                                                                                                    \
  for(int k = 0; k < nthreads; k++)                                                                                    \
  {                                                                                                                    \
    const int tid = ascending ? k : nthreads - 1 - k;                                                                  \
    call;                                                                                                              \
  }
    STAGE(mk_load<true>(a, T, P.data(), tid, nthreads, isrc.data()); fdc_zero_q(P.data(), tid, nthreads))
    STAGE(mk_green<true>(a, T, P.data(), tid, nthreads))
    STAGE(mk_solitary(a, T, P.data(), fdc_geo::PAD_SG, tid, nthreads))
    STAGE(mk_red_blue(a, T, P.data(), fdc_geo::PAD_RB, tid, nthreads))
    STAGE((mk_green_blocks<2, true>(a, T, P.data(), fdc_geo::PAD_G22, tid, nthreads)))
    STAGE(mk_derivatives<MK_FDC>(a, T, P.data(), tid, nthreads); fdc_q_yuv(T, P.data(), tid, nthreads))
    STAGE(mk_homogeneity<MK_FDC>(a, T, P.data(), homo.data(), tid, nthreads))
    STAGE(fdc_homosum(T, P.data(), homo.data(), tid, nthreads))
    STAGE(fdc_chroma(a, T, P.data(), isrc.data(), tid, nthreads))
    STAGE(fdc_final(a, T, P.data(), tid, nthreads))
#undef STAGE
  }
  return 0;
}
