/* Test infrastructure: nlm_pipe_kernel's half-height path on the paired window and the interleaved slots (pipe2_fill,
 * pipe2_colwalk_t, pipe2_b1_rows, pipe2_own_init, pipe2_accumulate in ansel_b200/csrc/nlm_group.cuh) compiled with g++ and run thread
 * by thread on the CPU in the order the kernel's barriers impose, with the product's own host-side planning.  Chunks that do not take
 * the half-height slots run the whole-pair slots as the kernel does.  Not part of the product. */
#define B200_KERNELS_ON_CPU
#include "cuda_on_cpu.h"
#include "../../include/b200iop.h"
#include "../../ansel_b200/csrc/nlm.cu"
#include <vector>

extern "C" int emul_nlm_pipe2_chunks = 0; /* chunks the last calls ran through the half-height slots */

template <bool NORM1, bool PROFILED, bool DIVC> static void run_chunks(const grp_args_t &a, int n_chunks)
{
  using cfg = pipe_cfg<0>;
  constexpr int R = 1, NT = cfg::NT, ACC_T = cfg::ACC_T, WP = cfg::WP;
  std::vector<float> smem((size_t)a.wrows * 3 * WP + (size_t)2 * PIPE_SLOTS * a.splane + a.n_patches);
  std::vector<grp_strip_t<cfg::KP, cfg::L, cfg::IL>> st(ACC_T);
  float *const W = smem.data(), *const S = W + a.wrows * 3 * WP;
  int *const shifts = reinterpret_cast<int *>(S + 2 * PIPE_SLOTS * a.splane);
  const int npairs = (a.n_patches + 1) / 2;
  for(int b = 0; b < n_chunks; b++)
  {
    for(auto &v : smem) v = __builtin_nanf(""); /* whatever a phase reads must have been written by an earlier one */
    const chunk_t c = chunk_of(a, b);
    if(pipe2_takes(a, c, R))
    { /* per patch pair, upper then lower half: phase A of the 96 scan threads (their walks carry over), phase B1 of the 32 lanes of
         warp 3, phase B2 of the accumulating half that owns those rows */
      emul_nlm_pipe2_chunks++;
      for(int t = 0; t < NT; t++) pipe2_fill<WP, NT>(a, c, W, t);
      for(int p = 0; p < a.n_patches; p++) shifts[p] = pipe2_shift<WP>(a, p);
      f2 *const P = pipe2_slots(smem.data(), a.wrows, WP);
      for(int t = 0; t < ACC_T; t++)
      {
        pipe2_own_init<WP>(a, c, W, st[t], t);
        st[t].sofs0 -= (t / PIPE2_ACC_HALF) * PIPE2_HROWS * GRP_SP;
      }
      std::vector<pipe2_colwalk_t<WP, NORM1>> walk(PIPE2_A_T);
      for(int q = 0; q < npairs; q++)
      {
        for(int t = 1; t < PIPE2_A_T && t < c.ncols; t++) walk[t].init(a, c, W, 2 * q, t);
        for(int hh = 0; hh < 2; hh++)
        {
          f2 *const Sh = P + ((2 * q + hh) % PIPE2_SLOTS) * PIPE2_HSP;
          for(int t = 1; t < PIPE2_A_T && t < c.ncols; t++)
          {
            if(hh == 0)
              walk[t].template half<0>(a, Sh + t);
            else
              walk[t].template half<(PIPE2_HROWS % 3)>(a, Sh + t);
          }
          for(int l = 0; l < 32; l++) pipe2_b1_rows<R>(c, Sh, l);
          const bool both = 2 * q + 1 < a.n_patches;
          for(int t = hh * PIPE2_ACC_HALF; t < (hh + 1) * PIPE2_ACC_HALF; t++)
            pipe2_accumulate<WP, PROFILED, DIVC>(a, W, Sh, shifts[2 * q], shifts[both ? 2 * q + 1 : 2 * q], both, st[t]);
        }
      }
      for(int t = 0; t < ACC_T; t++) grp_finish(a, c, st[t], t, (t / PIPE2_ACC_HALF) * PIPE2_HROWS);
      continue;
    }
    /* the whole-pair slots, unchanged */
    const int half = (c.ch + 1) / 2;
    for(int t = 0; t < NT; t++) grp_fill<WP, NT>(a, c, W, t);
    for(int p = 0; p < a.n_patches; p++) shifts[p] = grp_shift<WP>(a, p);
    for(int t = 0; t < ACC_T; t++) grp_own_init<WP>(a, c, W, st[t], t);
    for(int q = 0; q < npairs; q++)
    {
      const int slot = q % PIPE_SLOTS;
      float *const Sa = S + (2 * slot) * a.splane, *const Sb = Sa + a.splane;
      for(int t = 0; t < PIPE_SCAN_GROUP; t++)
        if(t < c.ncols) grp_scan_column<WP, R, NORM1>(a, c, W, Sa, Sb, 2 * q, t);
      for(int t = 0; t < ACC_T; t++) pipe_b1<R>(a, c, Sa, 2 * q, pipe_b1_task(t, half), half);
      for(int t = 0; t < ACC_T; t++)
      {
        if(c.interior)
        {
          grp_accumulate_pairs<WP, PROFILED, DIVC>(a, W + shifts[2 * q], Sa, st[t]);
          if(2 * q + 1 < a.n_patches) grp_accumulate_pairs<WP, PROFILED, DIVC>(a, W + shifts[2 * q + 1], Sb, st[t]);
        }
        else
        {
          grp_accumulate_edge<WP, PROFILED, DIVC>(a, c, W, Sa, st[t], 2 * q);
          grp_accumulate_edge<WP, PROFILED, DIVC>(a, c, W, Sb, st[t], 2 * q + 1);
        }
      }
    }
    for(int t = 0; t < ACC_T; t++) grp_finish(a, c, st[t], t);
  }
}

/* same arguments as b200_nlmeans_denoise_dev on host buffers, patch radius 1; smem_bytes = what an SM offers, ieee_div: the plain
 * division instead of Markstein's sequence.  Returns 1, or 0 where the pipelined kernel's half-height configuration does not take the
 * frame (the launcher then runs another kernel). */
extern "C" int emul_nlmeans_pipe2(const float *in, float *out, int width, int height, float scattering, float scale, float luma, float chroma,
                                  float center_weight, float sharpness, int search_radius, int decimate, const float *norm, int smem_bytes, int ieee_div)
{
  _mm_setcsr(_mm_getcsr() | 0x8040u);
  int n_patches = (2 * search_radius + 1) * (2 * search_radius + 1);
  if(decimate) n_patches = (n_patches + 1) / 2;
  std::vector<patch_t> patches(n_patches);
  const int shift_max = grp_define_patches(patches.data(), search_radius, scale, scattering, decimate);
  const float weight[4] = { luma, chroma, chroma, 1.0f }, invert[4] = { 1.0f - luma, 1.0f - chroma, 1.0f - chroma, 0.0f };
  grp_args_t g;
  g.in = (const float4 *)in;
  g.out = (float4 *)out;
  g.patches = patches.data();
  if(!grp_plan(g, n_patches, width, height, 1, center_weight, sharpness, norm, weight, invert, (luma == 1.0 && chroma == 1.0) ? 1 : 0, shift_max,
               smem_bytes, GRP_MAXG)
     || !grp_pipe_fits(g, smem_bytes, pipe_cfg<0>::WP))
    return 0;
  const int n = ((height + g.chk_h - 1) / g.chk_h) * g.n_cl;
  const bool profiled = !(center_weight < 0), norm1 = norm[0] == 1.0f && norm[1] == 1.0f && norm[2] == 1.0f;
  const bool divc = grp_division_by_constant(g) && !ieee_div;
  if(!profiled)
    norm1 ? run_chunks<true, false, false>(g, n) : run_chunks<false, false, false>(g, n);
  else if(divc)
    norm1 ? run_chunks<true, true, true>(g, n) : run_chunks<false, true, true>(g, n);
  else
    norm1 ? run_chunks<true, true, false>(g, n) : run_chunks<false, true, false>(g, n);
  return 1;
}
