/* Test infrastructure: the phases of the non-local-means group kernel (ansel_b200/csrc/nlm_group.cuh) compiled with g++
 * and run thread by thread on the CPU, phase after phase as the kernel's barriers order them, with the product's own
 * host-side planning (grp_plan, grp_define_patches).  Not part of the product. */
#define B200_KERNELS_ON_CPU
#include "cuda_on_cpu.h"
#include "../../include/b200iop.h"
#include "../../ansel_b200/csrc/nlm.cu"
#include <vector>

template <int R, int WP, bool NORM1, bool PROFILED, bool DIVC, int KP> static void run_chunks(const grp_args_t &a, int n_chunks)
{
  std::vector<float> smem((size_t)a.wrows * 3 * WP + (size_t)a.G * a.splane + GRP_MAXG);
  std::vector<grp_thread_t<KP>> st(GRP_NT);
  float *const W = smem.data(), *const S = W + a.wrows * 3 * WP;
  int *const shifts = reinterpret_cast<int *>(S + a.G * a.splane);
  for(int b = 0; b < n_chunks; b++)
  {
    for(auto &v : smem) v = __builtin_nanf(""); // whatever a phase reads must have been written by an earlier one
    const chunk_t c = chunk_of(a, b);
    for(int t = 0; t < GRP_NT; t++) grp_fill<WP>(a, c, W, t);
    for(int t = 0; t < GRP_NT; t++) grp_own_init<WP>(a, c, W, st[t], t);
    for(int p0 = 0; p0 < a.n_patches; p0 += a.G)
    {
      for(int t = 0; t < GRP_NT; t++) grp_phase_a<WP, R, NORM1>(a, c, W, S, shifts, p0, t);
      for(int t = 0; t < GRP_NT; t++) grp_phase_b1<R>(a, c, S, p0, t);
      for(int t = 0; t < GRP_NT; t++) grp_phase_b2<WP, PROFILED, DIVC, KP>(a, c, W, S, shifts, st[t], p0, t);
    }
    for(int t = 0; t < GRP_NT; t++) grp_finish(a, c, st[t], t);
  }
}

/* the pipelined kernel's order of work: per patch pair, scan group (phase A, then phase B1) into its slot of the ring, then the 256
 * accumulating threads; what the emulation cannot see is the barrier protocol between them */
extern "C" int emul_nlm_halves_chunks = 0; /* chunks the last calls ran through the half-height slots (the tests check that some did) */
template <int R, bool NORM1, bool PROFILED, bool DIVC, int CFG> static void run_pipe_chunks(const grp_args_t &a, int n_chunks)
{
  constexpr int PIPE_NT = pipe_cfg<CFG>::NT, PIPE_ACC_T = pipe_cfg<CFG>::ACC_T, WP = pipe_cfg<CFG>::WP;
  std::vector<float> smem((size_t)a.wrows * 3 * WP + (size_t)2 * PIPE_SLOTS * a.splane + a.n_patches);
  std::vector<grp_strip_t<pipe_cfg<CFG>::KP, pipe_cfg<CFG>::L, pipe_cfg<CFG>::IL>> st(PIPE_ACC_T);
  float *const W = smem.data(), *const S = W + a.wrows * 3 * WP;
  int *const shifts = reinterpret_cast<int *>(S + 2 * PIPE_SLOTS * a.splane);
  const int npairs = (a.n_patches + 1) / 2;
  for(int b = 0; b < n_chunks; b++)
  {
    for(auto &v : smem) v = __builtin_nanf("");
    const chunk_t c = chunk_of(a, b);
    const int half = (c.ch + 1) / 2;
    for(int t = 0; t < PIPE_NT; t++) grp_fill<WP, PIPE_NT>(a, c, W, t);
    for(int t = 0; t < PIPE_NT; t++)
      for(int p = t; p < a.n_patches; p += PIPE_NT) shifts[p] = grp_shift<WP>(a, p);
    for(int t = 0; t < PIPE_ACC_T; t++) grp_own_init<WP>(a, c, W, st[t], t);
    if(pipe_cfg<CFG>::HALVES && pipe2_takes(a, c, R))
    { /* the half-height slots: per patch pair, upper then lower half: phase A of the 96 scan threads (their walks carry over), phase B1 of the
         32 lanes of warp 3, phase B2 of the accumulating half that owns those rows */
      if constexpr(R == 1)
      {
        emul_nlm_halves_chunks++;
        for(int t = 0; t < PIPE_ACC_T; t++) st[t].sofs0 -= (t / PIPE2_ACC_HALF) * PIPE2_HROWS * GRP_SP;
        std::vector<grp_colwalk_t<WP, R, NORM1>> walk(PIPE2_A_T);
        for(int q = 0; q < npairs; q++)
        {
          for(int t = 1; t < PIPE2_A_T && t < c.ncols; t++) walk[t].init(a, c, W, 2 * q, t);
          for(int hh = 0; hh < 2; hh++)
          {
            const int slot = (2 * q + hh) % PIPE2_SLOTS;
            float *const Sh = S + slot * (2 * PIPE2_HSP);
            for(int t = 0; t < PIPE2_A_T; t++)
            {
              float *const Sa = Sh + t, *const Sb = Sa + PIPE2_HSP;
              if(t >= 1 && t < c.ncols)
              {
                if(hh == 0)
                  walk[t].template half<0>(a, Sa, Sb);
                else
                  walk[t].template half<(PIPE2_HROWS % 3)>(a, Sa, Sb);
              }
              else if(t == 0)
                for(int rr = 0; rr < PIPE2_HROWS; rr++) Sa[rr * GRP_SP] = Sb[rr * GRP_SP] = 0.0f;
            }
            for(int l = 0; l < 32; l++) pipe2_b1<R>(a, c, Sh, 2 * q, l);
            for(int t = hh * PIPE2_ACC_HALF; t < (hh + 1) * PIPE2_ACC_HALF; t++)
            {
              grp_accumulate_pairs<WP, PROFILED, DIVC>(a, W + shifts[2 * q], Sh, st[t]);
              if(2 * q + 1 < a.n_patches) grp_accumulate_pairs<WP, PROFILED, DIVC>(a, W + shifts[2 * q + 1], Sh + PIPE2_HSP, st[t]);
            }
          }
        }
        for(int t = 0; t < PIPE_ACC_T; t++) grp_finish(a, c, st[t], t, (t / PIPE2_ACC_HALF) * PIPE2_HROWS);
      }
      continue;
    }
    for(int q = 0; q < npairs; q++)
    {
      const int slot = q % PIPE_SLOTS;
      float *const Sa = S + (2 * slot) * a.splane, *const Sb = Sa + a.splane;
      for(int t = 0; t < PIPE_SCAN_GROUP; t++)
        if(t < c.ncols) grp_scan_column<WP, R, NORM1>(a, c, W, Sa, Sb, 2 * q, t);
      for(int t = 0; t < PIPE_ACC_T; t++) pipe_b1<R>(a, c, Sa, 2 * q, pipe_b1_task(t, half), half);
      for(int t = 0; t < PIPE_ACC_T; t++)
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
    for(int t = 0; t < PIPE_ACC_T; t++) grp_finish(a, c, st[t], t);
  }
}
template <int R, int CFG> static void run_pipe(const grp_args_t &a, int n, bool norm1, bool profiled, bool divc)
{
  if(!profiled)
    return norm1 ? run_pipe_chunks<R, true, false, false, CFG>(a, n) : run_pipe_chunks<R, false, false, false, CFG>(a, n);
  if(divc) return norm1 ? run_pipe_chunks<R, true, true, true, CFG>(a, n) : run_pipe_chunks<R, false, true, true, CFG>(a, n);
  return norm1 ? run_pipe_chunks<R, true, true, false, CFG>(a, n) : run_pipe_chunks<R, false, true, false, CFG>(a, n);
}

template <int R, int WP, int KP> static void run_rk(const grp_args_t &a, int n, bool norm1, bool profiled, bool divc)
{
  if(!profiled)
    return norm1 ? run_chunks<R, WP, true, false, false, KP>(a, n) : run_chunks<R, WP, false, false, false, KP>(a, n);
  if(divc) return norm1 ? run_chunks<R, WP, true, true, true, KP>(a, n) : run_chunks<R, WP, false, true, true, KP>(a, n);
  return norm1 ? run_chunks<R, WP, true, true, false, KP>(a, n) : run_chunks<R, WP, false, true, false, KP>(a, n);
}
template <int R> static void run_r(const grp_args_t &a, int n, bool norm1, bool profiled, bool divc)
{
  const bool tall = grp_pairs_per_thread(a) > GRP_KP_MIN;
  if(a.wp == GRP_WP_NARROW)
    return tall ? run_rk<R, GRP_WP_NARROW, GRP_KP_MAX>(a, n, norm1, profiled, divc) : run_rk<R, GRP_WP_NARROW, GRP_KP_MIN>(a, n, norm1, profiled, divc);
  return tall ? run_rk<R, GRP_WP_WIDE, GRP_KP_MAX>(a, n, norm1, profiled, divc) : run_rk<R, GRP_WP_WIDE, GRP_KP_MIN>(a, n, norm1, profiled, divc);
}

/* same arguments as b200_nlmeans_denoise_dev on host buffers; smem_bytes = what an SM offers, g_cap = patches in flight at most,
 * ieee_div: the plain division instead of Markstein's sequence; pipe: the pipelined kernel's order of work.  Returns the patches in
 * flight, 0 = the plan does not fit. */
extern "C" int emul_nlmeans_group(const float *in, float *out, int width, int height, float scattering, float scale, float luma, float chroma,
                                  float center_weight, float sharpness, int radius, int search_radius, int decimate, const float *norm,
                                  int smem_bytes, int g_cap, int ieee_div, int pipe)
{
  _mm_setcsr(_mm_getcsr() | 0x8040u);
  int n_patches = (2 * search_radius + 1) * (2 * search_radius + 1);
  if(decimate) n_patches = (n_patches + 1) / 2;
  std::vector<patch_t> patches(n_patches);
  const int shift_max = grp_define_patches(patches.data(), search_radius, scale, scattering, decimate);
  const float weight[4] = { luma, chroma, chroma, 1.0f }, invert[4] = { 1.0f - luma, 1.0f - chroma, 1.0f - chroma, 0.0f };
  const int pw = 2 * radius + 1;
  (void)pw;
  grp_args_t g;
  g.in = (const float4 *)in;
  g.out = (float4 *)out;
  g.patches = patches.data();
  if(!grp_plan(g, n_patches, width, height, radius, center_weight, sharpness, norm, weight, invert, (luma == 1.0 && chroma == 1.0) ? 1 : 0,
               shift_max, smem_bytes, g_cap))
    return 0;
  const int n_ct = (height + g.chk_h - 1) / g.chk_h;
  const bool profiled = !(center_weight < 0), norm1 = norm[0] == 1.0f && norm[1] == 1.0f && norm[2] == 1.0f;
  const bool divc = grp_division_by_constant(g) && !ieee_div;
  if(pipe)
  { /* returns -1 where the pipelined kernel does not take the frame (the launcher then uses the group kernel) */
    if(!grp_pipe_fits(g, smem_bytes, pipe_cfg<0>::WP)) return -1;
    const int n = n_ct * g.n_cl; /* pipe: 1 = half-height slots where a chunk takes them, 2 = whole-pair slots everywhere */
    if(pipe == 2)
      radius == 1 ? run_pipe<1, 1>(g, n, norm1, profiled, divc) : run_pipe<2, 1>(g, n, norm1, profiled, divc);
    else
      radius == 1 ? run_pipe<1, 0>(g, n, norm1, profiled, divc) : run_pipe<2, 0>(g, n, norm1, profiled, divc);
    return g.G;
  }
  if(radius == 1)
    run_r<1>(g, n_ct * g.n_cl, norm1, profiled, divc);
  else
    run_r<2>(g, n_ct * g.n_cl, norm1, profiled, divc);
  return g.G;
}

/* Which kernel, and which template instance of it, b200_nlmeans_denoise_dev launches for these arguments on a device offering smem_bytes of
 * shared memory per block, and how many chunks take the pipelined kernel's half-height slots.  Only the host-side planning runs (the
 * product's grp_define_patches, grp_plan, grp_pipe_fits, chunk_of, pipe2_takes); no kernel phase.  The development switches are read from the
 * environment as the launcher reads them.  route[]: kernel (0 = nlm_chunks_kernel, 1 = nlm_chunks_win_kernel, 2 = nlm_pipe_kernel,
 * 3 = nlm_group_kernel), R, WP, KP, N1, PR, DC, CFG, chunks on the half-height slots, chunks, patches in flight (group kernel). */
extern "C" void emul_nlm_route(int width, int height, float scattering, float scale, float luma, float chroma, float center_weight, float sharpness,
                               int radius, int search_radius, int decimate, const float *norm, int smem_bytes, int *route)
{
  for(int i = 0; i < 11; i++) route[i] = 0;
  int n_patches = (2 * search_radius + 1) * (2 * search_radius + 1);
  if(decimate) n_patches = (n_patches + 1) / 2;
  std::vector<patch_t> patches(n_patches);
  const int shift_max = grp_define_patches(patches.data(), search_radius, scale, scattering, decimate);
  const float weight[4] = { luma, chroma, chroma, 1.0f }, invert[4] = { 1.0f - luma, 1.0f - chroma, 1.0f - chroma, 0.0f };
  const int chk_h = slice_height(height), chk_w = slice_width(width);
  const int n_chunks = ((height + chk_h - 1) / chk_h) * ((width + chk_w - 1) / chk_w);
  route[9] = n_chunks;
  route[1] = radius;
  /* nlmeans_denoise_dev, nlm.cu:903-922 */
  const bool chunks_forced = getenv("B200_NLM_CHUNKS") || getenv("B200_NLM_WINDOW");
  grp_args_t g;
  g.patches = patches.data();
  int g_cap = GRP_MAXG;
  if(const char *e = getenv("B200_NLM_G")) g_cap = atoi(e);
  if(chunks_forced || !grp_plan(g, n_patches, width, height, radius, center_weight, sharpness, norm, weight, invert, (luma == 1.0 && chroma == 1.0) ? 1 : 0,
                                shift_max, smem_bytes, g_cap))
  {
    const int rows_e = chk_h + 2 * radius + 1, cols_w = chk_w + 2 * radius + 2;
    const long long win_bytes = 2LL * rows_e * cols_w * 16 + 2LL * chk_h * (cols_w | 1) * 4;
    route[0] = getenv("B200_NLM_WINDOW") && win_bytes <= smem_bytes ? 1 : 0;
    return;
  }
  /* launch_group, nlm.cu:795-824 (behind #ifndef B200_KERNELS_ON_CPU there, so restated here) */
  const bool profiled = !(center_weight < 0), norm1 = norm[0] == 1.0f && norm[1] == 1.0f && norm[2] == 1.0f;
  const bool divc = grp_division_by_constant(g) && !getenv("B200_NLM_IEEE_DIV");
  route[4] = norm1;
  route[5] = profiled;
  route[6] = profiled && divc;
  route[10] = g.G;
  if(grp_pipe_fits(g, smem_bytes, pipe_cfg<0>::WP) && !getenv("B200_NLM_NO_PIPE"))
  {
    const int cfg = getenv("B200_NLM_WHOLE_SLOTS") ? 1 : 0;
    route[0] = 2;
    route[2] = cfg ? pipe_cfg<1>::WP : pipe_cfg<0>::WP;
    route[3] = cfg ? pipe_cfg<1>::KP : pipe_cfg<0>::KP;
    route[7] = cfg;
    if(cfg == 0 && radius == 1) /* the kernel's own test, nlm_pipe_kernel in nlm_group.cuh */
      for(int b = 0; b < n_chunks; b++) route[8] += pipe2_takes(g, chunk_of(g, b), radius) ? 1 : 0;
    return;
  }
  route[0] = 3;
  route[2] = g.wp;
  route[3] = grp_pairs_per_thread(g) > GRP_KP_MIN ? GRP_KP_MAX : GRP_KP_MIN;
}
