// Non-local means, the group kernel: the pixels a chunk can touch live in shared memory once, G patch offsets are in
// flight at a time, and every thread works in every phase.  Included by nlm.cu inside its anonymous namespace.
//
// Reference: src/pixel/nlmeans_core.c nlmeans_denoise :315-532 (what fixes the float rounding order: the column sums
// run down the rows of a chunk :424-483 from init_column_sums :214-264, the distortion runs along each row :384-409,
// the output accumulates patch after patch :396-420).  Those three orders are sequential per (patch, column),
// per (patch, row) and per pixel -- and nothing else is: different patches have independent column sums and
// distortions.  So per group of G patches
//   phase A   thread = (two patches, column)  column sums down the rows, squared differences formed on the fly from the
//                                             window, the 2*radius+1 rows of a patch kept in registers -> S[g][row][col]
//   phase B1  thread = (patch, two rows)      running distortion along the rows, in place in S, the last 2*radius+1
//                                             column sums of a row kept in registers
//   phase B2  thread = its pixels (in pairs)  weights and accumulation in patch order, sums in registers for all patches
// with one __syncthreads between phases.  The inner arithmetic works on pairs of floats (packed_f32.cuh: two scalar
// instructions per pair on sm_90): two patches of one column in phase A, two rows in phase B1, two vertically
// adjacent pixels in phase B2.  No multiply may be contracted with the add it feeds: only Markstein's division uses a
// fused multiply-add.  The division by the constant 1 + center_weight is Markstein's
// sequence (q0 = x*rcp, r = fma(-q0, d, x), q = fma(r, rcp, q0)): correctly rounded for every x when rcp = RN(1/d) and
// nothing underflows (Markstein 1990; Brisebarre, Muller, Raina 2004, section 1), i.e. identical to the reference's
// divss; the host restricts it to parameter ranges where an underflowing x cannot change the weight
// (grp_division_by_constant in nlm.cu).
//
// Shared memory: the window as rows of three channel lines of WP floats (every offset between a pixel, its
// channels and the row below is a compile-time constant), then G planes of column sums with rows of GRP_SP floats
// (odd: a warp whose lanes are rows hits 32 banks).
//
// Chunks whose rows or columns leave the frame for some patch take the scalar paths below (validity tests per row,
// per pixel); they restate the same formulas and are what the packed paths are checked against.

constexpr int GRP_NT = 384;   // 64x72 chunk = 2304 pixel pairs = 6 per thread
constexpr int GRP_MAXG = 8;
constexpr int GRP_KP_MAX = (((MAX_CH + 1) / 2) * MAX_CW + GRP_NT - 1) / GRP_NT; // pixel pairs a thread owns: 7 at most,
constexpr int GRP_KP_MIN = 6;                                                   // 6 for chunks of up to 64 rows (a template parameter: registers)
// WP (template parameter): floats of one channel line of the window, >= chunk + 2 * (radius + largest shift) columns; 96 holds every
// unscattered search radius up to 10, 128 shifts up to 26.  One window row is 3 * WP floats.
constexpr int GRP_WP_NARROW = 96, GRP_WP_WIDE = 128;
constexpr int GRP_SP = MAX_CW + 2 * 2 + 1;     // 77: columns of column sums at radius <= 2, odd

struct grp_args_t
{
  const float4 *in;
  float4 *out;
  const patch_t *patches;
  int n_patches, width, height, chk_h, chk_w, n_cl, radius;
  float center_weight, sharpness, cp_norm, div_d, div_rcp;
  float norm[4], weight[4], invert[4];
  int skip_blend;
  int hs;           // largest |row shift| or |column shift| of the patch list
  int wcols, wrows; // window: chunk + radius + hs on every side (+1 row)
  int wp;           // floats of one channel line of the window (the kernel's WP): GRP_WP_NARROW or GRP_WP_WIDE, >= wcols
  int splane;       // floats of one plane of column sums / distortions: (chk_h + 1) * GRP_SP
  int G;            // patches in flight, even
};

struct chunk_t
{
  int top, bot, left, right, ch, cw;
  int cbase, ncols; // image column of S[.][0] (a column of zeros), columns of S
  int wr0, wc0;     // image row / column of window entry (0, 0)
  bool interior;    // no patch leaves the frame anywhere in this chunk's reach: every patch is valid, its rows regular, it covers
                    // the chunk, and every column but S[.][0] is live -- the packed paths without a geometry test
};

__device__ __forceinline__ chunk_t chunk_of(const grp_args_t &a, int block)
{
  chunk_t c;
  const int it = block / a.n_cl, il = block - it * a.n_cl;
  c.top = it * a.chk_h;
  c.left = il * a.chk_w;
  c.bot = min(c.top + a.chk_h, a.height);
  c.right = min(c.left + a.chk_w, a.width);
  c.ch = c.bot - c.top;
  c.cw = c.right - c.left;
  c.cbase = c.left - a.radius - 1;
  c.ncols = c.cw + 2 * a.radius + 1;
  c.wr0 = c.top - a.radius - a.hs;
  c.wc0 = c.left - a.radius - a.hs;
  const int reach = a.radius + a.hs;
  c.interior = c.top - reach >= 0 && c.bot + reach <= a.height && c.left - reach >= 0 && c.right + reach <= a.width
               && c.cw >= 2 * a.radius + 1;
  return c;
}

// patch geometry of nlmeans_denoise() :345-372 for one chunk, plus the rows on which both pixels of a pair exist
struct pgeo_t
{
  int srow, scol, row_min, row_max, col_min, col_max, pcol_min, pcol_max, lo, hi;
  bool valid;
};
__device__ __forceinline__ pgeo_t patch_geo_grp(const grp_args_t &a, const chunk_t &c, int p)
{
  pgeo_t g;
  g.valid = p < a.n_patches;
  if(!g.valid) return g;
  const int radius = a.radius, width = a.width, height = a.height;
  g.srow = a.patches[p].rows;
  g.scol = a.patches[p].cols;
  g.row_min = max(c.top, max(0, -g.srow));
  g.row_max = min(c.bot, height - max(0, g.srow));
  g.valid = g.row_min < g.row_max;
  g.col_min = max(c.left, -g.scol);
  g.col_max = min(c.right, width - g.scol);
  g.pcol_min = c.left - min(radius, min(c.left, c.left + g.scol));
  g.pcol_max = c.right + min(radius, min(width - c.right, width - (c.right + g.scol)));
  g.lo = max(0, -g.srow);                // rows rho with rho and rho + srow inside the frame: lo <= rho < hi
  g.hi = height - max(0, g.srow);
  return g;
}
// every row the column sums of this chunk read exists for this patch (no top / bottom edge of the frame in reach)
__device__ __forceinline__ bool rows_regular(const grp_args_t &a, const chunk_t &c, const pgeo_t &g)
{
  return c.top - a.radius >= g.lo && c.bot - 1 + a.radius < g.hi;
}
// the patch covers the whole chunk: no pixel of it is skipped (:351-366)
__device__ __forceinline__ bool covers_chunk(const chunk_t &c, const pgeo_t &g)
{
  return g.row_min == c.top && g.row_max == c.bot && g.col_min == c.left && g.col_max == c.right;
}

template <bool NORM1> __device__ __forceinline__ float pd3(float e0, float e1, float e2, float n0, float n1, float n2)
{ // pixel_difference(), :156-165, from the squares
  return NORM1 ? (e0 + e1) + e2 : (e0 * n0 + e1 * n1) + e2 * n2;
}

// ---- the window: every pixel this chunk reads, for every patch, once ---------------------------------------------
template <int WP, int NTHREADS = GRP_NT> __device__ __forceinline__ void grp_fill(const grp_args_t &a, const chunk_t &c, float *W, int tid)
{
  const int n = a.wrows * a.wcols;
  for(int idx = tid; idx < n; idx += NTHREADS)
  {
    const int wi = idx / a.wcols, wj = idx - wi * a.wcols;
    const int r = c.wr0 + wi, col = c.wc0 + wj;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if(r >= 0 && r < a.height && col >= 0 && col < a.width) v = __ldg(a.in + (size_t)r * a.width + col);
    float *const w = W + wi * (3 * WP) + wj;
    w[0] = v.x;
    w[WP] = v.y;
    w[2 * WP] = v.z;
  }
}

// ---- phase A -----------------------------------------------------------------------------------------------------
// one patch, one column, every edge case: rows that do not exist for the patch count as zero squares, which is what
// the three branches of :424-483 and the row range of init_column_sums() :232-233 amount to (nlm.cu phase_a).
template <int WP, int R, bool NORM1>
__device__ void grp_colsum_one(const grp_args_t &a, const chunk_t &c, const float *W, float *Sg, const pgeo_t &g, int k)
{
  const int col = c.cbase + k;
  float *sp = Sg + (g.row_min - c.top) * GRP_SP + k;
  if(!(col >= g.pcol_min && col < g.pcol_max))
  {
    for(int row = g.row_min; row < g.row_max; row++, sp += GRP_SP) *sp = 0.0f;
    return;
  }
  const float n0 = a.norm[0], n1 = a.norm[1], n2 = a.norm[2];
  const float *x = W + (g.row_min - R - c.wr0) * (3 * WP) + (col - c.wc0);
  const float *y = x + g.srow * (3 * WP) + g.scol;
  int rho = g.row_min - R;
  float ring[2 * R + 1][3];
  float cs = 0.0f;
#pragma unroll
  for(int i = 0; i < 2 * R + 1; i++, x += (3 * WP), y += (3 * WP), rho++)
  {
    float e0 = 0.0f, e1 = 0.0f, e2 = 0.0f;
    if(rho >= g.lo && rho < g.hi)
    {
      const float d0 = x[0] - y[0], d1 = x[WP] - y[WP], d2 = x[2 * WP] - y[2 * WP];
      e0 = d0 * d0;
      e1 = d1 * d1;
      e2 = d2 * d2;
      cs += pd3<NORM1>(e0, e1, e2, n0, n1, n2);
    }
    ring[i][0] = e0;
    ring[i][1] = e1;
    ring[i][2] = e2;
  }
  for(int row = g.row_min; row < g.row_max;)
  {
#pragma unroll
    for(int s = 0; s < 2 * R + 1; s++)
    {
      if(row < g.row_max)
      {
        *sp = cs;
        sp += GRP_SP;
        if(row + 1 < g.row_max)
        {
          float e0 = 0.0f, e1 = 0.0f, e2 = 0.0f;
          if(rho >= g.lo && rho < g.hi)
          {
            const float d0 = x[0] - y[0], d1 = x[WP] - y[WP], d2 = x[2 * WP] - y[2 * WP];
            e0 = d0 * d0;
            e1 = d1 * d1;
            e2 = d2 * d2;
          }
          cs += pd3<NORM1>(e0 - ring[s][0], e1 - ring[s][1], e2 - ring[s][2], n0, n1, n2); // diff_of_pixels_diff(), :168-180
          ring[s][0] = e0;
          ring[s][1] = e1;
          ring[s][2] = e2;
        }
        x += (3 * WP);
        y += (3 * WP);
        rho++;
        row++;
      }
    }
  }
}

// one window row as phase A reads it for two patches: the pixel, and the pixels at the two patch offsets
struct grp_row9_t
{
  float x0, x1, x2, a0, a1, a2, b0, b1, b2;
};
template <int WP> __device__ __forceinline__ grp_row9_t grp_load_row(const float *x, const float *ya, const float *yb)
{
  grp_row9_t r;
  r.x0 = x[0];
  r.x1 = x[WP];
  r.x2 = x[2 * WP];
  r.a0 = ya[0];
  r.a1 = ya[WP];
  r.a2 = ya[2 * WP];
  r.b0 = yb[0];
  r.b1 = yb[WP];
  r.b2 = yb[2 * WP];
  return r;
}
// its squared differences: lane x = patch a, lane y = patch b
__device__ __forceinline__ void grp_squares2(const grp_row9_t &r, f2 &e0, f2 &e1, f2 &e2)
{
  const f2 d0 = sub2(mk2(r.x0, r.x0), mk2(r.a0, r.b0));
  const f2 d1 = sub2(mk2(r.x1, r.x1), mk2(r.a1, r.b1));
  const f2 d2 = sub2(mk2(r.x2, r.x2), mk2(r.a2, r.b2));
  e0 = mk2(d0.x * d0.x, d0.y * d0.y);
  e1 = mk2(d1.x * d1.x, d1.y * d1.y);
  e2 = mk2(d2.x * d2.x, d2.y * d2.y);
}
template <bool NORM1> __device__ __forceinline__ f2 grp_pd2(f2 u0, f2 u1, f2 u2, f2 n0, f2 n1, f2 n2)
{
  if(NORM1) return add2(add2(u0, u1), u2);
  const f2 s0 = mul2(u0, n0), s1 = mul2(u1, n1), s2 = mul2(u2, n2);
  return mk2((s0.x + s1.x) + s2.x, (s0.y + s1.y) + s2.y);
}

// two patches of one column whose rows are all regular and whose column is live for both.  The running sum is the only thing a
// row hands to the next one: the nine window values of row r + 1 are fetched before row r is worked on, so their
// shared-memory latency runs under its arithmetic (the window has a spare row behind the last one read).
template <int WP, int R, bool NORM1>
__device__ void grp_colsum_pair(const grp_args_t &a, const chunk_t &c, const float *W, float *Sa, float *Sb, const pgeo_t &ga,
                                const pgeo_t &gb, int k)
{
  constexpr int RP = 3 * WP, N = 2 * R + 1;
  const int col = c.cbase + k;
  const f2 n0 = mk2(a.norm[0], a.norm[0]), n1 = mk2(a.norm[1], a.norm[1]), n2 = mk2(a.norm[2], a.norm[2]);
  const float *x = W + (c.top - R - c.wr0) * RP + (col - c.wc0);
  const float *ya = x + ga.srow * RP + ga.scol, *yb = x + gb.srow * RP + gb.scol;
  float *spa = Sa + k, *spb = Sb + k;
  f2 ring[N][3];
  f2 cs = mk2(0.0f, 0.0f);
  grp_row9_t nxt = grp_load_row<WP>(x, ya, yb);
#pragma unroll
  for(int i = 0; i < N; i++)
  {
    const grp_row9_t cur = nxt;
    nxt = grp_load_row<WP>(x + (i + 1) * RP, ya + (i + 1) * RP, yb + (i + 1) * RP);
    grp_squares2(cur, ring[i][0], ring[i][1], ring[i][2]);
    cs = add2(cs, grp_pd2<NORM1>(ring[i][0], ring[i][1], ring[i][2], n0, n1, n2));
  }
  x += N * RP;
  ya += N * RP;
  yb += N * RP;
  // rows top .. bot-1: store the sum, then slide it down by one row (the last row has no successor to slide to)
  int left = c.ch;
  for(; left > N; left -= N)
  {
#pragma unroll
    for(int s = 0; s < N; s++)
    {
      const grp_row9_t cur = nxt;
      nxt = grp_load_row<WP>(x + (s + 1) * RP, ya + (s + 1) * RP, yb + (s + 1) * RP);
      spa[s * GRP_SP] = cs.x;
      spb[s * GRP_SP] = cs.y;
      f2 e0, e1, e2;
      grp_squares2(cur, e0, e1, e2);
      cs = add2(cs, grp_pd2<NORM1>(sub2(e0, ring[s][0]), sub2(e1, ring[s][1]), sub2(e2, ring[s][2]), n0, n1, n2));
      ring[s][0] = e0;
      ring[s][1] = e1;
      ring[s][2] = e2;
    }
    x += N * RP;
    ya += N * RP;
    yb += N * RP;
    spa += N * GRP_SP;
    spb += N * GRP_SP;
  }
#pragma unroll
  for(int s = 0; s < N; s++)
  {
    if(s < left)
    {
      spa[s * GRP_SP] = cs.x;
      spb[s * GRP_SP] = cs.y;
      if(s + 1 < left)
      {
        const grp_row9_t cur = nxt;
        if(s + 2 < left) nxt = grp_load_row<WP>(x + (s + 1) * RP, ya + (s + 1) * RP, yb + (s + 1) * RP);
        f2 e0, e1, e2;
        grp_squares2(cur, e0, e1, e2);
        cs = add2(cs, grp_pd2<NORM1>(sub2(e0, ring[s][0]), sub2(e1, ring[s][1]), sub2(e2, ring[s][2]), n0, n1, n2));
      }
    }
  }
}

// the patches of a group as phase B2 wants them: their window shifts, in shared memory
template <int WP> __device__ __forceinline__ int grp_shift(const grp_args_t &a, int p) { return a.patches[p].rows * (3 * WP) + a.patches[p].cols; }

// phase A for one thread: column k (0 = the column of zeros) of patches pa and pa + 1 into the planes Sa, Sb
template <int WP, int R, bool NORM1>
__device__ __forceinline__ void grp_scan_column(const grp_args_t &a, const chunk_t &c, const float *W, float *Sa, float *Sb, int pa, int k)
{
  if(c.interior && pa + 1 < a.n_patches)
  {
    if(k == 0)
    { // the column of zeros left of the first live one (:228-231)
      for(int rr = 0; rr < c.ch; rr++) Sa[rr * GRP_SP] = Sb[rr * GRP_SP] = 0.0f;
    }
    else
    {
      pgeo_t ga, gb;
      ga.srow = a.patches[pa].rows;
      ga.scol = a.patches[pa].cols;
      gb.srow = a.patches[pa + 1].rows;
      gb.scol = a.patches[pa + 1].cols;
      grp_colsum_pair<WP, R, NORM1>(a, c, W, Sa, Sb, ga, gb, k);
    }
    return;
  }
  const pgeo_t ga = patch_geo_grp(a, c, pa), gb = patch_geo_grp(a, c, pa + 1);
  const int col = c.cbase + k;
  const bool la = ga.valid && col >= ga.pcol_min && col < ga.pcol_max, lb = gb.valid && col >= gb.pcol_min && col < gb.pcol_max;
  if(ga.valid && gb.valid && la && lb && rows_regular(a, c, ga) && rows_regular(a, c, gb))
    grp_colsum_pair<WP, R, NORM1>(a, c, W, Sa, Sb, ga, gb, k);
  else
  {
    if(ga.valid) grp_colsum_one<WP, R, NORM1>(a, c, W, Sa, ga, k);
    if(gb.valid) grp_colsum_one<WP, R, NORM1>(a, c, W, Sb, gb, k);
  }
}

template <int WP, int R, bool NORM1>
__device__ __forceinline__ void grp_phase_a(const grp_args_t &a, const chunk_t &c, const float *W, float *S, int *shifts, int p0, int tid)
{
  const int npairs = a.G / 2;
  if(tid < a.G) shifts[tid] = p0 + tid < a.n_patches ? grp_shift<WP>(a, p0 + tid) : 0;
  for(int t = tid; t < npairs * c.ncols; t += GRP_NT)
  {
    const int pi = t / c.ncols, k = t - pi * c.ncols;
    float *const Sa = S + (2 * pi) * a.splane;
    grp_scan_column<WP, R, NORM1>(a, c, W, Sa, Sa + a.splane, p0 + 2 * pi, k);
  }
}

// ---- phase B1: running distortion along each row (:384-387, 409), in place: D[col] lands in slot col - left ----------
// one row, every case
__device__ __forceinline__ void grp_row_one(float *Sr /* Sr[col] = column sum of `col` */, const pgeo_t &g, int radius)
{
  float distortion = 0.0f;
  for(int i = g.col_min - radius; i < min(g.col_min + radius, g.col_max); i++) distortion += Sr[i];
  for(int col = g.col_min; col < g.col_max; col++)
  {
    distortion += (Sr[col + radius] - Sr[col - radius - 1]);
    Sr[col - radius - 1] = distortion; // that slot is never read again
  }
}
// two rows (lane x: row, lane y: row + half) of a patch with at least 2*R+1 columns; the column sum leaving the window
// is the one read 2*R+1 steps earlier.  ZERO0: the column sum leaving at col_min is the column of zeros, taken as the constant
// instead of read (x - 0 is x for every x, and no stored sum is subnormal)
template <int R, bool ZERO0 = false> __device__ __forceinline__ void grp_row_pair(float *Sx, float *Sy, const pgeo_t &g)
{
  constexpr int N = 2 * R + 1;
  float *px = Sx + g.col_min - R - 1, *py = Sy + g.col_min - R - 1; // slot of D[col_min], column sum leaving at col_min
  f2 ring[N];
  f2 distortion = mk2(0.0f, 0.0f);
  ring[0] = ZERO0 ? mk2(0.0f, 0.0f) : mk2(px[0], py[0]);
#pragma unroll
  for(int i = 1; i < N; i++)
  {
    ring[i] = mk2(px[i], py[i]);
    distortion = add2(distortion, ring[i]);
  }
  // the column sums entering the window are fetched a block of N ahead of their use: only the running sum itself is a chain.
  // (The last fetch reads up to N floats behind the row's last column sum: the next row of the plane, or what follows the planes.)
  f2 nxt[N];
#pragma unroll
  for(int s = 0; s < N; s++) nxt[s] = mk2(px[s + N], py[s + N]);
  int left = g.col_max - g.col_min;
  for(; left >= N; left -= N)
  {
    f2 cur[N];
#pragma unroll
    for(int s = 0; s < N; s++) cur[s] = nxt[s];
#pragma unroll
    for(int s = 0; s < N; s++) nxt[s] = mk2(px[s + 2 * N], py[s + 2 * N]);
#pragma unroll
    for(int s = 0; s < N; s++)
    {
      distortion = add2(distortion, sub2(cur[s], ring[s]));
      ring[s] = cur[s];
      px[s] = distortion.x;
      py[s] = distortion.y;
    }
    px += N;
    py += N;
  }
#pragma unroll
  for(int s = 0; s < N; s++)
  {
    if(s < left)
    {
      distortion = add2(distortion, sub2(nxt[s], ring[s]));
      px[s] = distortion.x;
      py[s] = distortion.y;
    }
  }
}

// phase B1 for one thread: rows rr and rr + half of patch p, whose plane is Sp
template <int R> __device__ __forceinline__ void grp_scan_rows(const grp_args_t &a, const chunk_t &c, float *Sp, int p, int rr, int half)
{
  float *const Sx = Sp + rr * GRP_SP - c.cbase, *const Sy = Sx + half * GRP_SP;
  if(c.interior)
  {
    if(p >= a.n_patches) return;
    pgeo_t g;
    g.col_min = c.left;
    g.col_max = c.right;
    if(rr + half < c.ch)
      grp_row_pair<R>(Sx, Sy, g);
    else
      grp_row_one(Sx, g, R);
    return;
  }
  const pgeo_t g = patch_geo_grp(a, c, p);
  if(!g.valid || g.col_min >= g.col_max) return;
  const int rx = c.top + rr, ry = rx + half;
  const bool vx = rx >= g.row_min && rx < g.row_max, vy = ry >= g.row_min && ry < g.row_max;
  if(vx && vy && g.col_max - g.col_min >= 2 * R + 1)
    grp_row_pair<R>(Sx, Sy, g);
  else
  {
    if(vx) grp_row_one(Sx, g, R);
    if(vy) grp_row_one(Sy, g, R);
  }
}

template <int R> __device__ __forceinline__ void grp_phase_b1(const grp_args_t &a, const chunk_t &c, float *S, int p0, int tid)
{
  const int half = (c.ch + 1) / 2;
  for(int t = tid; t < a.G * half; t += GRP_NT)
  {
    const int gi = t / half, rr = t - gi * half;
    grp_scan_rows<R>(a, c, S + gi * a.splane, p0 + gi, rr, half);
  }
}

// ---- phase B2 --------------------------------------------------------------------------------------------------
// Two ways of dealing the pixel pairs of a chunk to the accumulating threads.  grp_thread_t: pair j = tid + k * NTHREADS in raster
// order (any chunk height, any thread count; the offsets of every pair live in registers).  grp_strip_t: a thread owns the pairs
// of ONE pair of rows at columns i, i + L, i + 2L, ...: the offsets of pair k are those of pair 0 plus k * L, immediates of the
// load instructions.  L = 8: a warp holds 8 lanes on each of 4 row pairs that lie 4 row pairs apart, 72 columns = 9 pairs per
// thread; with an odd window pitch (3 * WP) and the odd pitch of the planes the four row pairs of a warp start 8 banks apart:
// no bank conflicts in phase B2, whatever the patch shift.  L = 12: thread ta owns row pair ta / 12, 6 pairs per thread.
template <int KP_> struct grp_thread_t
{
  static constexpr int KP = KP_, IL = 1;
  float acc[KP][8]; // sums of the upper pixel (even slots) and of the lower pixel (odd slots): x x' y y' z z' w w'
  float ctr[KP][6]; // the pixels themselves: c0 c0' c1 c1' c2 c2'
  int wofs_[KP];    // window offset of the upper pixel (the chunk's first pixel for a pair that does not exist: harmless reads, never stored)
  int sofs_[KP];    // offset of its distortion in a plane of S
  unsigned upper;   // bit k: pair k exists
  unsigned lower;   // bit k: its lower pixel belongs to the chunk
  __device__ __forceinline__ int wofs(int k) const { return wofs_[k]; }
  __device__ __forceinline__ int sofs(int k) const { return sofs_[k]; }
};
template <int KP_, int L_, int IL_> struct grp_strip_t
{
  static constexpr int KP = KP_, L = L_, IL = IL_; // IL: pairs in flight in phase B2
  float acc[KP][8];
  float ctr[KP][6];
  int wofs0, sofs0; // of pair 0 (row pair 0 for a thread whose row pair is below the chunk: harmless reads, never stored)
  unsigned upper, lower;
  __device__ __forceinline__ int wofs(int k) const { return wofs0 + k * L; }
  __device__ __forceinline__ int sofs(int k) const { return sofs0 + k * L; }
};

template <int WP, int KP, int NTHREADS = GRP_NT>
__device__ __forceinline__ void grp_own_init(const grp_args_t &a, const chunk_t &c, const float *W, grp_thread_t<KP> &st, int tid)
{
  st.lower = st.upper = 0u;
#pragma unroll
  for(int k = 0; k < KP; k++)
  {
    const int j = tid + k * NTHREADS;
    const int pr = j / c.cw, pc = j - pr * c.cw;
#pragma unroll
    for(int i = 0; i < 8; i++) st.acc[k][i] = 0.0f;
    st.wofs_[k] = (c.top - c.wr0) * (3 * WP) + (c.left - c.wc0); // the chunk's first pixel: any patch shift stays inside the window
    st.sofs_[k] = 0;
    if(2 * pr < c.ch)
    {
      st.wofs_[k] = (c.top + 2 * pr - c.wr0) * (3 * WP) + (c.left + pc - c.wc0);
      st.sofs_[k] = 2 * pr * GRP_SP + pc;
      st.upper |= 1u << k;
      if(2 * pr + 1 < c.ch) st.lower |= 1u << k;
    }
    const float *const w = W + st.wofs_[k];
    st.ctr[k][0] = w[0];
    st.ctr[k][1] = w[(3 * WP)];
    st.ctr[k][2] = w[WP];
    st.ctr[k][3] = w[(3 * WP) + WP];
    st.ctr[k][4] = w[2 * WP];
    st.ctr[k][5] = w[(3 * WP) + 2 * WP];
  }
}
// row pair and first column of accumulating thread ta of a strip ownership
template <int L> __device__ __forceinline__ void grp_strip_of(int ta, int &pr, int &i)
{
  if(L == 8)
  {
    const int wa = ta >> 5, l = ta & 31;
    i = l & 7;
    pr = (wa & 3) + 4 * (l >> 3) + 16 * (wa >> 2);
  }
  else
  {
    pr = ta / L;
    i = ta - pr * L;
  }
}
template <int WP, int KP, int L, int IL>
__device__ __forceinline__ void grp_own_init(const grp_args_t &a, const chunk_t &c, const float *W, grp_strip_t<KP, L, IL> &st, int ta)
{
  int pr, i;
  grp_strip_of<L>(ta, pr, i);
  const bool rows = 2 * pr < c.ch;
  const int r0 = rows ? 2 * pr : 0;
  st.wofs0 = (c.top + r0 - c.wr0) * (3 * WP) + (c.left + i - c.wc0);
  st.sofs0 = r0 * GRP_SP + i;
  st.lower = st.upper = 0u;
#pragma unroll
  for(int k = 0; k < KP; k++)
  {
#pragma unroll
    for(int j = 0; j < 8; j++) st.acc[k][j] = 0.0f;
    if(rows && i + k * L < c.cw)
    {
      st.upper |= 1u << k;
      if(2 * pr + 1 < c.ch) st.lower |= 1u << k;
    }
    const float *const w = W + st.wofs(k);
    st.ctr[k][0] = w[0];
    st.ctr[k][1] = w[(3 * WP)];
    st.ctr[k][2] = w[WP];
    st.ctr[k][3] = w[(3 * WP) + WP];
    st.ctr[k][4] = w[2 * WP];
    st.ctr[k][5] = w[(3 * WP) + 2 * WP];
  }
}

// :389-420 for one pixel
template <bool PROFILED>
__device__ __forceinline__ float grp_weight(const grp_args_t &a, float dist, float c0, float c1, float c2, float q0, float q1, float q2)
{
  if(!PROFILED) return fast_mexp2(dist * a.sharpness);
  const float d0 = c0 - q0, d1 = c1 - q1, d2 = c2 - q2;
  const float pd = d0 * d0 * a.cp_norm + d1 * d1 * a.cp_norm + d2 * d2 * a.cp_norm;
  const float dissimilarity = (dist + pd) / a.div_d;
  return fast_mexp2(fmaxf(0.0f, dissimilarity * a.sharpness - 2.0f));
}
// dt_fast_mexp2f(), math/math.h:290-301, as the accumulation sees it: where the reference returns 0 this returns a
// subnormal, which every consumer (flush-to-zero multiplies and adds, like the reference's DAZ) reads as +0
// ANY: x may be negative or a NaN (the weights of the plain non-local means, :389-402): the conversion then has to be the
// reference's cvttss2si.  Otherwise x is max(0, .) of something (:404-420): never a NaN, and x * -2^23 saturates at the same
// INT_MIN on both machines.
template <bool ANY> __device__ __forceinline__ float grp_mexp2_daz(float x)
{
  const float v = x * -8388608.0f;
  const int k = ANY ? cvtt_x86(v) : __float2int_rz(v);
  return __int_as_float(max((int)(0x3f800000u + (unsigned)k), 0x007fffff));
}

// every pixel pair of the thread for one patch that covers the chunk: Wq = window + the patch's shift, Sg = its distortions
// The chain of one pixel pair is some twenty dependent operations long; left alone, ptxas walks the pairs one after the other
// through ten scratch registers.  The pairs are therefore taken IL at a time, stage by stage: IL independent chains in flight.
template <int WP, bool PROFILED, bool DIVC, class ST, int IL = ST::IL>
__device__ __forceinline__ void grp_accumulate_pairs(const grp_args_t &a, const float *Wq, const float *Sg, ST &st)
{
  constexpr int KP = ST::KP;
  static_assert(KP % IL == 0, "pairs per thread come in whole batches");
  const f2 cp = mk2(a.cp_norm, a.cp_norm), sharp = mk2(a.sharpness, a.sharpness);
  const f2 ndd = mk2(-a.div_d, -a.div_d), rcp = mk2(a.div_rcp, a.div_rcp);
#pragma unroll
  for(int k0 = 0; k0 < KP; k0 += IL)
  {
    f2 q0[IL], q1[IL], q2[IL], t[IL];
#pragma unroll
    for(int j = 0; j < IL; j++)
    {
      const float *const w = Wq + st.wofs(k0 + j);
      q0[j] = mk2(w[0], w[(3 * WP)]);
      q1[j] = mk2(w[WP], w[(3 * WP) + WP]);
      q2[j] = mk2(w[2 * WP], w[(3 * WP) + 2 * WP]);
      const float *const sp = Sg + st.sofs(k0 + j);
      t[j] = mk2(sp[0], sp[GRP_SP]); // the distortion
    }
    if(PROFILED)
    { // :404-420
      f2 e0[IL], e1[IL], e2[IL];
#pragma unroll
      for(int j = 0; j < IL; j++)
      {
        const int k = k0 + j;
        e0[j] = sub2(mk2(st.ctr[k][0], st.ctr[k][1]), q0[j]);
        e1[j] = sub2(mk2(st.ctr[k][2], st.ctr[k][3]), q1[j]);
        e2[j] = sub2(mk2(st.ctr[k][4], st.ctr[k][5]), q2[j]);
      }
#pragma unroll
      for(int j = 0; j < IL; j++)
      {
        e0[j] = mul2(e0[j], e0[j]);
        e1[j] = mul2(e1[j], e1[j]);
        e2[j] = mul2(e2[j], e2[j]);
      }
#pragma unroll
      for(int j = 0; j < IL; j++)
      {
        e0[j] = mul2(e0[j], cp);
        e1[j] = mul2(e1[j], cp);
        e2[j] = mul2(e2[j], cp);
      }
#pragma unroll
      for(int j = 0; j < IL; j++) e0[j] = mk2(e0[j].x + e1[j].x, e0[j].y + e1[j].y);
#pragma unroll
      for(int j = 0; j < IL; j++) e0[j] = mk2(e0[j].x + e2[j].x, e0[j].y + e2[j].y);
#pragma unroll
      for(int j = 0; j < IL; j++) t[j] = add2(t[j], e0[j]);
      if(DIVC)
      { // x / d, correctly rounded (see the head of this file).  +inf would come out of the sequence as NaN: FLT_MAX in
        // its place gives the same weight, 0 (the host checked FLT_MAX / d * sharpness > 128); a NaN stays one
#pragma unroll
        for(int j = 0; j < IL; j++) t[j] = mk2(min_nan(t[j].x, 3.402823466e38f), min_nan(t[j].y, 3.402823466e38f));
#pragma unroll
        for(int j = 0; j < IL; j++) e1[j] = mul2(t[j], rcp);
#pragma unroll
        for(int j = 0; j < IL; j++) e2[j] = fma2(e1[j], ndd, t[j]);
#pragma unroll
        for(int j = 0; j < IL; j++) t[j] = fma2(e2[j], rcp, e1[j]);
      }
      else
      {
#pragma unroll
        for(int j = 0; j < IL; j++) t[j] = mk2(t[j].x / a.div_d, t[j].y / a.div_d);
      }
#pragma unroll
      for(int j = 0; j < IL; j++) t[j] = mul2(t[j], sharp);
#pragma unroll
      for(int j = 0; j < IL; j++) t[j] = mk2(t[j].x - 2.0f, t[j].y - 2.0f);
#pragma unroll
      for(int j = 0; j < IL; j++) t[j] = mk2(fmaxf(0.0f, t[j].x), fmaxf(0.0f, t[j].y));
    }
    else
    {
#pragma unroll
      for(int j = 0; j < IL; j++) t[j] = mul2(t[j], sharp); // :389-402
    }
#pragma unroll
    for(int j = 0; j < IL; j++) t[j] = mk2(grp_mexp2_daz<!PROFILED>(t[j].x), grp_mexp2_daz<!PROFILED>(t[j].y)); // the weights
    // out += pixel * wt: products per lane, sums packed
#pragma unroll
    for(int j = 0; j < IL; j++)
    {
      q0[j] = mk2(q0[j].x * t[j].x, q0[j].y * t[j].y);
      q1[j] = mk2(q1[j].x * t[j].x, q1[j].y * t[j].y);
      q2[j] = mk2(q2[j].x * t[j].x, q2[j].y * t[j].y);
    }
#pragma unroll
    for(int j = 0; j < IL; j++)
    {
      const int k = k0 + j;
      const f2 a0 = add2(mk2(st.acc[k][0], st.acc[k][1]), q0[j]);
      const f2 a1 = add2(mk2(st.acc[k][2], st.acc[k][3]), q1[j]);
      const f2 a2 = add2(mk2(st.acc[k][4], st.acc[k][5]), q2[j]);
      const f2 a3 = add2(mk2(st.acc[k][6], st.acc[k][7]), t[j]);
      st.acc[k][0] = a0.x;
      st.acc[k][1] = a0.y;
      st.acc[k][2] = a1.x;
      st.acc[k][3] = a1.y;
      st.acc[k][4] = a2.x;
      st.acc[k][5] = a2.y;
      st.acc[k][6] = a3.x;
      st.acc[k][7] = a3.y;
    }
  }
}

// phase B2 for one thread and one patch of a chunk that is not in the interior of the frame
template <int WP, bool PROFILED, bool DIVC, class ST>
__device__ __forceinline__ void grp_accumulate_edge(const grp_args_t &a, const chunk_t &c, const float *W, const float *Sg, ST &st, int p)
{
  constexpr int KP = ST::KP;
  const pgeo_t g = patch_geo_grp(a, c, p);
  if(!g.valid || g.col_min >= g.col_max) return; // uniform
  const float *const Wq = W + g.srow * (3 * WP) + g.scol;
  if(covers_chunk(c, g))
  {
    grp_accumulate_pairs<WP, PROFILED, DIVC>(a, Wq, Sg, st);
    return;
  }
  // a patch that leaves the frame somewhere in this chunk: pixel by pixel
#pragma unroll
  for(int k = 0; k < KP; k++)
  {
    if(!((st.upper >> k) & 1u)) continue;
    const int rr = st.sofs(k) / GRP_SP, pc = st.sofs(k) - rr * GRP_SP;
    const int col = c.left + pc;
    if(col < g.col_min || col >= g.col_max) continue;
#pragma unroll
    for(int l = 0; l < 2; l++)
    {
      const int row = c.top + rr + l;
      if(row < g.row_min || row >= g.row_max) continue;
      const float *const w = Wq + st.wofs(k) + l * (3 * WP);
      const float q0 = w[0], q1 = w[WP], q2 = w[2 * WP];
      const float wt = grp_weight<PROFILED>(a, Sg[st.sofs(k) + l * GRP_SP], st.ctr[k][0 + l], st.ctr[k][2 + l], st.ctr[k][4 + l], q0, q1, q2);
      st.acc[k][0 + l] += q0 * wt;
      st.acc[k][2 + l] += q1 * wt;
      st.acc[k][4 + l] += q2 * wt;
      st.acc[k][6 + l] += 1.0f * wt;
    }
  }
}

template <int WP, bool PROFILED, bool DIVC, int KP>
__device__ __forceinline__ void grp_phase_b2(const grp_args_t &a, const chunk_t &c, const float *W, const float *S, const int *shifts,
                                             grp_thread_t<KP> &st, int p0, int tid)
{
  if(c.interior)
  {
    const int n = min(a.G, a.n_patches - p0);
    const float *Sg = S;
    for(int gi = 0; gi < n; gi++, Sg += a.splane) grp_accumulate_pairs<WP, PROFILED, DIVC>(a, W + shifts[gi], Sg, st);
    return;
  }
  for(int gi = 0; gi < a.G; gi++) grp_accumulate_edge<WP, PROFILED, DIVC>(a, c, W, S + gi * a.splane, st, p0 + gi);
}

// ---- normalise (and blend), :485-519 -----------------------------------------------------------------------------
template <class ST>
__device__ __forceinline__ void grp_finish(const grp_args_t &a, const chunk_t &c, const ST &st, int tid, int row_off = 0)
{ // row_off: chunk row of the plane row 0 the thread's offsets count from (the half-height slots: 32 for the lower half)
  constexpr int KP = ST::KP;
#pragma unroll
  for(int k = 0; k < KP; k++)
  {
    if(!((st.upper >> k) & 1u)) continue;
    const int rl = st.sofs(k) / GRP_SP, pc = st.sofs(k) - rl * GRP_SP, rr = rl + row_off;
#pragma unroll
    for(int l = 0; l < 2; l++)
    {
      if(l == 1 && !((st.lower >> k) & 1u)) continue;
      const size_t gidx = (size_t)(c.top + rr + l) * a.width + (c.left + pc);
      const float vx = st.acc[k][0 + l], vy = st.acc[k][2 + l], vz = st.acc[k][4 + l], vw = st.acc[k][6 + l];
      float4 o;
      if(a.skip_blend)
        o = make_float4(vx / vw, vy / vw, vz / vw, vw / vw);
      else
      {
        const float4 i4 = __ldg(a.in + gidx);
        o.x = (i4.x * a.invert[0]) + (vx / vw * a.weight[0]);
        o.y = (i4.y * a.invert[1]) + (vy / vw * a.weight[1]);
        o.z = (i4.z * a.invert[2]) + (vz / vw * a.weight[2]);
        o.w = (i4.w * a.invert[3]) + (vw / vw * a.weight[3]);
      }
      a.out[gidx] = o;
    }
  }
}

#ifndef B200_KERNELS_ON_CPU
template <int R, int WP, bool NORM1, bool PROFILED, bool DIVC, int KP>
__global__ void __launch_bounds__(GRP_NT, 1) nlm_group_kernel(const __grid_constant__ grp_args_t a)
{
  extern __shared__ __align__(16) float smem[];
  float *const W = smem, *const S = smem + a.wrows * (3 * WP);
  int *const shifts = reinterpret_cast<int *>(S + a.G * a.splane); // GRP_MAXG ints behind the planes
  const int tid = threadIdx.x;
  const chunk_t c = chunk_of(a, blockIdx.x);
  grp_fill<WP>(a, c, W, tid);
  __syncthreads();
  grp_thread_t<KP> st;
  grp_own_init<WP>(a, c, W, st, tid);
  for(int p0 = 0; p0 < a.n_patches; p0 += a.G)
  {
    grp_phase_a<WP, R, NORM1>(a, c, W, S, shifts, p0, tid);
    __syncthreads();
    grp_phase_b1<R>(a, c, S, p0, tid);
    __syncthreads();
    grp_phase_b2<WP, PROFILED, DIVC, KP>(a, c, W, S, shifts, st, p0, tid);
    __syncthreads();
  }
  grp_finish(a, c, st, tid);
}
#endif

// ---- the same phases as a pipeline: scan warps run ahead of the accumulating warps --------------------------------------------
// Two scan groups of 128 threads (phases A and B1 of a patch pair each, pairs dealt alternately) fill a ring of PIPE_SLOTS pair
// slots (2 planes each) in shared memory; ACC_T accumulating threads (KP pixel pairs each) drain it in patch order (phase B2).
// Named barriers: FULL[slot] (scan group arrives, accumulators wait), EMPTY[slot] (accumulators arrive, the scan group that
// wants the slot waits), one barrier per scan group between its phases A and B1.  The accumulators need two to three times the
// registers of the scan threads: setmaxnreg moves them.  Two shapes (pipe_cfg): 256 accumulating threads with 9 pixel pairs each
// (512 threads, launched with 128 registers) or 384 with 6 (640 threads, launched with 96): the second trades instruction-level
// for thread-level parallelism -- three accumulating warps per scheduler instead of two.
constexpr int PIPE_SCAN_GROUP = 128, PIPE_SLOTS = 3;
// The half-height slots below were measured faster than whole-pair slots.  What was tried around this shape and measured slower:
// three pixel pairs in flight in phase B2 (grp_accumulate_pairs<.., IL = 3>: the accumulators get faster, the frame does not -- their
// loads arrive in bursts in front of the scan warps' loads, and the scan warps are the critical path); phase B1 on two accumulating
// warps (the scan groups then run phase A only, but the accumulators wait for a chain of 72 dependent steps every pair); 384
// accumulating threads with 6 pairs each (64 registers for the scan threads spill their rings).
// On H100 (45 MP bench frame, 400 W, tools/nlm_pipe_roles.py): no warp of the half-height path waits at a barrier for more than a few per
// cent of the chunk -- every role works ~95 % of the time, and the phase-A walk sets the pace (removing its work moves the kernel time one
// for one).  Measured slower there: the half walk fully unrolled (21 % fewer instructions, 20 % more kernel time: 36 KB more code for
// the instruction caches next to the 19 KB accumulation loop); the two accumulating warps of a scheduler on the same half, in step
// (4 % slower than staggered); IL = 3 on top of the unrolled walk (no change).
// Pitches of the half-height path's 64-bit layout (pipe2_fill), WP = 97 and slot rows of GRP_SP = 77 f2, both odd.  A 64-bit access is
// served per half-warp: conflict-free when its 16 double-words fall in 16 distinct bank pairs (word index mod 16).  Phase A (lanes =
// consecutive columns of one row) and the fill are conflict-free at any pitch.  Phase B1 (lanes = the 32 rows of a half, one column):
// rows differ by 77 f2 -> an odd pitch.  Phase B2 (L = 8 strips: 8 consecutive columns on rows 8 apart per half-warp; four such groups per
// warp for c2): 8 * 77 = 8 (mod 16) for the slots, 8 * 97 = 8 (mod 16) for the f2 window plane, 8 * 97 = 8 (mod 32) for the c2 plane.
// A uniform patch shift moves every lane by the same offset and changes nothing.  Which is why the window is two planes and not rows
// of an f2 line followed by a c2 line: an f2 line needs an even row pitch (3 * WP even), and then rows 8 apart sit 0 or 16 banks apart,
// a two-way conflict on every c2 load of phase B2.  tools/nlm_pipe_banks.py checks every access at every shift of K = 7.
template <int CFG> struct pipe_cfg
{
  static constexpr int ACC_T = 256, KP = 9, L = 8, WP = 97, SCAN_REGS = 80, ACC_REGS = 176, NT = 2 * PIPE_SCAN_GROUP + ACC_T; // 256 x 80 + 256 x 176 = the register file
  static constexpr int IL = 1; // pixel pairs an accumulating thread keeps in flight in phase B2
  static constexpr bool HALVES = CFG == 0; // half-height slots (PIPE2_SLOTS) in the chunks that take them; CFG 1: whole-pair slots everywhere
};
constexpr int PIPE_N_CFG = 2;
// setmaxnreg.inc only ever gets what setmaxnreg.dec of the same block released: a shape that asks for more waits forever
template <int CFG> constexpr bool pipe_regs_balance()
{
  using c = pipe_cfg<CFG>;
  constexpr int launch = 65536 / c::NT / 8 * 8;
  return 2 * PIPE_SCAN_GROUP * (launch - c::SCAN_REGS) >= c::ACC_T * (c::ACC_REGS - launch) && c::ACC_REGS % 8 == 0 && c::SCAN_REGS % 8 == 0;
}
static_assert(pipe_regs_balance<0>(), "the accumulating warps take no more registers than the scan warps release");
constexpr int PIPE_MAX_ROWS = 64; // chunks of up to 64 rows: 2 * 32 row pairs = the 64 threads of phase B1, 2304 pixel pairs at most
constexpr int PIPE_BAR_FULL = 1, PIPE_BAR_EMPTY = PIPE_BAR_FULL + PIPE_SLOTS, PIPE_BAR_GROUP = PIPE_BAR_EMPTY + PIPE_SLOTS;
static_assert(pipe_cfg<0>::KP * pipe_cfg<0>::L >= MAX_CW && pipe_cfg<0>::ACC_T / pipe_cfg<0>::L * 2 >= PIPE_MAX_ROWS,
              "every pixel pair of a 64-row chunk has an accumulating thread");
constexpr int PIPE_WCOLS_MAX = 96; // window columns the pipelined kernel takes (pipe_cfg::WP holds them)
// phase B1 of a patch pair is 2 * half row tasks (two rows of one patch each).  They go to the upper half of the scan group (warp 3 has
// no column in phase A, warp 2 eleven): the schedulers 2 and 3 of the SM, which carry the lighter scan warps.  -1: no task.
__device__ __forceinline__ int pipe_b1_task(int t, int half)
{
  const int tb = t - PIPE_MAX_ROWS;
  return tb >= 0 && tb < 2 * half ? tb : -1;
}
template <int R> __device__ __forceinline__ void pipe_b1(const grp_args_t &a, const chunk_t &c, float *Sa, int p0, int tb, int half)
{
  if(tb < 0) return;
  const int gi = tb / half;
  grp_scan_rows<R>(a, c, Sa + gi * a.splane, p0 + gi, tb - gi * half, half);
}

// ---- half-height slots: phase B1 of one half under phase A of the next ------------------------------------------------------------
// In chunks of exactly 64 rows in the interior of the frame (all but the frame's rim) a slot holds HALF a patch pair: the column sums of
// rows 0..31 or 32..63 (two planes of 32 x GRP_SP floats), six slots in the room of the three whole-pair ones.  A scan group's warps
// 0..2 run phase A down a column as before -- the running sum and the ring of squares simply carry over from row 31 to row 32 -- and hand
// each finished half to the group's warp 3, which runs phase B1 on it (2 patches x 16 row pairs = its 32 lanes) while they are already in
// the next half.  The accumulating warps 0..3 own the row pairs of the upper halves, 4..7 those of the lower ones (grp_strip_of), and
// drain their own sequence of slots.  Barriers: FULL[slot] (warp 3 arrives, one accumulating half waits), EMPTY[slot] (that half arrives,
// the scan warps that want the slot wait), HANDOVER[group] (scan warps and warp 3 meet: the half is written, and warp 3 is done with the
// one before).  A slot is filled by the two groups in turn, three pairs apart; the group that fills it next reaches EMPTY[slot] only after it
// has written a half that needed the other group's previous half consumed, i.e. long after the other group passed the same barrier.
// Column 0 of a slot (the column of zeros) is never stored: phase B1 takes that column sum as the constant 0 (grp_row_pair<R, true>), so
// warp 0 of a scan group no longer writes 64 zeros per half in a branch of its own.  The walk runs six rows per loop trip: with three,
// the ring of squares and the prefetched row changed registers every trip and cost ~8 MOVs per row (44 instead of 36 instructions).
// Measured on an H100 80GB HBM3 at 400 W, bench frame: nlm_pipe_kernel 33.4 -> 31.8 ms (column of zeros) -> 30.4 ms (six rows per trip).
// These chunks keep the window and the slots in a layout of their own (pipe2_fill, pipe_cfg): a thread's two neighbouring values are one
// 64-bit access, which halves the shared-memory instructions at the same number of wavefronts; the helpers above (grp_colwalk_t, pipe2_b1)
// are those of the plain layout, which the group kernel and the emulation of the plain layout use.  Measured on an H100 80GB HBM3 at 700 W,
// bench frame, three alternated runs per build: nlm_pipe_kernel 26.9 -> 25.9 ms (phase-A loop 42.5 -> 39 instructions per row).
constexpr int PIPE2_SLOTS = 6, PIPE2_HROWS = 32, PIPE2_HSP = PIPE2_HROWS * GRP_SP; // floats of a half plane
constexpr int PIPE2_A_T = 96, PIPE2_ACC_HALF = 128;
constexpr int PIPE2_BAR_FULL = 1, PIPE2_BAR_EMPTY = PIPE2_BAR_FULL + PIPE2_SLOTS, PIPE2_BAR_HANDOVER = PIPE2_BAR_EMPTY + PIPE2_SLOTS; // 1..6, 7..12, 13..14
static_assert(PIPE2_BAR_HANDOVER + 2 <= 16, "sixteen named barriers per block");
static_assert(2 * PIPE2_SLOTS * PIPE2_HSP <= 2 * PIPE_SLOTS * (MAX_CH + 1) * GRP_SP, "the half slots fit the room of the whole-pair slots");

// phase A of two patches down one column, as a resumable walk: init() takes in the 2 * R + 1 rows above the chunk's first one, step<S>()
// stores the sums of a row and slides to the next (S = that row's place in the ring, row mod (2 * R + 1))
template <int WP, int R, bool NORM1> struct grp_colwalk_t
{
  static constexpr int RP = 3 * WP, N = 2 * R + 1;
  f2 ring[N][3];
  f2 cs;
  grp_row9_t nxt;
  const float *x, *ya, *yb;
  __device__ __forceinline__ void init(const grp_args_t &a, const chunk_t &c, const float *W, int pa, int k)
  {
    const int col = c.cbase + k;
    x = W + (c.top - R - c.wr0) * RP + (col - c.wc0);
    ya = x + a.patches[pa].rows * RP + a.patches[pa].cols;
    const int pb = pa + 1 < a.n_patches ? pa + 1 : pa; // the last patch of an odd list walks alone: its twin is itself, its plane unread
    yb = x + a.patches[pb].rows * RP + a.patches[pb].cols;
    cs = mk2(0.0f, 0.0f);
    nxt = grp_load_row<WP>(x, ya, yb);
#pragma unroll
    for(int i = 0; i < N; i++)
    {
      const grp_row9_t cur = nxt;
      nxt = grp_load_row<WP>(x + (i + 1) * RP, ya + (i + 1) * RP, yb + (i + 1) * RP);
      grp_squares2(cur, ring[i][0], ring[i][1], ring[i][2]);
      cs = add2(cs, grp_pd2<NORM1>(ring[i][0], ring[i][1], ring[i][2], mk2(a.norm[0], a.norm[0]), mk2(a.norm[1], a.norm[1]), mk2(a.norm[2], a.norm[2])));
    }
    x += N * RP;
    ya += N * RP;
    yb += N * RP;
  }
  // one row: its sums go to spa[0] / spb[0]; the window row that enters is the one fetched a step ago (the window has a spare row behind
  // the last one a chunk reads)
  template <int S> __device__ __forceinline__ void step(const grp_args_t &a, float *spa, float *spb)
  {
    const grp_row9_t cur = nxt;
    x += RP;
    ya += RP;
    yb += RP;
    nxt = grp_load_row<WP>(x, ya, yb);
    *spa = cs.x;
    *spb = cs.y;
    f2 e0, e1, e2;
    grp_squares2(cur, e0, e1, e2);
    cs = add2(cs, grp_pd2<NORM1>(sub2(e0, ring[S][0]), sub2(e1, ring[S][1]), sub2(e2, ring[S][2]), mk2(a.norm[0], a.norm[0]), mk2(a.norm[1], a.norm[1]),
                                 mk2(a.norm[2], a.norm[2])));
    ring[S][0] = e0;
    ring[S][1] = e1;
    ring[S][2] = e2;
  }
  // 32 rows of a half plane starting at ring place S0 (R == 1: three places)
  template <int S0> __device__ __forceinline__ void half(const grp_args_t &a, float *spa, float *spb)
  {
    static_assert(R == 1, "the half walk is written for rings of three rows");
    int r = 0;
    if(S0 == 2)
    {
      step<2>(a, spa, spb);
      r = 1;
    }
    else if(S0 == 1)
    {
      step<1>(a, spa, spb);
      step<2>(a, spa + GRP_SP, spb + GRP_SP);
      r = 2;
    }
#pragma unroll 2 // six rows per trip: the registers of the ring and of the prefetched row come back where they started (no MOVs)
    for(; r + 3 <= PIPE2_HROWS; r += 3)
    {
      step<0>(a, spa + r * GRP_SP, spb + r * GRP_SP);
      step<1>(a, spa + (r + 1) * GRP_SP, spb + (r + 1) * GRP_SP);
      step<2>(a, spa + (r + 2) * GRP_SP, spb + (r + 2) * GRP_SP);
    }
    if(r < PIPE2_HROWS) step<0>(a, spa + r * GRP_SP, spb + r * GRP_SP), r++;
    if(r < PIPE2_HROWS) step<1>(a, spa + r * GRP_SP, spb + r * GRP_SP);
  }
};
// where a chunk takes the half-height pipeline
__device__ __forceinline__ bool pipe2_takes(const grp_args_t &a, const chunk_t &c, int radius) { return radius == 1 && c.interior && c.ch == 2 * PIPE2_HROWS && a.n_patches >= 2; }
// phase B1 of one half for lane l of the group's warp 3: rows rr and rr + 16 of patch gi (planes Sa, Sa + PIPE2_HSP hold rows h0 .. h0 + 31)
template <int R> __device__ __forceinline__ void pipe2_b1(const grp_args_t &a, const chunk_t &c, float *Sa, int p0, int l)
{
  const int gi = l >> 4, rr = l & 15;
  if(p0 + gi >= a.n_patches) return;
  float *const Sx = Sa + gi * PIPE2_HSP + rr * GRP_SP - c.cbase, *const Sy = Sx + (PIPE2_HROWS / 2) * GRP_SP;
  pgeo_t g;
  g.col_min = c.left;
  g.col_max = c.right;
  grp_row_pair<R, true>(Sx, Sy, g); // column 0 of a half slot is never written: it holds the distortions of the half before
}

// ---- the half-height path's shared-memory layout: 64-bit accesses where a thread reads or writes two neighbouring values ----------
// Window: two planes of WP-element rows, one of float2 {c0, c1} and one of c2 (3 * WP floats per row, as grp_fill's); element (r, c)
// sits at r * WP + c in both, so a patch shift is one element offset for both planes.  Slots: one plane per half of a patch pair
// that holds f2 {patch a, patch b} per (row, column), rows of GRP_SP f2 (the two planes of the same slot, interleaved).  Bank
// reasoning at pipe_cfg; tools/nlm_pipe_banks.py checks it.
__device__ __forceinline__ float *pipe2_w2(float *W, int wrows, int wp) { return W + 2 * wrows * wp; } // the c2 plane behind the f2 plane
// the first float of the slots, rounded up to 8 bytes (2 * PIPE2_SLOTS * PIPE2_HSP + 1 floats fit the room of the whole-pair slots)
__device__ __forceinline__ f2 *pipe2_slots(float *smem, int wrows, int wp) { return reinterpret_cast<f2 *>(smem + ((wrows * 3 * wp + 1) & ~1)); }
static_assert(2 * PIPE2_SLOTS * PIPE2_HSP + 1 <= 2 * PIPE_SLOTS * (2 * PIPE2_HROWS + 1) * GRP_SP, "the aligned half slots fit the room of the whole-pair slots");

template <int WP, int NTHREADS> __device__ __forceinline__ void pipe2_fill(const grp_args_t &a, const chunk_t &c, float *W, int tid)
{
  f2 *const W01 = reinterpret_cast<f2 *>(W);
  float *const W2 = pipe2_w2(W, a.wrows, WP);
  const int n = a.wrows * a.wcols;
  for(int idx = tid; idx < n; idx += NTHREADS)
  {
    const int wi = idx / a.wcols, wj = idx - wi * a.wcols;
    const int r = c.wr0 + wi, col = c.wc0 + wj;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if(r >= 0 && r < a.height && col >= 0 && col < a.width) v = __ldg(a.in + (size_t)r * a.width + col);
    W01[wi * WP + wj] = mk2(v.x, v.y);
    W2[wi * WP + wj] = v.z;
  }
}
template <int WP> __device__ __forceinline__ int pipe2_shift(const grp_args_t &a, int p) { return a.patches[p].rows * WP + a.patches[p].cols; }

// phase A of two patches down one column (grp_colwalk_t on the paired window): a row is three LDS.64 and three LDS.32, its sums one STS.64
template <int WP, bool NORM1> struct pipe2_colwalk_t
{
  static constexpr int N = 3;
  f2 ring[N][3];
  f2 cs;
  f2 nx, na, nb; // the prefetched row: {c0, c1} of the pixel and of its two partners
  float nx2, na2, nb2;
  const f2 *x, *ya, *yb;
  const float *x2, *ya2, *yb2;
  __device__ __forceinline__ void load()
  {
    nx = x[0];
    na = ya[0];
    nb = yb[0];
    nx2 = x2[0];
    na2 = ya2[0];
    nb2 = yb2[0];
  }
  __device__ __forceinline__ void advance()
  {
    x += WP;
    ya += WP;
    yb += WP;
    x2 += WP;
    ya2 += WP;
    yb2 += WP;
  }
  __device__ __forceinline__ grp_row9_t row() const { return grp_row9_t{ nx.x, nx.y, nx2, na.x, na.y, na2, nb.x, nb.y, nb2 }; }
  __device__ __forceinline__ void init(const grp_args_t &a, const chunk_t &c, const float *W, int pa, int k)
  {
    const int o = (c.top - 1 - c.wr0) * WP + (c.cbase + k - c.wc0);
    const int pb = pa + 1 < a.n_patches ? pa + 1 : pa; // the last patch of an odd list walks alone: its twin is itself, its values unread
    const int sa = a.patches[pa].rows * WP + a.patches[pa].cols, sb = a.patches[pb].rows * WP + a.patches[pb].cols;
    const f2 *const W01 = reinterpret_cast<const f2 *>(W);
    const float *const W2 = W + 2 * a.wrows * WP;
    x = W01 + o;
    ya = x + sa;
    yb = x + sb;
    x2 = W2 + o;
    ya2 = x2 + sa;
    yb2 = x2 + sb;
    cs = mk2(0.0f, 0.0f);
    load();
#pragma unroll
    for(int i = 0; i < N; i++)
    {
      const grp_row9_t cur = row();
      advance();
      load();
      grp_squares2(cur, ring[i][0], ring[i][1], ring[i][2]);
      cs = add2(cs, grp_pd2<NORM1>(ring[i][0], ring[i][1], ring[i][2], mk2(a.norm[0], a.norm[0]), mk2(a.norm[1], a.norm[1]), mk2(a.norm[2], a.norm[2])));
    }
  }
  template <int S> __device__ __forceinline__ void step(const grp_args_t &a, f2 *sp)
  {
    const grp_row9_t cur = row();
    advance();
    load();
    *sp = cs;
    f2 e0, e1, e2;
    grp_squares2(cur, e0, e1, e2);
    cs = add2(cs, grp_pd2<NORM1>(sub2(e0, ring[S][0]), sub2(e1, ring[S][1]), sub2(e2, ring[S][2]), mk2(a.norm[0], a.norm[0]), mk2(a.norm[1], a.norm[1]),
                                 mk2(a.norm[2], a.norm[2])));
    ring[S][0] = e0;
    ring[S][1] = e1;
    ring[S][2] = e2;
  }
  // 32 rows of a half slot starting at ring place S0; sp: the thread's column in the slot's first row
  template <int S0> __device__ __forceinline__ void half(const grp_args_t &a, f2 *sp)
  {
    int r = 0;
    if(S0 == 2)
    {
      step<2>(a, sp);
      r = 1;
    }
    else if(S0 == 1)
    {
      step<1>(a, sp);
      step<2>(a, sp + GRP_SP);
      r = 2;
    }
#pragma unroll 2 // six rows per trip, as grp_colwalk_t::half
    for(; r + 3 <= PIPE2_HROWS; r += 3)
    {
      step<0>(a, sp + r * GRP_SP);
      step<1>(a, sp + (r + 1) * GRP_SP);
      step<2>(a, sp + (r + 2) * GRP_SP);
    }
    if(r < PIPE2_HROWS) step<0>(a, sp + r * GRP_SP), r++;
    if(r < PIPE2_HROWS) step<1>(a, sp + r * GRP_SP);
  }
};

// phase B1 of one half slot for lane l of the group's warp 3: row l of both patches (lane x: patch a, lane y: patch b), grp_row_pair<R, true>
// on f2 column sums -- the same additions in the same order per (patch, row), one LDS.64 and one STS.64 per column
template <int R> __device__ __forceinline__ void pipe2_b1_rows(const chunk_t &c, f2 *Sh, int l)
{
  constexpr int N = 2 * R + 1;
  f2 *p = Sh + l * GRP_SP + (c.left - R - 1 - c.cbase); // slot of D[left], column sum leaving at left (column 0: never stored, taken as 0)
  f2 ring[N];
  f2 distortion = mk2(0.0f, 0.0f);
  ring[0] = mk2(0.0f, 0.0f);
#pragma unroll
  for(int i = 1; i < N; i++)
  {
    ring[i] = p[i];
    distortion = add2(distortion, ring[i]);
  }
  f2 nxt[N];
#pragma unroll
  for(int s = 0; s < N; s++) nxt[s] = p[s + N];
  int left = c.right - c.left;
  for(; left >= N; left -= N)
  {
    f2 cur[N];
#pragma unroll
    for(int s = 0; s < N; s++) cur[s] = nxt[s];
#pragma unroll
    for(int s = 0; s < N; s++) nxt[s] = p[s + 2 * N];
#pragma unroll
    for(int s = 0; s < N; s++)
    {
      distortion = add2(distortion, sub2(cur[s], ring[s]));
      ring[s] = cur[s];
      p[s] = distortion;
    }
    p += N;
  }
#pragma unroll
  for(int s = 0; s < N; s++)
  {
    if(s < left)
    {
      distortion = add2(distortion, sub2(nxt[s], ring[s]));
      p[s] = distortion;
    }
  }
}

// grp_own_init (strip ownership) on the paired window: wofs0 counts elements of a plane (r * WP + c), each pixel one LDS.64 + one LDS.32
template <int WP, int KP, int L, int IL>
__device__ __forceinline__ void pipe2_own_init(const grp_args_t &a, const chunk_t &c, const float *W, grp_strip_t<KP, L, IL> &st, int ta)
{
  int pr, i;
  grp_strip_of<L>(ta, pr, i);
  const bool rows = 2 * pr < c.ch;
  const int r0 = rows ? 2 * pr : 0;
  st.wofs0 = (c.top + r0 - c.wr0) * WP + (c.left + i - c.wc0);
  st.sofs0 = r0 * GRP_SP + i;
  st.lower = st.upper = 0u;
  const f2 *const W01 = reinterpret_cast<const f2 *>(W);
  const float *const W2 = W + 2 * a.wrows * WP;
#pragma unroll
  for(int k = 0; k < KP; k++)
  {
#pragma unroll
    for(int j = 0; j < 8; j++) st.acc[k][j] = 0.0f;
    if(rows && i + k * L < c.cw)
    {
      st.upper |= 1u << k;
      if(2 * pr + 1 < c.ch) st.lower |= 1u << k;
    }
    const f2 u = W01[st.wofs(k)], d = W01[st.wofs(k) + WP];
    st.ctr[k][0] = u.x;
    st.ctr[k][1] = d.x;
    st.ctr[k][2] = u.y;
    st.ctr[k][3] = d.y;
    st.ctr[k][4] = W2[st.wofs(k)];
    st.ctr[k][5] = W2[st.wofs(k) + WP];
  }
}

// one pixel pair (acc, ctr: its slots in the strip) and one patch: grp_accumulate_pairs' arithmetic for IL = 1, operation for operation
template <bool PROFILED, bool DIVC>
__device__ __forceinline__ void pipe2_weigh(const grp_args_t &a, f2 q0, f2 q1, f2 q2, f2 t, const float *ctr, float *acc)
{
  if(PROFILED)
  { // :404-420
    f2 e0 = sub2(mk2(ctr[0], ctr[1]), q0), e1 = sub2(mk2(ctr[2], ctr[3]), q1), e2 = sub2(mk2(ctr[4], ctr[5]), q2);
    e0 = mul2(e0, e0);
    e1 = mul2(e1, e1);
    e2 = mul2(e2, e2);
    const f2 cp = mk2(a.cp_norm, a.cp_norm);
    e0 = mul2(e0, cp);
    e1 = mul2(e1, cp);
    e2 = mul2(e2, cp);
    e0 = mk2(e0.x + e1.x, e0.y + e1.y);
    e0 = mk2(e0.x + e2.x, e0.y + e2.y);
    t = add2(t, e0);
    if(DIVC)
    { // x / d, correctly rounded (grp_accumulate_pairs)
      const f2 ndd = mk2(-a.div_d, -a.div_d), rcp = mk2(a.div_rcp, a.div_rcp);
      t = mk2(min_nan(t.x, 3.402823466e38f), min_nan(t.y, 3.402823466e38f));
      e1 = mul2(t, rcp);
      e2 = fma2(e1, ndd, t);
      t = fma2(e2, rcp, e1);
    }
    else
      t = mk2(t.x / a.div_d, t.y / a.div_d);
    t = mul2(t, mk2(a.sharpness, a.sharpness));
    t = mk2(t.x - 2.0f, t.y - 2.0f);
    t = mk2(fmaxf(0.0f, t.x), fmaxf(0.0f, t.y));
  }
  else
    t = mul2(t, mk2(a.sharpness, a.sharpness)); // :389-402
  t = mk2(grp_mexp2_daz<!PROFILED>(t.x), grp_mexp2_daz<!PROFILED>(t.y)); // the weights
  q0 = mk2(q0.x * t.x, q0.y * t.y); // out += pixel * wt: products per lane, sums packed
  q1 = mk2(q1.x * t.x, q1.y * t.y);
  q2 = mk2(q2.x * t.x, q2.y * t.y);
  const f2 a0 = add2(mk2(acc[0], acc[1]), q0), a1 = add2(mk2(acc[2], acc[3]), q1), a2 = add2(mk2(acc[4], acc[5]), q2), a3 = add2(mk2(acc[6], acc[7]), t);
  acc[0] = a0.x;
  acc[1] = a0.y;
  acc[2] = a1.x;
  acc[3] = a1.y;
  acc[4] = a2.x;
  acc[5] = a2.y;
  acc[6] = a3.x;
  acc[7] = a3.y;
}
// phase B2 of one half slot: every pixel pair of the thread, patch a then (both: the pair has two patches) patch b.  Sh: the slot
// ({a, b} per row and column), sa / sb: the patches' element shifts (pipe2_shift).  A pixel's two distortions are one LDS.64, its
// partner's {c0, c1} one LDS.64 and c2 one LDS.32.  Every accumulator still takes patch a before patch b.
template <int WP, bool PROFILED, bool DIVC, class ST>
__device__ __forceinline__ void pipe2_accumulate(const grp_args_t &a, const float *W, const f2 *Sh, int sa, int sb, bool both, ST &st)
{
  constexpr int KP = ST::KP;
  const f2 *const W01 = reinterpret_cast<const f2 *>(W);
  const float *const W2 = W + 2 * a.wrows * WP;
  const f2 *const Wa = W01 + sa, *const Wb = W01 + sb;
  const float *const Wa2 = W2 + sa, *const Wb2 = W2 + sb;
#pragma unroll
  for(int k = 0; k < KP; k++)
  {
    const f2 du = Sh[st.sofs(k)], dl = Sh[st.sofs(k) + GRP_SP]; // {a, b} of the upper and of the lower pixel
    const int o = st.wofs(k);
    {
      const f2 u = Wa[o], d = Wa[o + WP];
      pipe2_weigh<PROFILED, DIVC>(a, mk2(u.x, d.x), mk2(u.y, d.y), mk2(Wa2[o], Wa2[o + WP]), mk2(du.x, dl.x), st.ctr[k], st.acc[k]);
    }
    if(both)
    {
      const f2 u = Wb[o], d = Wb[o + WP];
      pipe2_weigh<PROFILED, DIVC>(a, mk2(u.x, d.x), mk2(u.y, d.y), mk2(Wb2[o], Wb2[o + WP]), mk2(du.y, dl.y), st.ctr[k], st.acc[k]);
    }
  }
}

#ifndef B200_KERNELS_ON_CPU
__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// ---- where the warps of nlm_pipe_kernel spend their cycles (development builds with -DNLM_PIPE_TIMING only) ----------------------
// Every warp adds the clock() cycles between two marks to the role the interval belongs to; at its end lane 0 stores them, with the
// warp's first and last clock and the path the chunk took, at words [(block * warps + warp) * PIPE_TIMING_WORDS ..] of the buffer
// b200_nlm_pipe_timing() registered (tools/nlm_pipe_roles.py).  The product build compiles every mark to nothing.
enum pipe_role_t { PIPE_ROLE_FILL, PIPE_ROLE_WORK, PIPE_ROLE_FULL, PIPE_ROLE_EMPTY, PIPE_ROLE_HANDOVER, PIPE_ROLE_GROUP, PIPE_ROLE_FINISH, PIPE_ROLES };
constexpr int PIPE_TIMING_WORDS = PIPE_ROLES + 3; // + first clock, last clock, path (1: half-height slots, 2: whole-pair slots)
#ifdef NLM_PIPE_TIMING
__device__ unsigned *nlm_pipe_timing;
struct pipe_clock_t
{
  unsigned t0, t, acc[PIPE_ROLES];
  __device__ __forceinline__ pipe_clock_t()
  {
    t0 = t = (unsigned)clock();
#pragma unroll
    for(int r = 0; r < PIPE_ROLES; r++) acc[r] = 0u;
  }
  __device__ __forceinline__ void mark(int role)
  {
    const unsigned n = (unsigned)clock();
    acc[role] += n - t;
    t = n;
  }
  __device__ __forceinline__ void store(int path)
  {
    if(!nlm_pipe_timing || (threadIdx.x & 31)) return;
    unsigned *const o = nlm_pipe_timing + ((size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * PIPE_TIMING_WORDS;
#pragma unroll
    for(int r = 0; r < PIPE_ROLES; r++) o[r] = acc[r];
    o[PIPE_ROLES] = t0;
    o[PIPE_ROLES + 1] = t;
    o[PIPE_ROLES + 2] = path;
  }
};
#else
struct pipe_clock_t
{
  __device__ __forceinline__ void mark(int) {}
  __device__ __forceinline__ void store(int) {}
};
#endif

template <int R, bool NORM1, bool PROFILED, bool DIVC, int CFG>
__global__ void __launch_bounds__(pipe_cfg<CFG>::NT, 1) nlm_pipe_kernel(const __grid_constant__ grp_args_t a)
{
  using cfg = pipe_cfg<CFG>;
  constexpr int NT = cfg::NT, ACC_T = cfg::ACC_T, WP = cfg::WP;
  extern __shared__ __align__(16) float smem[];
  float *const W = smem, *const S = smem + a.wrows * (3 * WP);
  int *const shifts = reinterpret_cast<int *>(S + 2 * PIPE_SLOTS * a.splane); // window shift of every patch
  const int tid = threadIdx.x;
  pipe_clock_t clk;
  const chunk_t c = chunk_of(a, blockIdx.x);
  const bool halves = cfg::HALVES && R == 1 && pipe2_takes(a, c, R); // uniform over the block: it picks the window's layout
  if(halves)
  {
    pipe2_fill<WP, NT>(a, c, W, tid);
    for(int p = tid; p < a.n_patches; p += NT) shifts[p] = pipe2_shift<WP>(a, p);
  }
  else
  {
    grp_fill<WP, NT>(a, c, W, tid);
    for(int p = tid; p < a.n_patches; p += NT) shifts[p] = grp_shift<WP>(a, p);
  }
  __syncthreads();
  clk.mark(PIPE_ROLE_FILL);
  const int npairs = (a.n_patches + 1) / 2;
  if constexpr(cfg::HALVES && R == 1)
  if(halves)
  { // ---- half-height slots (see PIPE2_SLOTS), paired window and interleaved slots (pipe2_fill) ----
    f2 *const P = pipe2_slots(smem, a.wrows, WP);
    if(tid < 2 * PIPE_SCAN_GROUP)
    {
      asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(cfg::SCAN_REGS));
      const int group = tid / PIPE_SCAN_GROUP, t = tid - group * PIPE_SCAN_GROUP;
      if(t < PIPE2_A_T)
      {
        const bool live = t >= 1 && t < c.ncols;
        for(int q = group; q < npairs; q += 2)
        {
          pipe2_colwalk_t<WP, NORM1> walk;
          if(live) walk.init(a, c, W, 2 * q, t);
#pragma unroll
          for(int hh = 0; hh < 2; hh++)
          {
            const int w = 2 * q + hh, slot = w % PIPE2_SLOTS;
            f2 *const Sp = P + slot * PIPE2_HSP + t;
            clk.mark(PIPE_ROLE_WORK);
            if(w >= PIPE2_SLOTS) named_sync(PIPE2_BAR_EMPTY + slot, PIPE2_A_T + PIPE2_ACC_HALF);
            clk.mark(PIPE_ROLE_EMPTY);
            if(live)
            {
              if(hh == 0)
                walk.template half<0>(a, Sp);
              else
                walk.template half<(PIPE2_HROWS % 3)>(a, Sp);
            }
            clk.mark(PIPE_ROLE_WORK);
            named_sync(PIPE2_BAR_HANDOVER + group, PIPE_SCAN_GROUP);
            clk.mark(PIPE_ROLE_HANDOVER);
          }
        }
      }
      else
      {
        const int l = t - PIPE2_A_T;
        for(int q = group; q < npairs; q += 2)
          for(int hh = 0; hh < 2; hh++)
          {
            const int slot = (2 * q + hh) % PIPE2_SLOTS;
            clk.mark(PIPE_ROLE_WORK);
            named_sync(PIPE2_BAR_HANDOVER + group, PIPE_SCAN_GROUP);
            clk.mark(PIPE_ROLE_HANDOVER);
            pipe2_b1_rows<R>(c, P + slot * PIPE2_HSP, l);
            named_arrive(PIPE2_BAR_FULL + slot, 32 + PIPE2_ACC_HALF);
          }
      }
      clk.mark(PIPE_ROLE_WORK);
      clk.store(1);
    }
    else
    {
      asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(cfg::ACC_REGS));
      const int ta = tid - 2 * PIPE_SCAN_GROUP, hh = ta / PIPE2_ACC_HALF;
      grp_strip_t<cfg::KP, cfg::L, cfg::IL> st;
      pipe2_own_init<WP>(a, c, W, st, ta);
      st.sofs0 -= hh * PIPE2_HROWS * GRP_SP; // the plane of a slot starts at the half's first row
      for(int q = 0; q < npairs; q++)
      {
        const int w = 2 * q + hh, slot = w % PIPE2_SLOTS;
        clk.mark(PIPE_ROLE_WORK);
        named_sync(PIPE2_BAR_FULL + slot, 32 + PIPE2_ACC_HALF);
        clk.mark(PIPE_ROLE_FULL);
        const bool both = 2 * q + 1 < a.n_patches;
        pipe2_accumulate<WP, PROFILED, DIVC>(a, W, P + slot * PIPE2_HSP, shifts[2 * q], shifts[both ? 2 * q + 1 : 2 * q], both, st);
        if(w + PIPE2_SLOTS < 2 * npairs) named_arrive(PIPE2_BAR_EMPTY + slot, PIPE2_A_T + PIPE2_ACC_HALF);
      }
      clk.mark(PIPE_ROLE_WORK);
      grp_finish(a, c, st, ta, hh * PIPE2_HROWS);
      clk.mark(PIPE_ROLE_FINISH);
      clk.store(1);
    }
    return;
  }
  if(tid < 2 * PIPE_SCAN_GROUP)
  {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(cfg::SCAN_REGS));
    const int group = tid / PIPE_SCAN_GROUP, t = tid - group * PIPE_SCAN_GROUP;
    const int half = (c.ch + 1) / 2;
    const int tb = pipe_b1_task(t, half);
    for(int q = group; q < npairs; q += 2)
    {
      const int slot = q % PIPE_SLOTS;
      float *const Sa = S + (2 * slot) * a.splane, *const Sb = Sa + a.splane;
      clk.mark(PIPE_ROLE_WORK);
      if(q >= PIPE_SLOTS) named_sync(PIPE_BAR_EMPTY + slot, PIPE_SCAN_GROUP + ACC_T);
      clk.mark(PIPE_ROLE_EMPTY);
      if(t < c.ncols) grp_scan_column<WP, R, NORM1>(a, c, W, Sa, Sb, 2 * q, t);
      clk.mark(PIPE_ROLE_WORK);
      named_sync(PIPE_BAR_GROUP + group, PIPE_SCAN_GROUP);
      clk.mark(PIPE_ROLE_GROUP);
      pipe_b1<R>(a, c, Sa, 2 * q, tb, half);
      named_arrive(PIPE_BAR_FULL + slot, PIPE_SCAN_GROUP + ACC_T);
    }
    clk.mark(PIPE_ROLE_WORK);
    clk.store(2);
  }
  else
  {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(cfg::ACC_REGS));
    const int ta = tid - 2 * PIPE_SCAN_GROUP;
    grp_strip_t<cfg::KP, cfg::L, cfg::IL> st;
    grp_own_init<WP>(a, c, W, st, ta);
    // two loops, not one with the test inside: what the edge path keeps alive (the chunk's geometry) would otherwise take its
    // registers from the interior loop, where every register is a pixel pair more in flight
    if(c.interior)
    {
      for(int q = 0; q < npairs; q++)
      {
        const int slot = q % PIPE_SLOTS;
        const float *const Sa = S + (2 * slot) * a.splane;
        clk.mark(PIPE_ROLE_WORK);
        named_sync(PIPE_BAR_FULL + slot, PIPE_SCAN_GROUP + ACC_T);
        clk.mark(PIPE_ROLE_FULL);
        grp_accumulate_pairs<WP, PROFILED, DIVC>(a, W + shifts[2 * q], Sa, st);
        if(2 * q + 1 < a.n_patches) grp_accumulate_pairs<WP, PROFILED, DIVC>(a, W + shifts[2 * q + 1], Sa + a.splane, st);
        if(q + PIPE_SLOTS < npairs) named_arrive(PIPE_BAR_EMPTY + slot, PIPE_SCAN_GROUP + ACC_T);
      }
    }
    else
    {
      for(int q = 0; q < npairs; q++)
      {
        const int slot = q % PIPE_SLOTS;
        const float *const Sa = S + (2 * slot) * a.splane;
        clk.mark(PIPE_ROLE_WORK);
        named_sync(PIPE_BAR_FULL + slot, PIPE_SCAN_GROUP + ACC_T);
        clk.mark(PIPE_ROLE_FULL);
        grp_accumulate_edge<WP, PROFILED, DIVC>(a, c, W, Sa, st, 2 * q);
        grp_accumulate_edge<WP, PROFILED, DIVC>(a, c, W, Sa + a.splane, st, 2 * q + 1);
        if(q + PIPE_SLOTS < npairs) named_arrive(PIPE_BAR_EMPTY + slot, PIPE_SCAN_GROUP + ACC_T);
      }
    }
    clk.mark(PIPE_ROLE_WORK);
    grp_finish(a, c, st, ta);
    clk.mark(PIPE_ROLE_FINISH);
    clk.store(2);
  }
}
#endif
