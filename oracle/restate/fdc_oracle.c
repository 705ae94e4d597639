/* CPU restatement of frequency-domain chroma (FDC) for X-Trans sensors.  TEST INFRASTRUCTURE ONLY.
 *
 * Follows /root/reference/src/iop/demosaic/markesteijn.c xtrans_fdc_interpolate :525-1639.  Pinned bit for bit against those lines cut
 * verbatim (oracle/_ref/libref_fdc_strict.so, oracle/fdc.mk).
 *
 * Up to the 5x5 homogeneity sums this is Markesteijn's one-pass demosaicer with a border of 13 (tiles step by 96) and a fourth plane
 * filled in the 2x2 green blocks.  Then a directionality weight, four 13x13 complex filters over the raw tile and the inverse of the
 * modulation matrix give chroma, which a 5-point median and the hybrid / pure choice combine with the Markesteijn luma.
 *
 * The reference keeps its per-thread scratch as one block of 23 planes of 122x122 floats, and its stages reuse planes:
 *   planes 0-11 rgb[4][TS][TS][3] | 12 yuv[0], gmin, the bytes of homo[4][TS][TS] | 13 yuv[1], gmax, the bytes of homosum[4][TS][TS] |
 *   14 yuv[2] | 15-18 drv[4] | 19 i_src | 20 - | 21-22 fdc_chroma
 * The chroma stage reads homosum on rows 6 to mrow - 7 but the sums are written on rows 13 to mrow - 14 and columns 8 to mcol - 14 only;
 * the median carries the chroma of row 12, row mrow - 13 and column mcol - 13 into the output.  What those bytes hold is whatever the
 * float plane 13 held: gmax of this tile at its red/blue pixels, Pb of the fourth direction inside the YPbPr window, and elsewhere what
 * an earlier tile of the same thread (or the allocator) left.  So the scratch is restated byte for byte, with the same aliasing, and
 * the caller picks where it starts from:
 *   carried (zero_per_tile = 0): one block, filled with the byte `fill` once, carried from tile to tile in the order of one thread
 *                                (the reference run on one thread with its allocator filling the block the same way);
 *   zero per tile (zero_per_tile = 1): every tile starts from a zeroed block, and a NaN stored to plane 13 as gmax or Pb is the quiet NaN
 *                                0x7fc00000.  This is what the CUDA kernel computes: the bits of a NaN the arithmetic makes are the
 *                                hardware's (x86 keeps an operand's payload or makes 0xffc00000, depending on the order the compiler
 *                                gave the operands; the GPU makes 0x7fffffff), and the sums read those bits.
 *
 * The complex products are restated on float pairs as gcc compiles C's float complex without -ffast-math: a * b is
 * (ac - bd, ad + bc), and when both parts come out NaN, libgcc's __mulsc3 recovers infinities (C11 Annex G.5.1); real x complex
 * is two real products; real - complex negates the imaginary part.
 */
#include "oracle_common.h"
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "../../ansel_b200/csrc/fdc_tables.h"

#define TS 122
#define NPX (TS * TS)
#define PAD 13
#define NPLANES 23

typedef struct
{
  float re, im;
} cf_t;

typedef struct
{
  int width, height, rx, ry;
  const uint8_t *xt;
  short hex[3][3][8];
  int sgrow, sgcol, rowoffset, coloffset;
  float hybrid[2];
} fdc_t;

static int fc(const fdc_t *m, int row, int col) { return m->xt[((row + 600 + m->ry) % 6) * 6 + (col + 600 + m->rx) % 6]; }
static const short *hexat(const fdc_t *m, int row, int col) { return m->hex[(row + 600) % 3][(col + 600) % 3]; }
static int mirror(int n, int size) { return n >= size ? 2 * size - n - 2 : abs(n); }
static float sqrf(float x) { return x * x; }
static float clamps(float a, float l, float h) { return a > l ? (a < h ? a : h) : l; }

static cf_t cmul(cf_t x, cf_t y)
{
  float a = x.re, b = x.im, c = y.re, d = y.im;
  const float ac = a * c, bd = b * d, ad = a * d, bc = b * c;
  cf_t r = { ac - bd, ad + bc };
  if(isnan(r.re) && isnan(r.im))
  { /* libgcc2.c __mulsc3 */
    int recalc = 0;
    if(isinf(a) || isinf(b))
    {
      a = copysignf(isinf(a) ? 1.0f : 0.0f, a);
      b = copysignf(isinf(b) ? 1.0f : 0.0f, b);
      if(isnan(c)) c = copysignf(0.0f, c);
      if(isnan(d)) d = copysignf(0.0f, d);
      recalc = 1;
    }
    if(isinf(c) || isinf(d))
    {
      c = copysignf(isinf(c) ? 1.0f : 0.0f, c);
      d = copysignf(isinf(d) ? 1.0f : 0.0f, d);
      if(isnan(a)) a = copysignf(0.0f, a);
      if(isnan(b)) b = copysignf(0.0f, b);
      recalc = 1;
    }
    if(!recalc && (isinf(ac) || isinf(bd) || isinf(ad) || isinf(bc)))
    {
      if(isnan(a)) a = copysignf(0.0f, a);
      if(isnan(b)) b = copysignf(0.0f, b);
      if(isnan(c)) c = copysignf(0.0f, c);
      if(isnan(d)) d = copysignf(0.0f, d);
      recalc = 1;
    }
    if(recalc)
    {
      r.re = INFINITY * (a * c - b * d);
      r.im = INFINITY * (a * d + b * c);
    }
  }
  return r;
}
static cf_t cscale(float s, cf_t x) { return (cf_t){ s * x.re, s * x.im }; }
static cf_t csub(cf_t x, cf_t y) { return (cf_t){ x.re - y.re, x.im - y.im }; }
static cf_t cadd(cf_t x, cf_t y) { return (cf_t){ x.re + y.re, x.im + y.im }; }
static cf_t cconj(cf_t x) { return (cf_t){ x.re, -x.im }; }
static cf_t ctab(const float v[2]) { return (cf_t){ v[0], v[1] }; }

/* :1075-1133: hexagons, solitary greens, the phase of the modulators */
static void setup(fdc_t *m)
{
  static const short orth[12] = { 1, 0, 0, 1, -1, 0, 0, -1, 1, 0, 0, 1 };
  static const short patt[2][16] = { { 0, 1, 0, -1, 2, 0, -1, 0, 1, 1, 1, -1, 0, 0, 0, 0 }, { 0, 1, 0, -2, 1, 0, -2, 0, 1, 1, -2, -2, 1, -1, -1, 1 } };
  m->sgrow = m->sgcol = 0;
  memset(m->hex, 0, sizeof(m->hex));
  for(int row = 0; row < 3; row++)
    for(int col = 0; col < 3; col++)
    {
      const int g = fc(m, row, col) == 1;
      int ng = 0;
      for(int d = 0; d < 10; d += 2)
      {
        ng = fc(m, row + orth[d], col + orth[d + 2]) == 1 ? 0 : ng + 1;
        if(ng == 4)
        {
          m->sgrow = row;
          m->sgcol = col;
        }
        if(ng == g + 1)
          for(int c = 0; c < 8; c++)
          {
            const int v = orth[d] * patt[g][c * 2] + orth[d + 1] * patt[g][c * 2 + 1];
            const int h = orth[d + 2] * patt[g][c * 2] + orth[d + 3] * patt[g][c * 2 + 1];
            m->hex[row][col][c ^ (g * 2 & d)] = (short)(h + v * TS);
          }
      }
    }
  /* the first row of the solitary greens' phase, and on it the first such column whose right neighbour is red */
  m->rowoffset = m->coloffset = 0;
  const int r0 = m->sgrow; /* the first row in 0..5 with (row - sgrow) % 3 == 0 */
  for(int col = 0; col < 6; col++)
    if(!((col - m->sgcol) % 3) && fc(m, r0, col + 1) == 0)
    {
      m->rowoffset = 37 - r0 - PAD;
      m->coloffset = 37 - col - PAD;
      break;
    }
}

static float canon(int on, float x)
{
  if(!on || x == x) return x;
  const uint32_t q = 0x7fc00000u;
  memcpy(&x, &q, 4);
  return x;
}

static void tile(const fdc_t *m, float *out, const float *in, int top, int left, char *buf, int zero_per_tile)
{
  const int width = m->width, height = m->height;
  float(*const rgb)[NPX][3] = (float(*)[NPX][3])buf;
  float *const plane = (float *)buf;
  float *const yuv0 = plane + 12 * NPX, *const yuv1 = plane + 13 * NPX, *const yuv2 = plane + 14 * NPX;
  float *const gmin = yuv0, *const gmax = yuv1;
  float *const drv = plane + 15 * NPX;
  uint8_t *const homo = (uint8_t *)(plane + 12 * NPX), *const homosum = (uint8_t *)(plane + 13 * NPX);
  float *const i_src = plane + 19 * NPX, *const chroma = plane + 21 * NPX;
  const int mrow = top + TS < height + PAD ? top + TS : height + PAD, mcol = left + TS < width + PAD ? left + TS : width + PAD;

  /* :1188-1241 the tile, mirrored beyond the frame, as colour planes and as the raw tile */
  for(int row = top; row < mrow; row++)
    for(int col = left; col < mcol; col++)
    {
      const int p = (row - top) * TS + (col - left), f = fc(m, row, col);
      float v;
      if(col >= 0 && row >= 0 && col < width && row < height)
        v = in[(size_t)width * row + col];
      else
      {
        const int cy = mirror(row, height), cx = mirror(col, width);
        if(f == fc(m, cy, cx))
          v = in[(size_t)width * cy + cx];
        else
        {
          float sum = 0.0f;
          uint8_t count = 0;
          for(int y = row - 1; y <= row + 1; y++)
            for(int x = col - 1; x <= col + 1; x++)
            {
              const int yy = mirror(y, height), xx = mirror(x, width);
              if(fc(m, yy, xx) == f)
              {
                sum += in[(size_t)width * yy + xx];
                count++;
              }
            }
          v = sum / count;
        }
      }
      for(int c = 0; c < 3; c++) rgb[0][p][c] = c == f ? v : 0.0f;
      i_src[p] = v;
    }
  for(int d = 1; d < 4; d++) memcpy(rgb[d], rgb[0], sizeof(rgb[0]));

  /* :1253-1300 bounds of green at the red/blue pairs: the loop hops between the rows of a vertical pair; the last visit wins */
  for(int row = top + 3; row < mrow - 3; row++)
  {
    float lo = FLT_MAX, hi = 0.0f;
    for(int col = left + 3; col < mcol - 3; col++)
    {
      if(fc(m, row, col) == 1)
      {
        lo = FLT_MAX;
        hi = 0.0f;
        continue;
      }
      const int p = (row - top) * TS + (col - left);
      if(hi == 0.0f)
      {
        const short *hex = hexat(m, row, col);
        for(int c = 0; c < 6; c++)
        {
          const float g = rgb[0][p + hex[c]][1];
          if(lo > g) lo = g;
          if(hi < g) hi = g;
        }
      }
      gmin[p] = lo;
      gmax[p] = canon(zero_per_tile, hi);
      const int phase = (row - m->sgrow) % 3;
      if(phase == 1)
      {
        if(row < mrow - 4)
        {
          row++;
          col--;
        }
      }
      else if(phase == 2)
      {
        lo = FLT_MAX;
        hi = 0.0f;
        col += 2;
        if(col < mcol - 4 && row > top + 3) row--;
      }
    }
  }

  /* :1302-1324 green along the four directions */
  for(int row = top + 3; row < mrow - 3; row++)
    for(int col = left + 3; col < mcol - 3; col++)
    {
      const int f = fc(m, row, col);
      if(f == 1) continue;
      const int p = (row - top) * TS + (col - left);
      const float(*pix)[3] = rgb[0] + p;
      const short *hex = hexat(m, row, col);
      float color[4];
      color[0] = 0.6796875f * (pix[hex[1]][1] + pix[hex[0]][1]) - 0.1796875f * (pix[2 * hex[1]][1] + pix[2 * hex[0]][1]);
      color[1] = 0.87109375f * pix[hex[3]][1] + pix[hex[2]][1] * 0.13f + 0.359375f * (pix[0][f] - pix[-hex[2]][f]);
      for(int c = 0; c < 2; c++)
        color[2 + c] = 0.640625f * pix[hex[4 + c]][1] + 0.359375f * pix[-2 * hex[4 + c]][1]
                       + 0.12890625f * (2 * pix[0][f] - pix[3 * hex[4 + c]][f] - pix[-3 * hex[4 + c]][f]);
      const int flip = !((row - m->sgrow) % 3);
      for(int c = 0; c < 4; c++) rgb[c ^ flip][p][1] = clamps(color[c], gmin[p], gmax[p]);
    }

  /* :1326-1352 red and blue at the solitary greens */
  for(int row = (top - m->sgrow + 6 + 2) / 3 * 3 + m->sgrow; row < mrow - 6; row += 3)
    for(int col = (left - m->sgcol + 6 + 2) / 3 * 3 + m->sgcol; col < mcol - 6; col += 3)
    {
      float(*rfx)[3] = rgb[0] + (row - top) * TS + (col - left);
      int h = fc(m, row, col + 1);
      float diff[6] = { 0.0f };
      float color[2][6];
      for(int i = 1, d = 0; d < 6; d++, i ^= TS ^ 1, h ^= 2)
      {
        for(int c = 0; c < 2; c++, h ^= 2)
        {
          const int o = i << c;
          const float g = 2 * rfx[0][1] - rfx[o][1] - rfx[-o][1];
          color[h != 0][d] = g + rfx[o][h] + rfx[-o][h];
          if(d > 1) diff[d] += sqrf(rfx[o][1] - rfx[-o][1] - rfx[o][h] + rfx[-o][h]) + sqrf(g);
        }
        if(d < 2 || (d & 1))
        {
          const int k = d - ((d > 1) && (diff[d - 1] < diff[d]));
          rfx[0][0] = color[0][k] / 2.f;
          rfx[0][2] = color[1][k] / 2.f;
          rfx += NPX;
        }
      }
    }

  /* :1354-1366 red at the blue pixels, blue at the red ones */
  for(int row = top + 6; row < mrow - 6; row++)
    for(int col = left + 6; col < mcol - 6; col++)
    {
      const int f = 2 - fc(m, row, col);
      if(f == 1) continue;
      float(*rfx)[3] = rgb[0] + (row - top) * TS + (col - left);
      const int c = (row - m->sgrow) % 3 ? TS : 1;
      const int h = 3 * (c ^ TS ^ 1);
      for(int d = 0; d < 4; d++, rfx += NPX)
      {
        const int i = d > 1 || ((d ^ c) & 1)
                              || ((fabsf(rfx[0][1] - rfx[c][1]) + fabsf(rfx[0][1] - rfx[-c][1]))
                                  < 2.f * (fabsf(rfx[0][1] - rfx[h][1]) + fabsf(rfx[0][1] - rfx[-h][1])))
                          ? c
                          : h;
        rfx[0][f] = (rfx[i][f] + rfx[-i][f] + 2.f * rfx[0][1] - rfx[i][1] - rfx[-i][1]) / 2.f;
      }
    }

  /* :1368-1400 the 2x2 blocks of green: planes 0 and 1 along their hexagon pairs, planes 2 and 3 the mean of those two */
  for(int row = top + 8; row < mrow - 8; row++)
  {
    if(!((row - m->sgrow) % 3)) continue;
    for(int col = left + 8; col < mcol - 8; col++)
    {
      if(!((col - m->sgcol) % 3)) continue;
      const int p = (row - top) * TS + (col - left);
      const short *hex = hexat(m, row, col);
      float rb[2][3];
      for(int k = 0; k < 2; k++)
      {
        float(*rfx)[3] = rgb[k] + p;
        const int ha = hex[2 * k], hb = hex[2 * k + 1];
        if(ha + hb)
        {
          const float g = 3.f * rfx[0][1] - 2.f * rfx[ha][1] - rfx[hb][1];
          for(int c = 0; c < 4; c += 2) rb[k][c] = rfx[0][c] = (g + 2.f * rfx[ha][c] + rfx[hb][c]) / 3.f;
        }
        else
        {
          const float g = 2.f * rfx[0][1] - rfx[ha][1] - rfx[hb][1];
          for(int c = 0; c < 4; c += 2) rb[k][c] = rfx[0][c] = (g + rfx[ha][c] + rfx[hb][c]) / 2.f;
        }
      }
      for(int k = 2; k < 4; k++)
        for(int c = 0; c < 4; c += 2) rgb[k][p][c] = (rb[0][c] + rb[1][c]) * 0.5f;
    }
  }

  /* tile-local from here.  :1412-1446 YPbPr and its second differences along each direction (yuv keeps the fourth direction's) */
  const int nrow = mrow - top, ncol = mcol - left;
  static const int dir[4] = { 1, TS, TS + 1, TS - 1 };
  for(int d = 0; d < 4; d++)
  {
    for(int row = 8; row < nrow - 8; row++)
      for(int col = 8; col < ncol - 8; col++)
      {
        const int p = row * TS + col;
        const float *rx = rgb[d][p];
        const float y = 0.2627f * rx[0] + 0.6780f * rx[1] + 0.0593f * rx[2];
        yuv0[p] = y;
        yuv1[p] = canon(zero_per_tile, (rx[2] - y) * 0.56433f);
        yuv2[p] = (rx[0] - y) * 0.67815f;
      }
    const int f = dir[d];
    for(int row = 9; row < nrow - 9; row++)
      for(int col = 9; col < ncol - 9; col++)
      {
        const int p = row * TS + col;
        drv[d * NPX + p] = sqrf(2 * yuv0[p] - yuv0[p + f] - yuv0[p - f]) + sqrf(2 * yuv1[p] - yuv1[p + f] - yuv1[p - f])
                           + sqrf(2 * yuv2[p] - yuv2[p + f] - yuv2[p - f]);
      }
  }

  /* :1448-1460 homogeneity counts */
  memset(homo, 0, 4 * NPX);
  for(int row = 10; row < nrow - 10; row++)
    for(int col = 10; col < ncol - 10; col++)
    {
      const int p = row * TS + col;
      float tr = FLT_MAX;
      for(int d = 0; d < 4; d++)
        if(tr > drv[d * NPX + p]) tr = drv[d * NPX + p];
      tr *= 8;
      for(int d = 0; d < 4; d++)
        for(int v = -1; v <= 1; v++)
          for(int h = -1; h <= 1; h++) homo[d * NPX + p] += (drv[d * NPX + p + v * TS + h] <= tr) ? 1 : 0;
    }

  /* :1462-1480 5x5 sums, rolled along each row from column 8: column c sums the counts of columns max(11, c - 2) .. c + 2 */
  for(int d = 0; d < 4; d++)
    for(int row = PAD; row < nrow - PAD; row++)
    {
      homosum[d * NPX + row * TS + PAD - 5] = 0;
      for(int col = PAD - 4; col < ncol - PAD; col++)
      {
        unsigned s = 0;
        for(int k = (col - 2 > PAD - 2 ? col - 2 : PAD - 2); k <= col + 2; k++)
          for(int v = -2; v <= 2; v++) s += homo[d * NPX + (row + v) * TS + k];
        homosum[d * NPX + row * TS + col] = (uint8_t)s;
      }
    }

  /* :1482-1555 chroma */
  for(int row = 6; row < nrow - 6; row++)
    for(int col = 6; col < ncol - 6; col++)
    {
      uint8_t hm[4], maxval = 0;
      for(int d = 0; d < 4; d++)
      {
        hm[d] = homosum[d * NPX + row * TS + col];
        maxval = maxval < hm[d] ? hm[d] : maxval;
      }
      maxval -= maxval >> 3;
      static const float directionality[4] = { 1.0f, 0.0f, 0.5f, 0.5f };
      float dircount = 0, dirsum = 0.f;
      for(int d = 0; d < 4; d++)
        if(hm[d] >= maxval)
        {
          dircount++;
          dirsum += directionality[d];
        }
      const float w = dirsum / dircount;
      cf_t C[4];
      for(int k = 0; k < 4; k++)
      {
        cf_t acc = { 0.0f, 0.0f };
        for(int i = 0; i < 13; i++)
          for(int j = 0; j < 13; j++)
          {
            const float x = i_src[(row - 6 + i) * TS + col - 6 + j];
            acc = cadd(acc, cscale(x, ctab(fdc_harr[k][12 - i][12 - j])));
          }
        C[k] = acc;
      }
      const cf_t C2m = C[0], C5m = C[1], C7m = C[2], C10m = C[3];
      cf_t mod[8];
      for(int c = 0; c < 8; c++) mod[c] = ctab(fdc_modarr[(row + m->rowoffset) % 6][(col + m->coloffset) % 6][c]);
      cf_t q[8];
      q[4] = csub(cmul(cscale(w, C10m), mod[0]), cmul(cscale(1.0f - w, C2m), mod[1]));
      q[6] = cconj(q[4]);
      q[1] = cmul(C5m, mod[6]);
      q[2] = cconj(cscale(-0.5f, q[1]));
      q[5] = cconj(q[2]);
      q[3] = cmul(C7m, mod[7]);
      q[7] = cconj(q[1]);
      const cf_t L2 = cmul(q[4], csub(cconj(mod[0]), cconj(mod[1])));
      const cf_t L3 = cmul(q[6], csub(mod[2], mod[3]));
      const cf_t L6 = cmul(q[2], cadd(cconj(mod[4]), cconj(mod[5])));
      const cf_t L12 = cmul(q[5], cadd(mod[4], mod[5]));
      const cf_t L18 = cmul(q[7], mod[6]);
      cf_t z = { i_src[row * TS + col] - L2.re, -L2.im }; /* real - complex */
      z = csub(z, L3);
      z = csub(z, C5m);
      z = csub(z, L6);
      z = csub(z, cscale(2.0f, C7m));
      z = csub(z, L12);
      q[0] = csub(z, L18);
      float rgbpix[3] = { 0.f, 0.f, 0.f };
      for(int c = 0; c < 3; c++)
        for(int k = 0; k < 8; k++) rgbpix[c] += cmul(ctab(fdc_minv[c][k]), q[k]).re;
      const float y = 0.2627f * rgbpix[0] + 0.6780f * rgbpix[1] + 0.0593f * rgbpix[2];
      chroma[row * TS + col] = (rgbpix[2] - y) * 0.56433f;
      chroma[NPX + row * TS + col] = (rgbpix[0] - y) * 0.67815f;
    }

  /* :1557-1634 Markesteijn's average for luma, the median of the FDC chroma, hybrid or pure */
  for(int row = PAD; row < nrow - PAD; row++)
    for(int col = PAD; col < ncol - PAD; col++)
    {
      const int p = row * TS + col;
      uint8_t hm[4], maxval = 0;
      for(int d = 0; d < 4; d++)
      {
        hm[d] = homosum[d * NPX + p];
        maxval = maxval < hm[d] ? hm[d] : maxval;
      }
      maxval -= maxval >> 3;
      float avg[4] = { 0.f, 0.f, 0.f, 0.f };
      for(int d = 0; d < 4; d++)
        if(hm[d] >= maxval)
        {
          for(int c = 0; c < 3; c++) avg[c] += rgb[d][p][c];
          avg[3]++;
        }
      float rgbpix[3];
      for(int c = 0; c < 3; c++) rgbpix[c] = avg[c] / avg[3];
      const float y = 0.2627f * rgbpix[0] + 0.6780f * rgbpix[1] + 0.0593f * rgbpix[2];
      const float um = (rgbpix[2] - y) * 0.56433f;
      const float vm = (rgbpix[0] - y) * 0.67815f;
      float uvf[2];
      for(int ch = 0; ch < 2; ch++)
      {
        const float *cp = chroma + ch * NPX + p;
        float t[5] = { cp[-TS], cp[-1], cp[0], cp[1], cp[TS] };
        static const int net[7][2] = { { 0, 1 }, { 3, 4 }, { 0, 3 }, { 1, 4 }, { 1, 2 }, { 2, 3 }, { 1, 2 } };
        for(int k = 0; k < 7; k++)
          if(t[net[k][0]] > t[net[k][1]])
          {
            const float s = t[net[k][0]];
            t[net[k][0]] = t[net[k][1]];
            t[net[k][1]] = s;
          }
        uvf[ch] = t[2];
      }
      const float au = fabsf(uvf[0]), av = fabsf(uvf[1]), aum = fabsf(um), avm = fabsf(vm);
      const float u = (((au < aum) & (av < 1.02f * avm)) ? uvf[0] : um) * m->hybrid[0] + uvf[0] * m->hybrid[1];
      const float v = (((av < avm) & (au < 1.02f * avm)) ? uvf[1] : vm) * m->hybrid[0] + uvf[1] * m->hybrid[1];
      float *o = out + 4 * ((size_t)width * (row + top) + col + left);
      o[0] = y + 1.474600014746f * v;
      o[1] = y - 0.15498578286403f * u - 0.571353132557189f * v;
      o[2] = y + 1.77201282937288f * u;
    }
}

/* xtrans_fdc_interpolate(): in = the mosaic of the region, (x, y) its origin on the sensor, iso the image's exif_iso, xover_iso the
 * user's crossover (pure FDC above it, hybrid at and below).  zero_per_tile, fill: see the head of this file.  Lane 3 of out is left
 * alone. */
void orc_fdc(float *out, const float *in, int width, int height, int x, int y, const uint8_t xtrans[36], float iso, int xover_iso, int zero_per_tile,
             int fill)
{
  fdc_t m = { 0 };
  m.width = width;
  m.height = height;
  m.rx = x;
  m.ry = y;
  m.xt = xtrans;
  setup(&m);
  const int iiso = (int)iso;
  m.hybrid[0] = iiso > xover_iso ? 0.0f : 1.0f;
  m.hybrid[1] = iiso > xover_iso ? 1.0f : 0.0f;
  orc_fp_fast_mode(); /* the pipe's threads run with FTZ|DAZ (darktable.c:877, common/dtpthread.c:54) */
  char *buf = malloc(sizeof(float) * NPLANES * NPX);
  memset(buf, fill, sizeof(float) * NPLANES * NPX);
  for(int top = -PAD; top < height - PAD; top += TS - 2 * PAD)
    for(int left = -PAD; left < width - PAD; left += TS - 2 * PAD)
    {
      if(zero_per_tile) memset(buf, 0, sizeof(float) * NPLANES * NPX);
      tile(&m, out, in, top, left, buf, zero_per_tile);
    }
  free(buf);
}
