/* oracle/restate: lens correction (src/iop/lens.c) -- process() :680-923 and its host plan (get_modifier :620-653 over LensSerious's
 * ls_modifier_init / ls_eval_from_modifier, src/external/LensSerious/src/lensserious.c:36-407, 707-777, and the evaluators of
 * include/lensserious_eval.h).  TEST INFRASTRUCTURE ONLY.
 *
 * Restated as the reference runs it: the plan once, then row by row the six-float map of every output pixel, each channel sampled at
 * its own source position by dt_interpolation_compute_sample (pixel/interpolation.c:396-489, mirrored border), vignetting at the
 * source (correcting) or at the destination (reversing), the copy branches with ls_modifier_apply_vignetting.  Projection changes
 * and knot tables are refused as the library refuses them. */
#include "oracle_common.h"
#include "../../include/b200iop.h"
#include <float.h>
#include <stdlib.h>
#include <string.h>

/* ---- plan --------------------------------------------------------------------------------------------------------------------- */
typedef struct
{
  const void *p[4]; /* outer below, inner below, inner above, outer above */
  float d[4];
} nearest4_t;

static void n4_reset(nearest4_t *n)
{
  memset(n->p, 0, sizeof(n->p));
  n->d[0] = n->d[1] = -FLT_MAX;
  n->d[2] = n->d[3] = FLT_MAX;
}
static void n4_offer(nearest4_t *n, float d, const void *p)
{
  if(d < 0)
  {
    if(d > n->d[1]) { n->d[0] = n->d[1]; n->p[0] = n->p[1]; n->d[1] = d; n->p[1] = p; }
    else if(d > n->d[0]) { n->d[0] = d; n->p[0] = p; }
  }
  else
  {
    if(d < n->d[2]) { n->d[3] = n->d[2]; n->p[3] = n->p[2]; n->d[2] = d; n->p[2] = p; }
    else if(d < n->d[3]) { n->d[3] = d; n->p[3] = p; }
  }
}
static float spline(float y1, float y2, float y3, float y4, float t)
{
  const float t2 = t * t, t3 = t2 * t;
  const float m2 = (y1 == FLT_MAX) ? y3 - y2 : (y3 - y1) * 0.5f;
  const float m3 = (y4 == FLT_MAX) ? y3 - y2 : (y4 - y2) * 0.5f;
  return (2.f * t3 - 3.f * t2 + 1.f) * y2 + (t3 - 2.f * t2 + t) * m2 + (-2.f * t3 + 3.f * t2) * y3 + (t3 - t2) * m3;
}

static int orc_real_focal(const b200_ls_lens_t *L, float focal, float *out)
{
  if(!L->n_real_focal) return 0;
  nearest4_t n;
  n4_reset(&n);
  for(int i = 0; i < L->n_real_focal; i++)
  {
    if(L->real_focal[i].real_focal == 0.f) continue;
    const float d = focal - L->real_focal[i].focal;
    if(d == 0.0f) { *out = L->real_focal[i].real_focal; return 1; }
    n4_offer(&n, d, &L->real_focal[i]);
  }
  const b200_ls_calib_real_focal_t *a = n.p[0], *b = n.p[1], *c = n.p[2], *e = n.p[3];
  if(!b || !c)
  {
    if(b) { *out = b->real_focal; return 1; }
    if(c) { *out = c->real_focal; return 1; }
    return 0;
  }
  *out = spline(a ? a->real_focal : FLT_MAX, b->real_focal, c->real_focal, e ? e->real_focal : FLT_MAX, (focal - b->focal) / (c->focal - b->focal));
  return 1;
}

static int orc_dist(const b200_ls_lens_t *L, float focal, b200_ls_calib_dist_t *out)
{
  if(!L->n_dist) return 0;
  nearest4_t n;
  n4_reset(&n);
  int model = 0;
  for(int i = 0; i < L->n_dist; i++)
  {
    const b200_ls_calib_dist_t *k = &L->dist[i];
    if(!k->model) continue;
    if(!model) model = k->model;
    else if(model != k->model) continue;
    const float d = focal - k->focal;
    if(d == 0.0f) { *out = *k; return 1; }
    n4_offer(&n, d, k);
  }
  const b200_ls_calib_dist_t *a = n.p[0], *b = n.p[1], *c = n.p[2], *e = n.p[3];
  if(!b || !c)
  {
    if(b) { *out = *b; return 1; }
    if(c) { *out = *c; return 1; }
    return 0;
  }
  out->model = model;
  out->focal = focal;
  const float t = (focal - b->focal) / (c->focal - b->focal);
  for(int i = 0; i < 3; i++)
    out->terms[i] = spline(a ? a->terms[i] * a->focal : FLT_MAX, b->terms[i] * b->focal, c->terms[i] * c->focal, e ? e->terms[i] * e->focal : FLT_MAX, t) / focal;
  return 1;
}

static int orc_tca(const b200_ls_lens_t *L, float focal, b200_ls_calib_tca_t *out)
{
  if(!L->n_tca) return 0;
  nearest4_t n;
  n4_reset(&n);
  int model = 0;
  for(int i = 0; i < L->n_tca; i++)
  {
    const b200_ls_calib_tca_t *k = &L->tca[i];
    if(!k->model) continue;
    if(!model) model = k->model;
    else if(model != k->model) continue;
    const float d = focal - k->focal;
    if(d == 0.0f) { *out = *k; return 1; }
    n4_offer(&n, d, k);
  }
  const b200_ls_calib_tca_t *a = n.p[0], *b = n.p[1], *c = n.p[2], *e = n.p[3];
  if(!b || !c)
  {
    if(b) { *out = *b; return 1; }
    if(c) { *out = *c; return 1; }
    return 0;
  }
  out->model = model;
  out->focal = focal;
  const float t = (focal - b->focal) / (c->focal - b->focal);
  for(int i = 0; i < 6; i++)
  {
    const int f = i >= 2; /* terms 2..5 in the term x focal domain */
    const float ya = a ? a->terms[i] * (f ? a->focal : 1.f) : FLT_MAX;
    const float ye = e ? e->terms[i] * (f ? e->focal : 1.f) : FLT_MAX;
    out->terms[i] = spline(ya, b->terms[i] * (f ? b->focal : 1.f), c->terms[i] * (f ? c->focal : 1.f), ye, t) / (f ? focal : 1.f);
  }
  return 1;
}

static int orc_vig(const b200_ls_lens_t *L, float focal, float aperture, float distance, b200_ls_calib_vig_t *out)
{
  if(!L->n_vig) return 0;
  int model = 0;
  float wsum = 0.f, dmin = FLT_MAX, acc[3] = { 0.f, 0.f, 0.f };
  const float span = L->max_focal - L->min_focal;
  for(int i = 0; i < L->n_vig; i++)
  {
    const b200_ls_calib_vig_t *k = &L->vig[i];
    if(!k->model) continue;
    if(!model) model = k->model;
    else if(model != k->model) continue;
    float f1 = focal - L->min_focal, f2 = k->focal - L->min_focal;
    if(span != 0.f) { f1 /= span; f2 /= span; }
    const float a1 = 4.f / aperture, a2 = 4.f / k->aperture, d1 = 0.1f / distance, d2 = 0.1f / k->distance;
    const float d = sqrtf((f2 - f1) * (f2 - f1) + (a2 - a1) * (a2 - a1) + (d2 - d1) * (d2 - d1));
    if(d < 0.0001f) { *out = *k; return 1; }
    if(d < dmin) dmin = d;
    const float w = (float)fabs(1.0 / pow((double)d, 3.5));
    for(int j = 0; j < 3; j++) acc[j] += w * k->terms[j];
    wsum += w;
  }
  if(dmin > 1.f || wsum <= 0.f || dmin == FLT_MAX) return 0;
  out->model = model;
  out->focal = focal, out->aperture = aperture, out->distance = distance;
  for(int j = 0; j < 3; j++) out->terms[j] = acc[j] / wsum;
  return 1;
}

int orc_lens_plan(const b200_lens_data_t *d, int width, int height, int monochrome, int *modflags, b200_lens_eval_t *e)
{
  memset(e, 0, sizeof(*e));
  *modflags = 0;
  if(!d->ls_have || d->crop <= 0.f) return 0;
  const int todo = d->modify_flags & (monochrome ? ~B200_LENS_MODIFY_TCA : ~0);
  const b200_ls_lens_t *L = &d->ls_lens;
  const float w = width >= 2 ? (float)(width - 1) : 1.f, h = height >= 2 ? (float)(height - 1) : 1.f;
  const float size = w < h ? w : h, iar = w < h ? h / w : w / h;
  const float arc = sqrtf((L->aspect_ratio > 0.f ? L->aspect_ratio : 1.5f) * (L->aspect_ratio > 0.f ? L->aspect_ratio : 1.5f) + 1.f);
  const float cc = 1.f / sqrtf(iar * iar + 1.f) * L->crop_factor / d->crop * arc;
  e->norm_scale = 2.f / size * cc;
  e->norm_unscale = size * 0.5f / cc;
  e->center_x = (w / size + L->center_x) * cc;
  e->center_y = (h / size + L->center_y) * cc;
  const int from = L->type, to = d->target_geom == B200_LENS_UNKNOWN ? from : d->target_geom;
  const int radial = from != B200_LENS_PANORAMIC && from != B200_LENS_EQUIRECTANGULAR && to != B200_LENS_PANORAMIC && to != B200_LENS_EQUIRECTANGULAR
                     && from != B200_LENS_UNKNOWN && to != B200_LENS_UNKNOWN;
  float gf = d->focal, rf = 0.f;
  b200_ls_calib_dist_t hd;
  const int hd_ok = orc_dist(L, d->focal, &hd);
  if(orc_real_focal(L, d->focal, &rf) && rf > 0.f)
  {
    float hugin = 1.f;
    if(hd_ok && hd.model == B200_LS_DIST_POLY3) hugin = 1.f - hd.terms[0];
    if(hd_ok && hd.model == B200_LS_DIST_PTLENS) hugin = 1.f - hd.terms[0] - hd.terms[1] - hd.terms[2];
    gf = rf / hugin;
  }
  e->geom_focal = gf * L->crop_factor * arc / 21.633307f;
  e->reverse = d->inverse ? 1 : 0;
  e->geom_from = e->reverse ? to : from;
  e->geom_to = e->reverse ? from : to;
  b200_ls_calib_dist_t dist = { 0 };
  b200_ls_calib_tca_t tca = { 0 };
  b200_ls_calib_vig_t vig = { 0 };
  int en = 0;
  if(from != to && radial && d->focal > 0.f) en |= B200_LS_ENABLE_GEOMETRY;
  if((todo & B200_LENS_MODIFY_DISTORTION) && orc_dist(L, d->focal, &dist)) en |= B200_LS_ENABLE_DISTORTION;
  if((todo & B200_LENS_MODIFY_TCA) && orc_tca(L, d->focal, &tca)) en |= B200_LS_ENABLE_TCA;
  if((todo & B200_LENS_MODIFY_VIGNETTING) && orc_vig(L, d->focal, d->aperture, d->distance, &vig)) en |= B200_LS_ENABLE_VIGNETTING;
  e->scale = 1.f;
  if((todo & B200_LENS_MODIFY_SCALE) && d->scale != 1.0f && d->scale > 0.f)
  {
    e->scale = e->reverse ? d->scale : 1.f / d->scale;
    en |= B200_LS_ENABLE_SCALE;
  }
  if(e->reverse && (en & B200_LS_ENABLE_DISTORTION) && dist.model == B200_LS_DIST_POLY3 && dist.terms[0] == 0.f) en &= ~B200_LS_ENABLE_DISTORTION;
  if(e->reverse && (en & B200_LS_ENABLE_TCA) && tca.model == B200_LS_TCA_LINEAR && (tca.terms[0] == 0.f || tca.terms[1] == 0.f)) en &= ~B200_LS_ENABLE_TCA;
  e->enabled = en;
  e->vig_scale = e->norm_scale * (1.f / arc);
  e->vig_center_x = e->center_x * (1.f / arc);
  e->vig_center_y = e->center_y * (1.f / arc);
  e->dist_model = dist.model, e->tca_model = tca.model, e->vig_model = vig.model;
  memcpy(e->dist_terms, dist.terms, sizeof(e->dist_terms));
  memcpy(e->tca_terms, tca.terms, sizeof(e->tca_terms));
  memcpy(e->vig_terms, vig.terms, sizeof(e->vig_terms));
  if(e->reverse && tca.model == B200_LS_TCA_LINEAR && (en & B200_LS_ENABLE_TCA))
  {
    e->tca_terms[0] = 1.f / tca.terms[0];
    e->tca_terms[1] = 1.f / tca.terms[1];
  }
  int done = 0;
  if(en & B200_LS_ENABLE_DISTORTION) done |= B200_LENS_MODIFY_DISTORTION;
  if(en & B200_LS_ENABLE_TCA) done |= B200_LENS_MODIFY_TCA;
  if(en & B200_LS_ENABLE_VIGNETTING) done |= B200_LENS_MODIFY_VIGNETTING;
  if((en & B200_LS_ENABLE_GEOMETRY) && radial) done |= B200_LENS_MODIFY_GEOMETRY;
  if(en & B200_LS_ENABLE_SCALE) done |= B200_LENS_MODIFY_SCALE;
  *modflags = done;
  return 0;
}

/* ---- evaluators --------------------------------------------------------------------------------------------------------------- */
/* Newton for Rd = f(Ru): six steps, stop on a relative step of 1e-6; the factor Ru/Rd, 1 when it fails */
static float newton_factor(const b200_lens_eval_t *p, float rd)
{
  if(rd == 0.f) return 1.f;
  const float *k = p->dist_terms;
  float ru = rd;
  int ok = 0;
  if(p->dist_model < B200_LS_DIST_POLY3 || p->dist_model > B200_LS_DIST_PTLENS) return 1.f;
  for(int s = 0; s < 6 && !ok; s++)
  {
    float f, fp;
    if(p->dist_model == B200_LS_DIST_POLY3)
    {
      f = k[0] * ru * ru * ru + (1.f - k[0]) * ru - rd;
      fp = 3.f * k[0] * ru * ru + (1.f - k[0]);
    }
    else if(p->dist_model == B200_LS_DIST_POLY5)
    {
      const float r2 = ru * ru;
      f = ru * (1.f + k[0] * r2 + k[1] * r2 * r2) - rd;
      fp = 1.f + 3.f * k[0] * r2 + 5.f * k[1] * r2 * r2;
    }
    else
    {
      const float d0 = 1.f - k[0] - k[1] - k[2];
      f = ru * (k[0] * ru * ru * ru + k[1] * ru * ru + k[2] * ru + d0) - rd;
      fp = 4.f * k[0] * ru * ru * ru + 3.f * k[1] * ru * ru + 2.f * k[2] * ru + d0;
    }
    if(fp == 0.f) return 1.f;
    const float step = f / fp;
    ru -= step;
    if(fabsf(step) <= 1e-6f * fabsf(ru)) ok = 1;
  }
  return (!ok || ru < 0.f) ? 1.f : ru / rd;
}

static void map6(const b200_lens_eval_t *p, float xu, float yu, float *o)
{
  float x = xu * p->norm_scale - p->center_x, y = yu * p->norm_scale - p->center_y;
  const int en = p->enabled;
  if(!p->reverse && (en & B200_LS_ENABLE_SCALE)) { x *= p->scale; y *= p->scale; }
  if(p->reverse && (en & B200_LS_ENABLE_DISTORTION))
  {
    const float m = newton_factor(p, sqrtf(x * x + y * y));
    x *= m;
    y *= m;
  }
  if(!p->reverse && (en & B200_LS_ENABLE_DISTORTION))
  {
    const float r2 = x * x + y * y, *k = p->dist_terms;
    float m = 1.f;
    if(p->dist_model == B200_LS_DIST_POLY3) m = (1.f - k[0]) + k[0] * r2;
    else if(p->dist_model == B200_LS_DIST_POLY5) m = 1.f + k[0] * r2 + k[1] * r2 * r2;
    else if(p->dist_model == B200_LS_DIST_PTLENS)
    {
      const float r = sqrtf(r2);
      m = k[0] * r2 * r + k[1] * r2 + k[2] * r + (1.f - k[0] - k[1] - k[2]);
    }
    x *= m;
    y *= m;
  }
  if(p->reverse && (en & B200_LS_ENABLE_SCALE)) { x *= p->scale; y *= p->scale; }
  float c[3][2] = { { x, y }, { x, y }, { x, y } };
  if((en & B200_LS_ENABLE_TCA) && p->tca_model == B200_LS_TCA_LINEAR)
    for(int ch = 0; ch < 2; ch++) { c[2 * ch][0] *= p->tca_terms[ch]; c[2 * ch][1] *= p->tca_terms[ch]; }
  else if((en & B200_LS_ENABLE_TCA) && p->tca_model == B200_LS_TCA_POLY3)
    for(int ch = 0; ch < 2; ch++)
    {
      const float v = p->tca_terms[ch], cc = p->tca_terms[2 + ch], b = p->tca_terms[4 + ch];
      float *q = c[2 * ch];
      if(!p->reverse)
      {
        const float r2 = q[0] * q[0] + q[1] * q[1];
        const float m = b * r2 + v + ((cc != 0.f) ? cc * sqrtf(r2) : 0.f);
        q[0] *= m;
        q[1] *= m;
        continue;
      }
      const float rd = sqrtf(q[0] * q[0] + q[1] * q[1]);
      if(rd == 0.f) continue;
      float ru = rd;
      int ok = 0;
      for(int s = 0; s < 6 && !ok; s++)
      {
        const float r2 = ru * ru;
        const float f = b * r2 * ru + cc * r2 + v * ru - rd, fp = 3.f * b * r2 + 2.f * cc * ru + v;
        if(fp == 0.f) break;
        const float step = f / fp;
        ru -= step;
        if(fabsf(step) <= 1e-6f * fabsf(ru)) ok = 1;
      }
      if(ok && ru > 0.f)
      {
        q[0] *= ru / rd;
        q[1] *= ru / rd;
      }
    }
  for(int ch = 0; ch < 3; ch++)
  {
    o[2 * ch] = (c[ch][0] + p->center_x) * p->norm_unscale;
    o[2 * ch + 1] = (c[ch][1] + p->center_y) * p->norm_unscale;
  }
}

static float vignette(const b200_lens_eval_t *p, float xu, float yu)
{
  const float x = xu * p->vig_scale - p->vig_center_x, y = yu * p->vig_scale - p->vig_center_y;
  const float r2 = x * x + y * y, r4 = r2 * r2;
  const float c = 1.f + p->vig_terms[0] * r2 + p->vig_terms[1] * r4 + p->vig_terms[2] * r4 * r2;
  const float m = p->reverse ? c : 1.f / c;
  return m > 0.f ? m : 0.f;
}

static float tap(int itor, float t)
{
  const float a = fabsf(t);
  if(itor == B200_INTERPOLATION_BILINEAR) return 1.0f - a;
  if(itor == B200_INTERPOLATION_BICUBIC)
    return a <= 1.0f ? ((3.0f * (t * t) - 5.0f * a) * a + 2.0f) * 0.5f : (a * (5.0f * a - 8.0f - t * t) + 4.0f) * 0.5f;
  return a <= 1.0f ? (7.0f / 6.0f) * (a * a * a) - 2.0f * (a * a) + (8.0f / 9.0f)
                   : 2.0f * (a * a) - (7.0f / 18.0f) * (a * a * a) - (10.0f / 3.0f) * a + (16.0f / 9.0f);
}

static int mirror(int i, int n) { return i < 0 ? -i : (i > n - 1 ? 2 * (n - 1) - i : i); }

/* one lane of the RGBA frame at (x, y) inside it */
static float sample(const float *in, int lane, float x, float y, int w, int h, int itor)
{
  const int hw = itor == B200_INTERPOLATION_BILINEAR ? 1 : 2;
  float kx[4], ky[4];
  const int x0 = (int)floorf(x) - hw + 1, y0 = (int)floorf(y) - hw + 1;
  for(int k = 0; k < 2 * hw; k++)
  {
    kx[k] = tap(itor, (x - (float)x0) + (float)k * -1.0f);
    ky[k] = tap(itor, (y - (float)y0) + (float)k * -1.0f);
  }
  float s = 0.f;
  for(int i = 0; i < 2 * hw; i++)
  {
    float r = 0.0f;
    for(int j = 0; j < 2 * hw; j++) r += kx[j] * in[((size_t)mirror(y0 + i, h) * w + mirror(x0 + j, w)) * 4 + lane];
    s += ky[i] * r;
  }
  return fmaxf(0.0f, s / (1.0f * 1.0f));
}

int orc_lens(const float *in, float *out, const b200_lens_data_t *d, int itor, int monochrome, int mask_display, int in_x, int in_y, int in_w,
             int in_h, double in_scale, int out_x, int out_y, int out_w, int out_h, int buf_in_w, int buf_in_h)
{
  orc_fp_fast_mode(); /* the pipe's threads run with FTZ|DAZ (darktable.c:877) */
  const int same_shape = in_w == out_w && in_h == out_h;
  if(!d->ls_have || d->crop <= 0.0f)
  {
    if(!same_shape) return B200_ERR_UNSUPPORTED;
    memcpy(out, in, sizeof(float) * 4 * out_w * out_h);
    return 0;
  }
  const float ow = in_scale * buf_in_w, oh = in_scale * buf_in_h;
  int mf;
  b200_lens_eval_t p;
  orc_lens_plan(d, (int)ow, (int)oh, monochrome, &mf, &p);
  if((p.enabled & B200_LS_ENABLE_GEOMETRY) || p.dist_model == B200_LS_DIST_KNOTS || p.vig_model == B200_LS_VIG_KNOTS) return B200_ERR_UNSUPPORTED;
  const int vig = (mf & B200_LENS_MODIFY_VIGNETTING) != 0;
  const int geo = (mf & (B200_LENS_MODIFY_TCA | B200_LENS_MODIFY_DISTORTION | B200_LENS_MODIFY_GEOMETRY | B200_LENS_MODIFY_SCALE)) != 0;
  if(geo && (in_w < 3 || in_h < 3)) return B200_ERR_UNSUPPORTED;
  if(!geo)
  {
    if(!same_shape) return B200_ERR_UNSUPPORTED;
    memcpy(out, in, sizeof(float) * 4 * out_w * out_h);
    if(!vig) return 0;
    const int x0 = d->inverse ? out_x : in_x, y0 = d->inverse ? out_y : in_y;
    for(int y = 0; y < out_h; y++)
      for(int x = 0; x < out_w; x++)
      {
        const float v = vignette(&p, (float)x0 + (float)x, (float)(y0 + y));
        for(int c = 0; c < 3; c++) out[((size_t)y * out_w + x) * 4 + c] *= v;
      }
    return 0;
  }
  for(int y = 0; y < out_h; y++)
    for(int x = 0; x < out_w; x++)
    {
      float m[6], px[4] = { 0.f, 0.f, 0.f, 0.f };
      map6(&p, (float)out_x + (float)x, (float)(out_y + y), m);
      for(int c = 0; c < 4; c++)
      {
        if(c == 3 && !(mask_display & B200_DISPLAY_MASK)) break;
        const int k = c == 3 ? 1 : c; /* lane 3 follows the green position */
        if(d->do_nan_checks && (!isfinite(m[2 * k]) || !isfinite(m[2 * k + 1]))) continue;
        const float sx = fmaxf(fminf(m[2 * k] - in_x, in_w - 1.0f), 0.0f), sy = fmaxf(fminf(m[2 * k + 1] - in_y, in_h - 1.0f), 0.0f);
        px[c] = sample(in, c, sx, sy, in_w, in_h, itor);
        if(c < 3 && vig && !d->inverse) px[c] *= vignette(&p, m[2 * k], m[2 * k + 1]);
      }
      if(vig && d->inverse)
      {
        const float v = vignette(&p, (float)(out_x + x), (float)(out_y + y));
        for(int c = 0; c < 3; c++) px[c] *= v;
      }
      if(monochrome) px[0] = px[2] = px[1];
      float *o = out + ((size_t)y * out_w + x) * 4;
      for(int c = 0; c < ((mask_display & B200_DISPLAY_MASK) ? 4 : 3); c++) o[c] = px[c];
    }
  return 0;
}
