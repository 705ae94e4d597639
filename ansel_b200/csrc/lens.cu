// lens correction (src/iop/lens.c process() :680-923): distortion, transverse chromatic aberration (TCA), the linear scale and pa
// vignetting, in both directions, bit for bit against the reference's lines under C float semantics.
//
// The maths is LensSerious's (src/external/LensSerious): the host resolves the lens at the shooting configuration into one flat
// block (b200_lens_eval_t, a mirror of ls_eval_t: get_modifier lens.c:620-653 -> ls_modifier_init lensserious.c:268-407 ->
// ls_eval_from_modifier :707-777), and every output pixel evaluates its own three source positions from it (ls_eval_map,
// lensserious_eval.h:601-660), as the reference's row loop does through ls_modifier_apply_subpixel_geometry.  There is no
// displacement map: lens_kernel runs one thread per output pixel, computes the map, samples the input once per channel with the
// user's warp interpolator (dt_interpolation_compute_sample, pixel/interpolation.c:396-489: mirrored border, norm 1) and folds
// the vignetting in where the reference does (lens.c:718-726).  When TCA is off the three positions are the same floats, so the
// pixel is sampled once as a float4 with the same per-lane order of operations.
//
// Blocks are 32 x 4 output pixels: neighbouring output pixels read overlapping taps, which L1 serves.  Compulsory traffic is the
// frame in and out, 32 B/px.
#ifndef B200_KERNELS_ON_CPU // tests/emul/emul_lens.cpp compiles the plan, the evaluators and the kernels of this file with g++
#include "runtime.h"
#include <mutex>
#endif
#include <float.h>
#include <math.h>
#include <string.h>
#include "interp_taps.cuh"

namespace b200
{
namespace
{
// ---- the host plan ---------------------------------------------------------------------------------------------------------------
// The calibrations are interpolated across focal length as lensfun 0.3.4 does: a Hermite spline through the two nearest
// calibrations on either side of the target (one-sided tangents where an outer neighbour is missing), distortion and the TCA terms
// beyond the first two in the term x focal domain; vignetting by inverse-distance weighting with p = 3.5 over every calibration.
struct lens_bracket_t
{
  const void *v[4]; // far below, near below, near above, far above
  float d[4];
};

void bracket_init(lens_bracket_t *s)
{
  memset(s->v, 0, sizeof(s->v));
  s->d[0] = s->d[1] = -FLT_MAX;
  s->d[2] = s->d[3] = FLT_MAX;
}

void bracket_add(lens_bracket_t *s, const float dist, const void *val)
{
  if(dist < 0)
  {
    if(dist > s->d[1])
    {
      s->d[0] = s->d[1], s->v[0] = s->v[1];
      s->d[1] = dist, s->v[1] = val;
    }
    else if(dist > s->d[0])
      s->d[0] = dist, s->v[0] = val;
  }
  else
  {
    if(dist < s->d[2])
    {
      s->d[3] = s->d[2], s->v[3] = s->v[2];
      s->d[2] = dist, s->v[2] = val;
    }
    else if(dist < s->d[3])
      s->d[3] = dist, s->v[3] = val;
  }
}

// FLT_MAX for a missing outer neighbour: the tangent there becomes the chord
float hermite(const float y1, const float y2, const float y3, const float y4, const float t)
{
  const float t2 = t * t, t3 = t2 * t;
  const float tg2 = (y1 == FLT_MAX) ? y3 - y2 : (y3 - y1) * 0.5f;
  const float tg3 = (y4 == FLT_MAX) ? y3 - y2 : (y4 - y2) * 0.5f;
  return (2.f * t3 - 3.f * t2 + 1.f) * y2 + (t3 - 2.f * t2 + t) * tg2 + (-2.f * t3 + 3.f * t2) * y3 + (t3 - t2) * tg3;
}

bool lens_real_focal(const b200_ls_lens_t *L, const float focal, float *res)
{
  if(L->n_real_focal == 0) return false;
  lens_bracket_t s;
  bracket_init(&s);
  for(int i = 0; i < L->n_real_focal; i++)
  {
    const b200_ls_calib_real_focal_t *c = &L->real_focal[i];
    if(c->real_focal == 0.f) continue;
    const float df = focal - c->focal;
    if(df == 0.0f)
    {
      *res = c->real_focal;
      return true;
    }
    bracket_add(&s, df, c);
  }
  const b200_ls_calib_real_focal_t *lo = (const b200_ls_calib_real_focal_t *)s.v[1], *hi = (const b200_ls_calib_real_focal_t *)s.v[2];
  const b200_ls_calib_real_focal_t *fl = (const b200_ls_calib_real_focal_t *)s.v[0], *fh = (const b200_ls_calib_real_focal_t *)s.v[3];
  if(!lo || !hi)
  {
    if(!lo && !hi) return false;
    *res = lo ? lo->real_focal : hi->real_focal;
    return true;
  }
  const float t = (focal - lo->focal) / (hi->focal - lo->focal);
  *res = hermite(fl ? fl->real_focal : FLT_MAX, lo->real_focal, hi->real_focal, fh ? fh->real_focal : FLT_MAX, t);
  return true;
}

bool lens_dist(const b200_ls_lens_t *L, const float focal, b200_ls_calib_dist_t *res)
{
  if(L->n_dist == 0) return false;
  lens_bracket_t s;
  bracket_init(&s);
  int model = B200_LS_DIST_NONE;
  for(int i = 0; i < L->n_dist; i++)
  {
    const b200_ls_calib_dist_t *c = &L->dist[i];
    if(c->model == B200_LS_DIST_NONE) continue;
    if(model == B200_LS_DIST_NONE) model = c->model;
    else if(model != c->model) continue; // the first model met wins
    const float df = focal - c->focal;
    if(df == 0.0f)
    {
      *res = *c;
      return true;
    }
    bracket_add(&s, df, c);
  }
  const b200_ls_calib_dist_t *lo = (const b200_ls_calib_dist_t *)s.v[1], *hi = (const b200_ls_calib_dist_t *)s.v[2];
  const b200_ls_calib_dist_t *fl = (const b200_ls_calib_dist_t *)s.v[0], *fh = (const b200_ls_calib_dist_t *)s.v[3];
  if(!lo || !hi)
  {
    if(!lo && !hi) return false;
    *res = lo ? *lo : *hi;
    return true;
  }
  res->model = model;
  res->focal = focal;
  const float t = (focal - lo->focal) / (hi->focal - lo->focal);
  for(int i = 0; i < 3; i++)
    res->terms[i] = hermite(fl ? fl->terms[i] * fl->focal : FLT_MAX, lo->terms[i] * lo->focal, hi->terms[i] * hi->focal,
                            fh ? fh->terms[i] * fh->focal : FLT_MAX, t)
                    / focal;
  return true;
}

bool lens_tca(const b200_ls_lens_t *L, const float focal, b200_ls_calib_tca_t *res)
{
  if(L->n_tca == 0) return false;
  lens_bracket_t s;
  bracket_init(&s);
  int model = B200_LS_TCA_NONE;
  for(int i = 0; i < L->n_tca; i++)
  {
    const b200_ls_calib_tca_t *c = &L->tca[i];
    if(c->model == B200_LS_TCA_NONE) continue;
    if(model == B200_LS_TCA_NONE) model = c->model;
    else if(model != c->model) continue;
    const float df = focal - c->focal;
    if(df == 0.0f)
    {
      *res = *c;
      return true;
    }
    bracket_add(&s, df, c);
  }
  const b200_ls_calib_tca_t *lo = (const b200_ls_calib_tca_t *)s.v[1], *hi = (const b200_ls_calib_tca_t *)s.v[2];
  const b200_ls_calib_tca_t *fl = (const b200_ls_calib_tca_t *)s.v[0], *fh = (const b200_ls_calib_tca_t *)s.v[3];
  if(!lo || !hi)
  {
    if(!lo && !hi) return false;
    *res = lo ? *lo : *hi;
    return true;
  }
  res->model = model;
  res->focal = focal;
  const float t = (focal - lo->focal) / (hi->focal - lo->focal);
  for(int i = 0; i < 6; i++)
  { // the first two terms (vr/vb, kr/kb) are interpolated as they are, the others in the term x focal domain
    const bool raw = i < 2;
    const float s0 = raw ? 1.f : (fl ? fl->focal : 1.f), s1 = raw ? 1.f : lo->focal, s2 = raw ? 1.f : hi->focal;
    const float s3 = raw ? 1.f : (fh ? fh->focal : 1.f), s4 = raw ? 1.f : focal;
    res->terms[i] = hermite(fl ? fl->terms[i] * s0 : FLT_MAX, lo->terms[i] * s1, hi->terms[i] * s2, fh ? fh->terms[i] * s3 : FLT_MAX, t) / s4;
  }
  return true;
}

float lens_vig_distance(const b200_ls_lens_t *L, const b200_ls_calib_vig_t *c, const float focal, const float aperture, const float distance)
{
  float f1 = focal - L->min_focal, f2 = c->focal - L->min_focal;
  const float df = L->max_focal - L->min_focal;
  if(df != 0.f)
  {
    f1 /= df;
    f2 /= df;
  }
  const float a1 = 4.f / aperture, a2 = 4.f / c->aperture;
  const float d1 = 0.1f / distance, d2 = 0.1f / c->distance;
  return sqrtf((f2 - f1) * (f2 - f1) + (a2 - a1) * (a2 - a1) + (d2 - d1) * (d2 - d1));
}

bool lens_vig(const b200_ls_lens_t *L, const float focal, const float aperture, const float distance, b200_ls_calib_vig_t *res)
{
  if(L->n_vig == 0) return false;
  int model = B200_LS_VIG_NONE;
  float total = 0.f, nearest = FLT_MAX;
  float terms[3] = { 0.f, 0.f, 0.f };
  for(int i = 0; i < L->n_vig; i++)
  {
    const b200_ls_calib_vig_t *c = &L->vig[i];
    if(c->model == B200_LS_VIG_NONE) continue;
    if(model == B200_LS_VIG_NONE) model = c->model;
    else if(model != c->model) continue;
    const float dist = lens_vig_distance(L, c, focal, aperture, distance);
    if(dist < 0.0001f)
    {
      *res = *c;
      return true;
    }
    if(dist < nearest) nearest = dist;
    const float w = (float)fabs(1.0 / pow((double)dist, 3.5)); // the weight in double, truncated once
    for(int k = 0; k < 3; k++) terms[k] += w * c->terms[k];
    total += w;
  }
  if(nearest > 1.f) return false;
  if(total <= 0.f || nearest == FLT_MAX) return false;
  res->model = model;
  res->focal = focal;
  res->aperture = aperture;
  res->distance = distance;
  for(int k = 0; k < 3; k++) res->terms[k] = terms[k] / total;
  return true;
}

// get_modifier + ls_modifier_init + ls_eval_from_modifier: returns the DT_LENS_MODIFY_* axes resolved
int lens_plan(const b200_lens_data_t *d, const int width, const int height, const int monochrome, b200_lens_eval_t *e)
{
  memset(e, 0, sizeof(*e));
  if(!d->ls_have || d->crop <= 0.f) return 0;
  const int filter = monochrome ? ~B200_LENS_MODIFY_TCA : ~0;
  const int todo = d->modify_flags & filter;
  int want = 0;
  if(todo & B200_LENS_MODIFY_DISTORTION) want |= B200_LS_ENABLE_DISTORTION;
  if(todo & B200_LENS_MODIFY_TCA) want |= B200_LS_ENABLE_TCA;
  if(todo & B200_LENS_MODIFY_VIGNETTING) want |= B200_LS_ENABLE_VIGNETTING;
  if(todo & B200_LENS_MODIFY_GEOMETRY) want |= B200_LS_ENABLE_GEOMETRY;
  if(todo & B200_LENS_MODIFY_SCALE) want |= B200_LS_ENABLE_SCALE;
  const int reverse = d->inverse ? 1 : 0;
  const b200_ls_lens_t *L = &d->ls_lens;

  // the coordinate system: lensfun measures the frame between pixel centres (size - 1) and normalises it to the calibration sensor
  const float w = (width >= 2) ? (float)(width - 1) : 1.f;
  const float h = (height >= 2) ? (float)(height - 1) : 1.f;
  const float size = (w < h) ? w : h;
  const float image_ar = (w < h) ? h / w : w / h;
  const float ar = (L->aspect_ratio > 0.f) ? L->aspect_ratio : 1.5f;
  const float arc = sqrtf(ar * ar + 1.f);
  const float cc = 1.f / sqrtf(image_ar * image_ar + 1.f) * L->crop_factor / d->crop * arc;
  const float norm_scale = 2.f / size * cc;
  const float center_x = (w / size + L->center_x) * cc;
  const float center_y = (h / size + L->center_y) * cc;
  e->norm_scale = norm_scale;
  e->norm_unscale = size * 0.5f / cc;
  e->center_x = center_x;
  e->center_y = center_y;

  const int from = L->type;
  const int to = (d->target_geom == B200_LENS_UNKNOWN) ? from : d->target_geom;
  const bool radial = from != B200_LENS_PANORAMIC && from != B200_LENS_EQUIRECTANGULAR && to != B200_LENS_PANORAMIC
                      && to != B200_LENS_EQUIRECTANGULAR && from != B200_LENS_UNKNOWN && to != B200_LENS_UNKNOWN;
  const bool geometry_unsupported = (from != to) && !radial;
  // the projection runs on the real focal over hugin's correction when the lens carries real-focal points, on the nominal otherwise
  float geom_focal_mm = d->focal;
  {
    b200_ls_calib_dist_t hd;
    const bool have = lens_dist(L, d->focal, &hd);
    float rf = 0.f;
    if(lens_real_focal(L, d->focal, &rf) && rf > 0.f)
    {
      float hugin = 1.f;
      if(have && hd.model == B200_LS_DIST_POLY3) hugin = 1.f - hd.terms[0];
      else if(have && hd.model == B200_LS_DIST_PTLENS) hugin = 1.f - hd.terms[0] - hd.terms[1] - hd.terms[2];
      geom_focal_mm = rf / hugin;
    }
  }
  e->geom_focal = geom_focal_mm * L->crop_factor * arc / 21.633307f; // half the diagonal of a 36 x 24 mm frame
  e->geom_from = reverse ? to : from;
  e->geom_to = reverse ? from : to;

  int enabled = 0;
  b200_ls_calib_dist_t dist;
  b200_ls_calib_tca_t tca;
  b200_ls_calib_vig_t vig;
  memset(&dist, 0, sizeof(dist));
  memset(&tca, 0, sizeof(tca));
  memset(&vig, 0, sizeof(vig));
  if(from != to && radial && d->focal > 0.f) enabled |= B200_LS_ENABLE_GEOMETRY;
  if((want & B200_LS_ENABLE_DISTORTION) && lens_dist(L, d->focal, &dist)) enabled |= B200_LS_ENABLE_DISTORTION;
  if((want & B200_LS_ENABLE_TCA) && lens_tca(L, d->focal, &tca)) enabled |= B200_LS_ENABLE_TCA;
  if((want & B200_LS_ENABLE_VIGNETTING) && lens_vig(L, d->focal, d->aperture, d->distance, &vig)) enabled |= B200_LS_ENABLE_VIGNETTING;
  if((want & B200_LS_ENABLE_SCALE) && d->scale != 1.0f && d->scale > 0.f)
  { // the correcting pass scales by the reciprocal, the reverse pass by the factor itself
    e->scale = reverse ? d->scale : 1.f / d->scale;
    enabled |= B200_LS_ENABLE_SCALE;
  }
  else
    e->scale = 1.f;
  // the two axes without an inverse at these coefficients are dropped in reverse, as lensfun drops them
  if(reverse && (enabled & B200_LS_ENABLE_DISTORTION) && dist.model == B200_LS_DIST_POLY3 && dist.terms[0] == 0.f)
    enabled &= ~B200_LS_ENABLE_DISTORTION;
  if(reverse && (enabled & B200_LS_ENABLE_TCA) && tca.model == B200_LS_TCA_LINEAR && (tca.terms[0] == 0.f || tca.terms[1] == 0.f))
    enabled &= ~B200_LS_ENABLE_TCA;

  const float inv_arc = 1.f / arc;
  e->vig_scale = norm_scale * inv_arc;
  e->vig_center_x = center_x * inv_arc;
  e->vig_center_y = center_y * inv_arc;
  e->enabled = enabled;
  e->dist_model = dist.model;
  e->tca_model = tca.model;
  e->vig_model = vig.model;
  for(int i = 0; i < 3; i++) e->dist_terms[i] = dist.terms[i];
  for(int i = 0; i < 6; i++) e->tca_terms[i] = tca.terms[i];
  for(int i = 0; i < 3; i++) e->vig_terms[i] = vig.terms[i];
  e->reverse = reverse;
  if(reverse && e->tca_model == B200_LS_TCA_LINEAR && (enabled & B200_LS_ENABLE_TCA))
  { // reverse linear TCA is stored as the reciprocals
    e->tca_terms[0] = 1.f / tca.terms[0];
    e->tca_terms[1] = 1.f / tca.terms[1];
  }

  int done = 0;
  if(enabled & B200_LS_ENABLE_DISTORTION) done |= B200_LENS_MODIFY_DISTORTION;
  if(enabled & B200_LS_ENABLE_TCA) done |= B200_LENS_MODIFY_TCA;
  if(enabled & B200_LS_ENABLE_VIGNETTING) done |= B200_LENS_MODIFY_VIGNETTING;
  if((enabled & B200_LS_ENABLE_GEOMETRY) && !geometry_unsupported) done |= B200_LENS_MODIFY_GEOMETRY;
  if(enabled & B200_LS_ENABLE_SCALE) done |= B200_LENS_MODIFY_SCALE;
  return done;
}

// ---- the per-pixel evaluators (lensserious_eval.h), in the reference's order of operations -----------------------------------------
constexpr int LENS_NEWTON_STEPS = 6;
constexpr float LENS_NEWTON_RTOL = 1e-6f;

__host__ __device__ __forceinline__ void lens_dist_apply(const b200_lens_eval_t &p, float *x, float *y)
{
  const float xu = *x, yu = *y;
  const float ru2 = xu * xu + yu * yu;
  float m = 1.f;
  if(p.dist_model == B200_LS_DIST_POLY3)
  {
    const float k1 = p.dist_terms[0];
    m = (1.f - k1) + k1 * ru2;
  }
  else if(p.dist_model == B200_LS_DIST_POLY5)
    m = 1.f + p.dist_terms[0] * ru2 + p.dist_terms[1] * ru2 * ru2;
  else if(p.dist_model == B200_LS_DIST_PTLENS)
  {
    const float a = p.dist_terms[0], b = p.dist_terms[1], c = p.dist_terms[2];
    const float r = sqrtf(ru2);
    m = a * ru2 * r + b * ru2 + c * r + (1.f - a - b - c);
  }
  *x = xu * m;
  *y = yu * m;
}

// Newton on the unscaled equation, six steps, converged on the relative step; 1 (no correction) when it does not converge
__host__ __device__ __forceinline__ float lens_undist_factor(const b200_lens_eval_t &p, const float rd)
{
  if(rd == 0.f) return 1.f;
  float ru = rd;
  bool converged = false;
  if(p.dist_model == B200_LS_DIST_POLY3)
  {
    const float k1 = p.dist_terms[0], k1c = 1.f - k1;
    for(int s = 0; s < LENS_NEWTON_STEPS && !converged; s++)
    {
      const float f = k1 * ru * ru * ru + k1c * ru - rd;
      const float fp = 3.f * k1 * ru * ru + k1c;
      if(fp == 0.f) return 1.f;
      const float dd = f / fp;
      ru -= dd;
      if(fabsf(dd) <= LENS_NEWTON_RTOL * fabsf(ru)) converged = true;
    }
  }
  else if(p.dist_model == B200_LS_DIST_POLY5)
  {
    const float k1 = p.dist_terms[0], k2 = p.dist_terms[1];
    for(int s = 0; s < LENS_NEWTON_STEPS && !converged; s++)
    {
      const float ru2 = ru * ru;
      const float f = ru * (1.f + k1 * ru2 + k2 * ru2 * ru2) - rd;
      const float fp = 1.f + 3.f * k1 * ru2 + 5.f * k2 * ru2 * ru2;
      if(fp == 0.f) return 1.f;
      const float dd = f / fp;
      ru -= dd;
      if(fabsf(dd) <= LENS_NEWTON_RTOL * fabsf(ru)) converged = true;
    }
  }
  else if(p.dist_model == B200_LS_DIST_PTLENS)
  {
    const float a = p.dist_terms[0], b = p.dist_terms[1], c = p.dist_terms[2];
    const float d0 = 1.f - a - b - c;
    for(int s = 0; s < LENS_NEWTON_STEPS && !converged; s++)
    {
      const float f = ru * (a * ru * ru * ru + b * ru * ru + c * ru + d0) - rd;
      const float fp = 4.f * a * ru * ru * ru + 3.f * b * ru * ru + 2.f * c * ru + d0;
      if(fp == 0.f) return 1.f;
      const float dd = f / fp;
      ru -= dd;
      if(fabsf(dd) <= LENS_NEWTON_RTOL * fabsf(ru)) converged = true;
    }
  }
  else
    return 1.f;
  if(!converged || ru < 0.f) return 1.f;
  return ru / rd;
}

__host__ __device__ __forceinline__ void lens_tca_apply(const b200_lens_eval_t &p, float *xr, float *yr, float *xb, float *yb)
{
  if(p.tca_model == B200_LS_TCA_LINEAR)
  { // reverse: the plan stored the reciprocals
    const float kr = p.tca_terms[0], kb = p.tca_terms[1];
    *xr *= kr, *yr *= kr;
    *xb *= kb, *yb *= kb;
    return;
  }
  if(p.tca_model != B200_LS_TCA_POLY3) return;
  for(int ch = 0; ch < 2; ch++)
  { // terms packed vr vb cr cb br bb
    const float v = p.tca_terms[ch], c = p.tca_terms[2 + ch], b = p.tca_terms[4 + ch];
    float *px = ch ? xb : xr, *py = ch ? yb : yr;
    if(!p.reverse)
    {
      const float x = *px, y = *py;
      const float ru2 = x * x + y * y;
      const float m = b * ru2 + v + ((c != 0.f) ? c * sqrtf(ru2) : 0.f);
      *px = x * m, *py = y * m;
      continue;
    }
    const float rd = sqrtf(*px * *px + *py * *py);
    if(rd == 0.f) continue;
    float ru = rd;
    bool ok = false;
    for(int s = 0; s < LENS_NEWTON_STEPS && !ok; s++)
    {
      const float ru2 = ru * ru;
      const float f = b * ru2 * ru + c * ru2 + v * ru - rd;
      const float fp = 3.f * b * ru2 + 2.f * c * ru + v;
      if(fp == 0.f) break;
      const float dd = f / fp;
      ru -= dd;
      if(fabsf(dd) <= LENS_NEWTON_RTOL * fabsf(ru)) ok = true;
    }
    if(ok && ru > 0.f)
    { // a channel that does not converge keeps its coordinate
      const float m = ru / rd;
      *px *= m, *py *= m;
    }
  }
}

// ls_eval_map for a plan without geometry and knot tables: out = xr yr xg yg xb yb, absolute source positions in pixels
__host__ __device__ __forceinline__ void lens_map(const b200_lens_eval_t &p, const float xu, const float yu, float *out)
{
  float x = xu * p.norm_scale - p.center_x;
  float y = yu * p.norm_scale - p.center_y;
  if(!p.reverse && (p.enabled & B200_LS_ENABLE_SCALE)) x *= p.scale, y *= p.scale;
  if(p.reverse && (p.enabled & B200_LS_ENABLE_DISTORTION))
  {
    const float m = lens_undist_factor(p, sqrtf(x * x + y * y));
    x *= m, y *= m;
  }
  if(!p.reverse && (p.enabled & B200_LS_ENABLE_DISTORTION)) lens_dist_apply(p, &x, &y);
  if(p.reverse && (p.enabled & B200_LS_ENABLE_SCALE)) x *= p.scale, y *= p.scale;
  float xr = x, yr = y, xb = x, yb = y;
  if(p.enabled & B200_LS_ENABLE_TCA) lens_tca_apply(p, &xr, &yr, &xb, &yb);
  out[0] = (xr + p.center_x) * p.norm_unscale;
  out[1] = (yr + p.center_y) * p.norm_unscale;
  out[2] = (x + p.center_x) * p.norm_unscale;
  out[3] = (y + p.center_y) * p.norm_unscale;
  out[4] = (xb + p.center_x) * p.norm_unscale;
  out[5] = (yb + p.center_y) * p.norm_unscale;
}

// ls_eval_vignette_factor for the pa model: the multiplier of a pixel at absolute position (xu, yu); 1 without vignetting
__host__ __device__ __forceinline__ float lens_vignette(const b200_lens_eval_t &p, const float xu, const float yu)
{
  if(!(p.enabled & B200_LS_ENABLE_VIGNETTING)) return 1.f;
  const float x = xu * p.vig_scale - p.vig_center_x;
  const float y = yu * p.vig_scale - p.vig_center_y;
  const float r2 = x * x + y * y;
  const float r4 = r2 * r2;
  const float c = 1.f + p.vig_terms[0] * r2 + p.vig_terms[1] * r4 + p.vig_terms[2] * r4 * r2;
  const float m = p.reverse ? c : (1.f / c);
  return (m > 0.f) ? m : 0.f;
}

__host__ __device__ __forceinline__ bool finite2(const float a, const float b) { return isfinite(a) && isfinite(b); }

// dt_interpolation_compute_sample at (x, y) in [0, w-1] x [0, h-1] of an RGBA frame: the taps of _compute_upsampling_kernel, the
// mirrored border (i < 0 -> -i, i > max -> 2 max - i; whole support inside for w, h >= 3), rows of columns accumulated in order,
// max(0, s) (the norm is 1).  LANES = 4 samples the whole pixel with the same per-lane operations.
template <int ITOR, int LANES>
__host__ __device__ __forceinline__ void lens_sample(const float *__restrict__ in, const int lane, const float x, const float y, const int w, const int h,
                                                     float *res)
{
  constexpr int W = ITOR == B200_INTERPOLATION_BILINEAR ? 1 : 2;
  float kh[2 * W], kv[2 * W];
  const int fx = (int)floorf(x) - W + 1, fy = (int)floorf(y) - W + 1;
  const float tx = x - (float)fx, ty = y - (float)fy;
#pragma unroll
  for(int k = 0; k < 2 * W; k++)
  {
    kh[k] = tap_weight(ITOR, tx + (float)k * -1.0f);
    kv[k] = tap_weight(ITOR, ty + (float)k * -1.0f);
  }
  const int ix = (int)x - (W - 1), iy = (int)y - (W - 1);
  float s[LANES];
#pragma unroll
  for(int c = 0; c < LANES; c++) s[c] = 0.f;
#pragma unroll
  for(int i = 0; i < 2 * W; i++)
  {
    int yy = iy + i;
    yy = yy < 0 ? -yy : (yy > h - 1 ? 2 * (h - 1) - yy : yy);
    const float *row = in + (size_t)yy * w * 4;
    float hs[LANES];
#pragma unroll
    for(int c = 0; c < LANES; c++) hs[c] = 0.f;
#pragma unroll
    for(int j = 0; j < 2 * W; j++)
    {
      int xx = ix + j;
      xx = xx < 0 ? -xx : (xx > w - 1 ? 2 * (w - 1) - xx : xx);
      if constexpr(LANES == 4)
      {
        const float4 v = *(const float4 *)(row + (size_t)xx * 4);
        hs[0] += kh[j] * v.x;
        hs[1] += kh[j] * v.y;
        hs[2] += kh[j] * v.z;
        hs[3] += kh[j] * v.w;
      }
      else
        hs[0] += kh[j] * row[(size_t)xx * 4 + lane];
    }
#pragma unroll
    for(int c = 0; c < LANES; c++) s[c] += kv[i] * hs[c];
  }
#pragma unroll
  for(int c = 0; c < LANES; c++) res[c] = fmaxf(0.0f, s[c]);
}

struct lens_geom_t
{
  int in_w, in_h, in_x, in_y;      // roi_in
  int out_w, out_h, out_x, out_y;  // roi_out
  int nan_checks, monochrome, mask, vignette;
};

// one output pixel of process()'s resampling loops (:747-805 reversing, :845-898 correcting)
template <int ITOR>
__host__ __device__ __forceinline__ void lens_pixel(const float *__restrict__ in, float *__restrict__ out, const b200_lens_eval_t &p, const lens_geom_t &g,
                                                    const int x, const int y)
{
  float m[6];
  lens_map(p, (float)g.out_x + (float)x, (float)(g.out_y + y), m);
  const float wm1 = g.in_w - 1.0f, hm1 = g.in_h - 1.0f;
  float px[4] = { 0.f, 0.f, 0.f, 0.f };
  const bool same = m[0] == m[2] && m[1] == m[3] && m[4] == m[2] && m[5] == m[3]; // no TCA: one position for every lane
  if(same && (!g.nan_checks || finite2(m[2], m[3])))
  {
    const float sx = fmaxf(fminf(m[2] - g.in_x, wm1), 0.0f), sy = fmaxf(fminf(m[3] - g.in_y, hm1), 0.0f);
    lens_sample<ITOR, 4>(in, 0, sx, sy, g.in_w, g.in_h, px);
    if(g.vignette && !p.reverse)
    {
      const float v = lens_vignette(p, m[2], m[3]);
      px[0] *= v, px[1] *= v, px[2] *= v;
    }
  }
  else
  {
#pragma unroll
    for(int c = 0; c < 3; c++)
    {
      if(g.nan_checks && !finite2(m[2 * c], m[2 * c + 1])) continue; // stays 0
      const float sx = fmaxf(fminf(m[2 * c] - g.in_x, wm1), 0.0f), sy = fmaxf(fminf(m[2 * c + 1] - g.in_y, hm1), 0.0f);
      lens_sample<ITOR, 1>(in, c, sx, sy, g.in_w, g.in_h, px + c);
      if(g.vignette && !p.reverse) px[c] *= lens_vignette(p, m[2 * c], m[2 * c + 1]);
    }
    if(g.mask && (!g.nan_checks || finite2(m[2], m[3])))
    {
      const float sx = fmaxf(fminf(m[2] - g.in_x, wm1), 0.0f), sy = fmaxf(fminf(m[3] - g.in_y, hm1), 0.0f);
      lens_sample<ITOR, 1>(in, 3, sx, sy, g.in_w, g.in_h, px + 3);
    }
  }
  if(g.vignette && p.reverse)
  {
    const float v = lens_vignette(p, (float)(g.out_x + x), (float)(g.out_y + y));
    px[0] *= v, px[1] *= v, px[2] *= v;
  }
  if(g.monochrome) px[0] = px[2] = px[1];
  float *o = out + ((size_t)y * g.out_w + x) * 4;
  if(g.mask)
    *(float4 *)o = make_float4(px[0], px[1], px[2], px[3]);
  else
    o[0] = px[0], o[1] = px[1], o[2] = px[2]; // lane 3 as the caller's buffer holds it
}

// ls_modifier_apply_vignetting over a copied frame (:810-822, :903-916): lanes 0-2 scaled, lane 3 kept
__host__ __device__ __forceinline__ void lens_vignette_pixel(float *__restrict__ io, const b200_lens_eval_t &p, const int w, const int x0, const int y0,
                                                             const int x, const int y)
{
  const float v = lens_vignette(p, (float)x0 + (float)x, (float)(y0 + y));
  float *o = io + ((size_t)y * w + x) * 4;
  o[0] *= v, o[1] *= v, o[2] *= v;
}

constexpr int LBX = 32, LBY = 4;

template <int ITOR>
__global__ void __launch_bounds__(LBX *LBY) lens_kernel(const float *__restrict__ in, float *__restrict__ out, const __grid_constant__ b200_lens_eval_t p,
                                                          const lens_geom_t g)
{
  const int x = blockIdx.x * LBX + threadIdx.x, y = blockIdx.y * LBY + threadIdx.y;
  if(x < g.out_w && y < g.out_h) lens_pixel<ITOR>(in, out, p, g, x, y);
}

__global__ void __launch_bounds__(LBX *LBY) lens_vignette_kernel(float *__restrict__ io, const __grid_constant__ b200_lens_eval_t p, const int w, const int h,
                                                                 const int x0, const int y0)
{
  const int x = blockIdx.x * LBX + threadIdx.x, y = blockIdx.y * LBY + threadIdx.y;
  if(x < w && y < h) lens_vignette_pixel(io, p, w, x0, y0, x, y);
}
} // namespace
} // namespace b200

#ifndef B200_KERNELS_ON_CPU
using namespace b200;

extern "C" int b200_lens_plan(const b200_lens_data_t *d, int width, int height, int monochrome, int *modflags, b200_lens_eval_t *eval)
{
  if(!d || !modflags || !eval) return fail(B200_ERR_ARG, "lens: NULL argument");
  *modflags = lens_plan(d, width, height, monochrome, eval);
  return B200_OK;
}

// The plan depends on the data block, the frame size and the monochrome flag only; a pipe asks for it once per tile and frame.
namespace
{
struct lens_plan_entry_t
{
  bool used;
  b200_lens_data_t data;
  int width, height, monochrome, modflags;
  b200_lens_eval_t eval;
};
constexpr int LENS_PLANS = 4;
lens_plan_entry_t lens_plans[LENS_PLANS];
int lens_plan_next = 0;
std::mutex lens_plan_mutex;

int cached_plan(const b200_lens_data_t *d, const int width, const int height, const int monochrome, b200_lens_eval_t *eval)
{
  std::lock_guard<std::mutex> lock(lens_plan_mutex);
  for(const lens_plan_entry_t &e : lens_plans)
    if(e.used && e.width == width && e.height == height && e.monochrome == monochrome && !memcmp(&e.data, d, sizeof(*d)))
    {
      *eval = e.eval;
      return e.modflags;
    }
  lens_plan_entry_t &e = lens_plans[lens_plan_next];
  lens_plan_next = (lens_plan_next + 1) % LENS_PLANS;
  e.used = true;
  e.data = *d;
  e.width = width, e.height = height, e.monochrome = monochrome;
  e.modflags = lens_plan(d, width, height, monochrome, &e.eval);
  *eval = e.eval;
  return e.modflags;
}
} // namespace

static int lens_check(const b200_piece_t *piece, const void *in, const void *out)
{
  if(!piece || !in || !out) return fail(B200_ERR_ARG, "lens: NULL argument");
  if(!piece->data || piece->data_size < sizeof(b200_lens_piece_t)) return fail(B200_ERR_ARG, "lens: piece->data is not a b200_lens_piece_t");
  if(in == out) return fail(B200_ERR_ARG, "lens: in-place processing is not supported");
  if(piece->channels != 4) return fail(B200_ERR_ARG, "lens: %u channels (RGBA float only)", piece->channels);
  if(piece->roi_in.width < 1 || piece->roi_in.height < 1 || piece->roi_out.width < 1 || piece->roi_out.height < 1)
    return fail(B200_ERR_ARG, "lens: empty ROI");
  const int itor = ((const b200_lens_piece_t *)piece->data)->interpolation;
  if(itor < B200_INTERPOLATION_BILINEAR || itor > B200_INTERPOLATION_MITCHELL) return fail(B200_ERR_ARG, "lens: interpolator %d", itor);
  return B200_OK;
}

extern "C" int b200_lens_process_dev(const b200_piece_t *piece, const void *d_in, void *d_out, void *stream)
{
  int rc = lens_check(piece, d_in, d_out);
  if(rc) return rc;
  const b200_lens_piece_t *lp = (const b200_lens_piece_t *)piece->data;
  const b200_lens_data_t *d = &lp->data;
  const b200_roi_t &ri = piece->roi_in, &ro = piece->roi_out;
  const bool same_shape = ri.width == ro.width && ri.height == ro.height;
  const size_t out_bytes = (size_t)ro.width * ro.height * 16;
  cudaStream_t s = (cudaStream_t)stream;
  if(!d->ls_have || d->crop <= 0.0f)
  { // :692-696
    if(!same_shape) return fail(B200_ERR_UNSUPPORTED, "lens: a copy from a %dx%d roi_in to a %dx%d roi_out", ri.width, ri.height, ro.width, ro.height);
    if((rc = bind_device(piece->devid))) return rc;
    B200_CUDA_TRY(cudaMemcpyAsync(d_out, d_in, out_bytes, cudaMemcpyDeviceToDevice, s));
    return B200_OK;
  }
  const int monochrome = (piece->image_flags & (B200_IMAGE_MONOCHROME | B200_IMAGE_MONOCHROME_BAYER)) ? 1 : 0;
  // :701, :707: a double product stored as a float, passed to get_modifier's int parameters
  const float orig_w = ri.scale * piece->buf_in_width, orig_h = ri.scale * piece->buf_in_height;
  b200_lens_eval_t p;
  const int modflags = cached_plan(d, (int)orig_w, (int)orig_h, monochrome, &p);
  if(p.enabled & B200_LS_ENABLE_GEOMETRY)
    return fail(B200_ERR_UNSUPPORTED, "lens: a projection change (lens type %d -> %d) needs tanf/asinf, which are not restated", p.geom_from, p.geom_to);
  if(p.dist_model == B200_LS_DIST_KNOTS || p.vig_model == B200_LS_VIG_KNOTS)
    return fail(B200_ERR_UNSUPPORTED, "lens: knot-table calibrations are not built");
  const bool vignette = (modflags & B200_LENS_MODIFY_VIGNETTING) != 0;
  const bool geometry = (modflags & (B200_LENS_MODIFY_TCA | B200_LENS_MODIFY_DISTORTION | B200_LENS_MODIFY_GEOMETRY | B200_LENS_MODIFY_SCALE)) != 0;
  if(geometry && (ri.width < 3 || ri.height < 3))
    return fail(B200_ERR_UNSUPPORTED, "lens: a %dx%d roi_in is smaller than the interpolator's support", ri.width, ri.height);
  if(!geometry && !same_shape)
    return fail(B200_ERR_UNSUPPORTED, "lens: a copy from a %dx%d roi_in to a %dx%d roi_out", ri.width, ri.height, ro.width, ro.height);
  if((rc = bind_device(piece->devid))) return rc;
  const dim3 block(LBX, LBY);
  if(!geometry)
  { // :808-823, :901-916: the copy, then the vignetting in the frame of the direction (roi_out reversing, roi_in correcting)
    B200_CUDA_TRY(cudaMemcpyAsync(d_out, d_in, out_bytes, cudaMemcpyDeviceToDevice, s));
    if(vignette)
    {
      const int x0 = d->inverse ? ro.x : ri.x, y0 = d->inverse ? ro.y : ri.y;
      lens_vignette_kernel<<<dim3((unsigned)((ro.width + LBX - 1) / LBX), (unsigned)((ro.height + LBY - 1) / LBY)), block, 0, s>>>((float *)d_out, p, ro.width,
                                                                                                                                  ro.height, x0, y0);
      B200_CUDA_TRY(cudaGetLastError());
    }
    return B200_OK;
  }
  const lens_geom_t g = { ri.width, ri.height, ri.x, ri.y, ro.width, ro.height, ro.x, ro.y, d->do_nan_checks ? 1 : 0, monochrome,
                          (piece->mask_display & B200_DISPLAY_MASK) ? 1 : 0, vignette ? 1 : 0 };
  const dim3 grid((unsigned)((ro.width + LBX - 1) / LBX), (unsigned)((ro.height + LBY - 1) / LBY));
  const float *src = (const float *)d_in;
  float *dst = (float *)d_out;
  switch(lp->interpolation)
  {
    case B200_INTERPOLATION_BILINEAR: lens_kernel<B200_INTERPOLATION_BILINEAR><<<grid, block, 0, s>>>(src, dst, p, g); break;
    case B200_INTERPOLATION_BICUBIC: lens_kernel<B200_INTERPOLATION_BICUBIC><<<grid, block, 0, s>>>(src, dst, p, g); break;
    default: lens_kernel<B200_INTERPOLATION_MITCHELL><<<grid, block, 0, s>>>(src, dst, p, g); break;
  }
  B200_CUDA_TRY(cudaGetLastError());
  return B200_OK;
}

extern "C" int b200_lens_process_host(const b200_piece_t *piece, const void *in, void *out)
{
  int rc = lens_check(piece, in, out);
  if(rc) return rc;
  const size_t in_bytes = (size_t)piece->roi_in.width * piece->roi_in.height * 16, out_bytes = (size_t)piece->roi_out.width * piece->roi_out.height * 16;
  // without the mask display the resampling leaves lane 3 as it finds it
  return through_device(piece, in, in_bytes, out, out_bytes, !(piece->mask_display & B200_DISPLAY_MASK), b200_lens_process_dev);
}

extern "C" void b200_lens_tiling(const b200_piece_t *piece, b200_tiling_t *t)
{ // tiling_callback :1065-1098
  if(!piece || !t) return;
  t->factor = 2.0f;
  t->maxbuf = 1.0f;
  t->factor_cl = 2.0f;
  t->maxbuf_cl = 1.0f;
  t->overhead = 0;
  t->overlap = 4;
  t->xalign = 1;
  t->yalign = 1;
}
#endif // B200_KERNELS_ON_CPU
