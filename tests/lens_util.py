"""lens correction (src/iop/lens.c) through the checkers: the oracle (oracle/restate/lens_oracle.c), the reference's own lines compiled in
place beside LensSerious's lensserious.c (oracle/_ref/libref_lens_{strict,fast}.so from oracle/lens.mk) and the product's plan and
kernels under g++ (tests/emul/emul_lens.cpp).  The calibrations are synthetic ls_lens_t values.  Checkers only."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import util
import ansel_b200 as ab

EMUL = os.path.join(util.ROOT, "tests", "emul")
ITORS = {ab.INTERPOLATION_BILINEAR: b"bilinear", ab.INTERPOLATION_BICUBIC: b"bicubic", ab.INTERPOLATION_MITCHELL: b"mitchell"}
DIST = (ab.LS_DIST_NONE, ab.LS_DIST_POLY3, ab.LS_DIST_POLY5, ab.LS_DIST_PTLENS)
TCA = (ab.LS_TCA_NONE, ab.LS_TCA_LINEAR, ab.LS_TCA_POLY3)
# (roi_in x, y, w, h, roi_out x, y, w, h, roi scale, buf_in w, h): the whole frame, and a zoomed-out crop shifted inside it
ROIS = ((0, 0, 61, 43, 0, 0, 61, 43, 1.0, 61, 43), (9, 5, 52, 40, 12, 7, 47, 35, 0.5, 150, 104))
# (do_nan_checks, monochrome, mask display)
FLAGS = ((1, 0, 0), (0, 1, 1), (1, 1, 0), (0, 0, 1))

# per model: the terms at focal 18, 24, 35, 55 mm (strong enough to move pixels by several px on a 61 px frame)
DIST_TERMS = {ab.LS_DIST_POLY3: ((-0.031,), (-0.018,), (-0.006,), (0.004,)),
              ab.LS_DIST_POLY5: ((-0.052, 0.011), (-0.031, 0.006), (-0.012, 0.002), (0.006, -0.001)),
              ab.LS_DIST_PTLENS: ((0.012, -0.045, 0.021), (0.008, -0.027, 0.013), (0.004, -0.011, 0.006), (0.001, 0.003, -0.002))}
TCA_TERMS = {ab.LS_TCA_LINEAR: ((1.0012, 0.9991), (1.0008, 0.9994), (1.0005, 0.9997), (1.0003, 0.9998)),
             ab.LS_TCA_POLY3: ((1.0011, 0.9993, 0.0004, -0.0003, 0.0006, -0.0005), (1.0008, 0.9995, 0.0003, -0.0002, 0.0004, -0.0004),
                               (1.0005, 0.9997, 0.0, -0.0001, 0.0002, -0.0002), (1.0002, 0.9999, 0.0001, 0.0, 0.0001, -0.0001))}
FOCALS = (18.0, 24.0, 35.0, 55.0)


def lens_data(dist=ab.LS_DIST_PTLENS, tca=ab.LS_TCA_POLY3, vig=True, inverse=0, nan_checks=1, focal=28.0, scale=1.0, crop=1.53,
              target_geom=ab.LENS_UNKNOWN, lens_type=ab.LENS_RECTILINEAR, ls_have=1, real_focal=False) -> ab.LensData:
    d = ab.LensData()
    d.modify_flags = ab.LENS_MODIFY_DISTORTION | ab.LENS_MODIFY_TCA | ab.LENS_MODIFY_VIGNETTING | (ab.LENS_MODIFY_SCALE if scale != 1.0 else 0)
    d.inverse, d.scale, d.crop, d.focal, d.aperture, d.distance = inverse, scale, crop, focal, 5.6, 10.0
    d.target_geom, d.do_nan_checks, d.tca_override, d.ls_have = target_geom, nan_checks, 0, ls_have
    L = d.ls_lens
    L.type, L.crop_factor, L.aspect_ratio, L.min_focal, L.max_focal = lens_type, 1.534, 1.5, 18.0, 55.0
    L.center_x, L.center_y = 0.012, -0.008
    if dist != ab.LS_DIST_NONE:
        L.n_dist = len(FOCALS)
        for i, f in enumerate(FOCALS):
            L.dist[i].model, L.dist[i].focal = dist, f
            for k, t in enumerate(DIST_TERMS[dist][i]):
                L.dist[i].terms[k] = t
    if tca != ab.LS_TCA_NONE:
        L.n_tca = len(FOCALS)
        for i, f in enumerate(FOCALS):
            L.tca[i].model, L.tca[i].focal = tca, f
            for k, t in enumerate(TCA_TERMS[tca][i]):
                L.tca[i].terms[k] = t
    if vig:
        n = 0
        for f in FOCALS:
            for ap, k1 in ((4.0, -0.42), (8.0, -0.21)):
                for dist_m in (1.0, 1000.0):
                    c = L.vig[n]
                    c.model, c.focal, c.aperture, c.distance = ab.LS_VIG_PA, f, ap, dist_m
                    c.terms[0], c.terms[1], c.terms[2] = k1 * (24.0 / f), 0.11 * (24.0 / f), -0.03
                    n += 1
        L.n_vig = n
    if real_focal:
        L.n_real_focal = 3
        for i, (f, rf) in enumerate(((18.0, 17.1), (35.0, 33.9), (55.0, 53.0))):
            L.real_focal[i].focal, L.real_focal[i].real_focal = f, rf
    return d


def frame(w: int, h: int, seed: int, extremes: bool = True) -> np.ndarray:
    """RGBA: ramps and noise over [-0.1, 1.5] with a grid of edges, and where `extremes`, NaN, +-inf, negatives and subnormals"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.empty((h, w, 4), np.float32)
    for c in range(4):
        img[..., c] = (x / max(w - 1, 1)) * (0.4 + 0.2 * c) + (y / max(h - 1, 1)) * (0.7 - 0.1 * c) + 0.3 * (((x // 7 + y // 5) % 2) - 0.5)
    img += rng.normal(0.0, 0.03, img.shape).astype(np.float32)
    if extremes:
        special = np.array([np.nan, np.inf, -np.inf, -0.3, 1e-40, -1e-40, 0.0, -0.0, 3e38, 1e-38], np.float32)
        mask = rng.random(img.shape) < 0.02
        img[mask] = rng.choice(special, int(mask.sum()))
    return np.ascontiguousarray(img)


def same_bits(a, b):
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _args(img, out, d, roi):
    ix, iy, iw, ih, ox, oy, ow, oh, s, bw, bh = roi
    return [util.fptr(img), util.fptr(out), C.byref(d)], [ix, iy, iw, ih, C.c_double(s), ox, oy, ow, oh, bw, bh]


def fill(roi, seed=3):
    """the caller's output buffer: what lane 3 keeps where the module leaves it"""
    ow, oh = roi[6], roi[7]
    return np.random.default_rng(seed).uniform(-2.0, 2.0, (oh, ow, 4)).astype(np.float32)


def oracle(img, d, itor, roi, monochrome=0, mask=0):
    out = fill(roi)
    head, tail = _args(img, out, d, roi)
    rc = util.oracle().orc_lens(*head, itor, monochrome, mask, *tail)
    return rc, out


def emul_lib():
    if "emul_lens" not in util._cache:
        so = os.path.join(EMUL, "libemul_lens.so")
        srcs = [os.path.join(EMUL, "emul_lens.cpp"), os.path.join(EMUL, "cuda_on_cpu.h"), os.path.join(util.ROOT, "ansel_b200", "csrc", "lens.cu"),
                os.path.join(util.ROOT, "ansel_b200", "csrc", "interp_taps.cuh"), os.path.join(util.ROOT, "include", "b200iop.h")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.run(["g++", "-O1", "-std=c++17", "-fno-fast-math", "-ffp-contract=off", "-I", EMUL, "-shared", "-fPIC", "-o", so, srcs[0]],
                           check=True)
        util._cache["emul_lens"] = C.CDLL(so)
    return util._cache["emul_lens"]


def emul(img, d, itor, roi, monochrome=0, mask=0):
    out = fill(roi)
    head, tail = _args(img, out, d, roi)
    rc = emul_lib().emul_lens(*head, itor, monochrome, mask, *tail)
    return rc, out


def ref_lib(kind: str = "strict"):
    """oracle/_ref/libref_lens_{kind}.so, built from /root/reference where it exists; None when it was never built"""
    key = "lens_" + kind
    if key not in util._cache:
        if os.path.isdir("/root/reference/src"):
            subprocess.run(["make", "-s", "-C", util.ORACLE_DIR, "-f", "lens.mk"], check=True)
        path = os.path.join(util.ORACLE_DIR, "_ref", f"libref_lens_{kind}.so")
        util._cache[key] = C.CDLL(path) if os.path.exists(path) else None
    return util._cache[key]


def ref(img, d, itor, roi, monochrome=0, mask=0, kind="strict"):
    lib = ref_lib(kind)
    util.oracle().orc_fp_fast_mode()   # FTZ|DAZ on this thread, as the reference's pipe threads have it (darktable.c:877)
    src = util.aligned_empty(img.shape)
    src[...] = img
    out = util.aligned_empty((roi[7], roi[6], 4))
    out[...] = fill(roi)
    head, tail = _args(src, out, d, roi)
    rc = lib.ref_lens(*head, ITORS[itor], monochrome, mask, *tail)
    return rc, np.array(out)


def plans(d, w, h, monochrome=0):
    """(modflags, eval bytes) of the library, the oracle, the emulated plan and (where built) the reference"""
    res = {}
    for name, fn in (("lib", ab.lib().b200_lens_plan), ("oracle", util.oracle().orc_lens_plan), ("emul", emul_lib().emul_lens_plan)):
        mf, ev = C.c_int(-1), ab.LensEval()
        assert fn(C.byref(d), w, h, monochrome, C.byref(mf), C.byref(ev)) == 0
        res[name] = (mf.value, bytes(ev))
    r = ref_lib("strict")
    if r is not None:
        mf, ev = C.c_int(-1), ab.LensEval()
        r.ref_lens_plan(C.byref(d), w, h, monochrome, C.byref(mf), C.byref(ev))
        res["ref"] = (mf.value, bytes(ev))
    return res


def piece(roi, lp, *, monochrome=0, mask=0, devid=0):
    ix, iy, iw, ih, ox, oy, ow, oh, s, bw, bh = roi
    p = ab.make_piece(iw, ih, filters=0, channels=4, roi_x=ix, roi_y=iy, out_width=ow, out_height=oh, scale=s, devid=devid)
    p.roi_out.x, p.roi_out.y = ox, oy
    p.buf_in_width, p.buf_in_height = bw, bh
    p.mask_display = mask
    p.image_flags = ab.IMAGE_MONOCHROME if monochrome else 0
    p.data, p.data_size = C.addressof(lp), C.sizeof(lp)
    p._keepalive = lp
    return p
