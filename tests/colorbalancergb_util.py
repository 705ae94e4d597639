"""colour balance rgb (src/iop/colorbalancergb.c) through the checkers: the oracle (oracle/restate/colorbalancergb_oracle.c), the reference's own
lines compiled in place (oracle/_ref/libref_colorbalancergb_{strict,fast}.so from oracle/colorbalancergb.mk, whose commit_params() also makes
the data blocks and gamut LUTs) and the product's kernel under g++ (tests/emul/emul_colorbalancergb.cpp).  Checkers only."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import util
import ansel_b200 as ab

EMUL = os.path.join(util.ROOT, "tests", "emul")
ADOBE_TO_XYZ_D50 = np.array([[0.6097559, 0.2052401, 0.1492240], [0.3111242, 0.6256560, 0.0632197], [0.0194811, 0.0608902, 0.7448387]])
PROFILES = {"rec2020": util.profile_pair(util.REC2020_TO_XYZ_D50), "srgb": util.profile_pair(util.SRGB_TO_XYZ_D50),
            "adobergb": util.profile_pair(ADOBE_TO_XYZ_D50)}
FORMULAS = (ab.COLORBALANCE_SATURATION_JZAZBZ, ab.COLORBALANCE_SATURATION_DTUCS)

_P = ("shadows_Y", "shadows_C", "shadows_H", "midtones_Y", "midtones_C", "midtones_H", "highlights_Y", "highlights_C", "highlights_H",
      "global_Y", "global_C", "global_H", "shadows_weight", "white_fulcrum", "highlights_weight", "chroma_shadows", "chroma_highlights",
      "chroma_global", "chroma_midtones", "saturation_global", "saturation_highlights", "saturation_midtones", "saturation_shadows",
      "hue_angle", "brilliance_global", "brilliance_highlights", "brilliance_midtones", "brilliance_shadows", "mask_grey_fulcrum", "vibrance",
      "grey_fulcrum", "contrast")
# $MIN / $MAX of dt_iop_colorbalancergb_params_t (colorbalancergb.c:88-134)
RANGES = {"shadows_H": (0, 360), "midtones_H": (0, 360), "highlights_H": (0, 360), "global_H": (0, 360), "shadows_C": (0, 1), "midtones_C": (0, 1),
          "highlights_C": (0, 1), "global_C": (0, 1), "shadows_weight": (0, 3), "highlights_weight": (0, 3), "white_fulcrum": (-16, 16),
          "hue_angle": (-180, 180), "mask_grey_fulcrum": (0, 1), "grey_fulcrum": (0, 1)}


class Params(C.Structure):
    """dt_iop_colorbalancergb_params_t (colorbalancergb.c:88-134): the user parameters commit_params() reads."""
    _fields_ = [(n, C.c_float) for n in _P] + [("saturation_formula", C.c_int)]


def defaults() -> Params:
    p = Params()
    p.shadows_weight = p.highlights_weight = p.white_fulcrum = 1.0
    p.mask_grey_fulcrum = p.grey_fulcrum = 0.1845
    p.saturation_formula = ab.COLORBALANCE_SATURATION_DTUCS
    return p


def presets():
    """the five presets of init_presets (colorbalancergb.c:461-505), the last one the scene-referred default"""
    out = []
    p = defaults()
    p.saturation_formula = ab.COLORBALANCE_SATURATION_JZAZBZ
    p.chroma_global, p.saturation_shadows, p.saturation_midtones, p.saturation_highlights = 0.2, 0.1, 0.05, -0.05
    out.append(("basic colorfulness (legacy)", p))
    for name, shadows in (("natural skin", 0.30), ("vibrant colors", 0.5), ("standard", 0.25), ("scene-referred default", 0.25)):
        q = Params.from_buffer_copy(p)
        q.saturation_formula = ab.COLORBALANCE_SATURATION_DTUCS
        q.chroma_global = 0.0
        q.saturation_global, q.saturation_shadows, q.saturation_midtones, q.saturation_highlights = 0.2, shadows, 0.0, 0.0
        out.append((name, q))
    return out


# sub-ranges that keep a frame alive: over the full ranges, saturation and brilliance sums often drive max_zero(1 + ...) to 0 and
# extreme white fulcrums darken the rest, so many full-range blocks give (nearly) black frames
MODERATE = {"white_fulcrum": (-2, 3), "shadows_weight": (0.5, 2), "highlights_weight": (0.5, 2), "mask_grey_fulcrum": (0.1, 0.3),
            "grey_fulcrum": (0.1, 0.3)}


def random_params(rng, formula, moderate: bool = False) -> Params:
    """a block drawn over the $MIN..$MAX ranges, or (moderate) over sub-ranges: the [-1, 1] and [0, 1] parameters scaled by 0.3"""
    p = Params()
    for n in _P:
        lo, hi = RANGES.get(n, (-1, 1))
        if moderate:
            lo, hi = MODERATE.get(n, (lo, hi) if n.endswith("_H") or n == "hue_angle" else (0.3 * lo, 0.3 * hi))
        setattr(p, n, float(rng.uniform(lo, hi)))
    p.saturation_formula = formula
    return p


def blocks():
    """the parameter matrix: the five presets, 120 blocks over the full ranges and 40 over the moderate sub-ranges, both formulas"""
    rng = np.random.default_rng(20261019)
    out = [(name, p) for name, p in presets()]
    out += [(f"random {k}", random_params(rng, FORMULAS[k % 2])) for k in range(120)]
    out += [(f"moderate {k}", random_params(rng, FORMULAS[k % 2], moderate=True)) for k in range(40)]
    return out


def hue_frame(w: int, h: int, seed: int) -> np.ndarray:
    """RGBA of saturated colours at random hues and brightnesses: the gamut lookup meets every part of the hue circle, its wrap included"""
    rng = np.random.default_rng(seed)
    rgb = rng.random((h, w, 3), dtype=np.float32)
    rgb = rgb ** 3 * rng.choice(np.float32([0.1, 0.5, 1.0, 3.0]), (h, w, 1))
    return np.ascontiguousarray(np.concatenate([rgb, rng.random((h, w, 1), dtype=np.float32)], axis=2))


def frame(w: int, h: int, seed: int) -> np.ndarray:
    """RGBA: a smooth scene with saturated patches up to 4x white, a grey ramp (zero chroma) and NaN, +-inf, negatives, subnormals"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.empty((h, w, 4), np.float32)
    for c in range(3):
        img[..., c] = 0.02 + 0.9 * (0.5 + 0.5 * np.sin(x * (0.11 + 0.05 * c) + y * (0.07 - 0.02 * c) + c))
    img[..., :3] *= rng.choice(np.float32([0.05, 0.2, 1.0, 4.0]), (h, w, 1))
    img[..., 3] = rng.uniform(0, 1, (h, w))
    img[: h // 6, :, :3] = (x[: h // 6, :, None] / max(w - 1, 1)) * 1.5    # greys
    special = np.array([np.nan, np.inf, -np.inf, -0.3, 1e-40, -1e-40, 0.0, -0.0, 3e38, 1e-38, 7.5], np.float32)
    mask = rng.random(img.shape) < 0.03
    img[mask] = rng.choice(special, int(mask.sum()))
    return np.ascontiguousarray(img)


def same_bits(a, b):
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def ref_lib(kind: str = "strict"):
    """oracle/_ref/libref_colorbalancergb_{kind}.so, built from /root/reference where it exists; None when it was never built"""
    key = "colorbalancergb_" + kind
    if key not in util._cache:
        if os.path.isdir("/root/reference/src"):
            subprocess.run(["make", "-s", "-C", util.ORACLE_DIR, "-f", "colorbalancergb.mk"], check=True)
        path = os.path.join(util.ORACLE_DIR, "_ref", f"libref_colorbalancergb_{kind}.so")
        util._cache[key] = C.CDLL(path) if os.path.exists(path) else None
        if util._cache[key] is not None:
            util._cache[key].ref_colorbalancergb_layout.restype = C.c_size_t
    return util._cache[key]


def _m(a):
    return np.ascontiguousarray(a, np.float32)


def commit(p: Params, profile=None, lut_fill: float = 0.0, mask_display: int = 0, kind: str = "strict"):
    """(data block, LUT) as the reference's commit_params() leaves them; profile None: no work profile (the LUT stays the fill)"""
    data, lut = ab.ColorbalancergbData(), np.full(360, lut_fill, np.float32)
    mi, mo = (None, None) if profile is None else (_m(PROFILES[profile][0]), _m(PROFILES[profile][1]))
    util.oracle().orc_fp_fast_mode_all()
    ref_lib(kind).ref_colorbalancergb_commit(C.byref(p), C.byref(data), util.fptr(lut), None if mi is None else util.fptr(mi),
                                             None if mo is None else util.fptr(mo), C.c_float(lut_fill), mask_display, 0)
    return data, lut


def piece(data, profile: str, lut) -> ab.ColorbalancergbPiece:
    return ab.colorbalancergb_piece(data, PROFILES[profile], lut)


def ref(img, cp: ab.ColorbalancergbPiece, kind: str = "strict", fill: float = -7.0):
    h, w = img.shape[:2]
    src = util.aligned_empty(img.shape)
    src[...] = img
    out = util.aligned_empty(img.shape)
    out[...] = fill
    mi = _m(np.array(cp.work_profile.matrix_in)[:, :3])
    mo = _m(np.array(cp.work_profile.matrix_out)[:, :3])
    lut = _m(np.array(cp.gamut_LUT))
    util.oracle().orc_fp_fast_mode_all()
    rc = ref_lib(kind).ref_colorbalancergb(util.fptr(src), util.fptr(out), w, h, C.byref(cp.data), util.fptr(lut), util.fptr(mi), util.fptr(mo))
    return rc, np.array(out)


def oracle(img, cp, fill: float = -7.0):
    out = np.full(img.shape, fill, np.float32)
    rc = util.oracle().orc_colorbalancergb(util.fptr(img), util.fptr(out), C.c_size_t(img.size // 4), C.byref(cp))
    return rc, out


def emul_lib():
    if "emul_colorbalancergb" not in util._cache:
        so = os.path.join(EMUL, "libemul_colorbalancergb.so")
        srcs = [os.path.join(EMUL, "emul_colorbalancergb.cpp"), os.path.join(EMUL, "cuda_on_cpu.h"),
                os.path.join(util.ROOT, "ansel_b200", "csrc", "colorbalancergb.cu"), os.path.join(util.ROOT, "ansel_b200", "csrc", "flt32_math.cuh"),
                os.path.join(util.ROOT, "include", "b200iop.h")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.run(["g++", "-O1", "-std=c++17", "-fno-fast-math", "-ffp-contract=off", "-I", EMUL, "-shared", "-fPIC", "-o", so, srcs[0]],
                           check=True)
        util._cache["emul_colorbalancergb"] = C.CDLL(so)
    return util._cache["emul_colorbalancergb"]


def emul(img, cp, fill: float = -7.0):
    out = np.full(img.shape, fill, np.float32)
    rc = emul_lib().emul_colorbalancergb(util.fptr(img), util.fptr(out), C.c_size_t(img.size // 4), C.byref(cp))
    return rc, out


class AdapterData(C.Structure):
    """dt_iop_colorbalancergb_data_t as the module adapter receives it: the hashed prefix, then the runtime pointers (:187-191)"""
    _fields_ = [("prefix", ab.ColorbalancergbData), ("work_profile", C.c_void_p), ("gamut_LUT", C.POINTER(C.c_float)), ("chroma_LUT", C.c_void_p)]


def adapter_data(data, lut) -> AdapterData:
    d = AdapterData()
    C.memmove(C.addressof(d.prefix), bytes(data), C.sizeof(ab.ColorbalancergbData))
    d._lut = np.ascontiguousarray(lut, np.float32)  # noqa
    d.gamut_LUT = util.fptr(d._lut)
    return d
