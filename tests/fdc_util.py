"""Helpers of the FDC (frequency-domain chroma, X-Trans) tests: the reference's lines compiled in place (oracle/_ref/libref_fdc_{strict,fast}.so
from oracle/fdc.mk), the oracle (oracle/restate/fdc_oracle.c), the kernel's stages compiled with g++ (tests/emul/emul_fdc.cpp) and the CUDA path."""
import ctypes as C
import os
import subprocess

import numpy as np

import util
from vng_util import XTRANS

XOVER = 1600  # the preference's default, data/anselconfig.xml.in:1814
# (width, height, x, y): one tile (the reference's first tile covers 96 px), several tiles in both directions, ROI phases 0..5, widths that are
# not a multiple of 6, and a frame just above the smallest the reference can mirror
CASES = {"one_tile": (96, 90, 0, 0), "multi": (300, 210, 0, 0), "roi": (197, 131, 1, 4), "roi2": (250, 148, 3, 2), "phase": (103, 211, 5, 5),
         "narrow": (40, 230, 4, 1), "small": (30, 17, 2, 3)}
ISOS = (100.0, 1600.0, 1600.9, 3200.0)  # hybrid, hybrid (at the crossover; the reference compares int(iso)), hybrid, pure


def case(name, seed=6, special=True):
    w, h, x, y = CASES[name]
    m = util.frame_natural(w, h, seed)
    if special and h > 40 and w > 30:
        m[20, 8] = 0.0
        m[30, 21] = np.nan
        m[25, 14] = np.inf
        m[11, 27] = -np.inf
        m[17, 19] = -0.125
        m[22, 25] = 1e-41          # subnormal: flushed by DAZ
        m[33, 9] = -0.0
    if h > 70 and w > 70:
        m[40:52, 40:52] = 0.25     # a flat patch
        m[55:65, 10:22] = 0.0      # a black patch: the maxima of green are 0.0f, the loop's marker of a new pair
    return np.ascontiguousarray(m, np.float32), x, y


def _prep(m):
    h, w = m.shape
    out, src = util.aligned_empty((h, w, 4)), util.aligned_empty(m.shape)
    out[...] = -7.0
    src[...] = m
    return out, src, np.ascontiguousarray(XTRANS)


def oracle(m, x=0, y=0, iso=100.0, xover=XOVER, zero_per_tile=1, fill=0):
    out, src, xt = _prep(m)
    h, w = m.shape
    f = util.oracle().orc_fdc
    f.restype = None
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_float, C.c_int, C.c_int, C.c_int]
    f(out.ctypes.data, src.ctypes.data, w, h, x, y, xt.ctypes.data, iso, xover, zero_per_tile, fill)
    return np.array(out)


_REF = {}


def ref_lib(kind="strict"):
    """None where the reference is not built and cannot be"""
    if kind not in _REF:
        so = os.path.join(util.ORACLE_DIR, "_ref", f"libref_fdc_{kind}.so")
        if os.path.isdir("/root/reference/src"):
            subprocess.run(["make", "-s", "-C", util.ORACLE_DIR, "-f", "fdc.mk"], check=True)
        _REF[kind] = C.CDLL(so) if os.path.exists(so) else None
    return _REF[kind]


def ref(m, x=0, y=0, iso=100.0, xover=XOVER, fill=0, nthreads=1, kind="strict"):
    lib = ref_lib(kind)
    if lib is None:
        return None
    out, src, xt = _prep(m)
    h, w = m.shape
    f = lib.ref_fdc
    f.restype = None
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_float, C.c_int, C.c_int, C.c_int]
    f(out.ctypes.data, src.ctypes.data, w, h, x, y, xt.ctypes.data, iso, xover, fill, nthreads)
    return np.array(out)


def ref_tables():
    lib = ref_lib("strict")
    if lib is None:
        return None
    t = np.zeros(3 * 8 * 2, np.float32), np.zeros(6 * 6 * 8 * 2, np.float32), np.zeros(4 * 13 * 13 * 2, np.float32)
    lib.ref_fdc_tables(*(a.ctypes.data for a in t))
    return t


_EMUL = None


def emul_lib():
    """ansel_b200/csrc/markesteijn.cu (FDC instance) compiled with g++ (tests/emul/emul_fdc.cpp)"""
    global _EMUL
    if _EMUL is None:
        here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
        so = os.path.join(here, "libemul_fdc.so")
        csrc = os.path.join(here, "..", "..", "ansel_b200", "csrc")
        srcs = [os.path.join(here, "emul_fdc.cpp"), os.path.join(here, "cuda_on_cpu.h"), os.path.join(csrc, "markesteijn.cu"),
                os.path.join(csrc, "fdc_tables.h")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.run(["g++", "-O1", "-std=c++17", "-fno-fast-math", "-ffp-contract=off", "-I", here, "-shared", "-fPIC", "-o", so, srcs[0]], check=True)
        _EMUL = C.CDLL(so)
    return _EMUL


def emul(m, x=0, y=0, iso=100.0, xover=XOVER, nthreads=96, ascending=0):
    """the kernel's stages run thread by thread on the CPU, the threads of a stage in descending (or ascending) order"""
    out, src, xt = _prep(m)
    h, w = m.shape
    f = emul_lib().emul_fdc
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int]
    pure = int(int(iso) > xover)  # iop/demosaic/markesteijn.c:1138-1139: int iso = exif_iso; pure FDC if iso > xover_iso
    assert f(out.ctypes.data, src.ctypes.data, w, h, x, y, xt.ctypes.data, pure, nthreads, ascending) == 0
    return np.array(out)


def same_bits(a, b):
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def differing(a, b):
    """pixels whose three colour lanes are not all the same bits"""
    return int((~same_bits(a[..., :3], b[..., :3])).any(axis=-1).sum())
