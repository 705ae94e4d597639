"""CPU: nlm_pipe_kernel's half-height path on its 64-bit shared-memory layout (the paired window, the interleaved patch-pair slots:
pipe2_* in ansel_b200/csrc/nlm_group.cuh) compiled with g++ and run thread by thread in the kernel's barrier order, against the oracle
bit for bit.  Test infrastructure only; the `-m gpu` tests run the same path through nvcc."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import util

SMEM = 232448  # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100 (227 KB)


@pytest.fixture(scope="module")
def emul():
    emul_dir = os.path.join(util.ROOT, "tests", "emul")
    csrc = os.path.join(util.ROOT, "ansel_b200", "csrc")
    so = os.path.join(emul_dir, "libemul_nlm_pipe2.so")
    srcs = [os.path.join(emul_dir, "emul_nlm_pipe2.cpp"), os.path.join(emul_dir, "cuda_on_cpu.h"), os.path.join(csrc, "nlm.cu"),
            os.path.join(csrc, "nlm_group.cuh"), os.path.join(csrc, "packed_f32.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fno-fast-math", "-ffp-contract=off", "-mfma", "-I", emul_dir, "-shared", "-fPIC", "-o", so,
                        srcs[0]], check=True)
    return C.CDLL(so)


def run(lib, img, *, scattering=0.0, scale=1.0, luma=1.0, chroma=1.0, center_weight=0.1, sharpness=0.005, K=7, decimate=0,
        norm=(1.0, 1.0, 1.0, 1.0), ieee_div=0):
    """(chunks that took the half-height slots, output)"""
    h, w = img.shape[:2]
    src = np.ascontiguousarray(img)
    out = np.full_like(src, np.nan)
    before = C.c_int.in_dll(lib, "emul_nlm_pipe2_chunks").value
    ok = lib.emul_nlmeans_pipe2(util.fptr(src), util.fptr(out), w, h, C.c_float(scattering), C.c_float(scale), C.c_float(luma), C.c_float(chroma),
                                C.c_float(center_weight), C.c_float(sharpness), K, decimate, (C.c_float * 4)(*norm), SMEM, ieee_div)
    assert ok, "the pipelined kernel does not take this configuration"
    return C.c_int.in_dll(lib, "emul_nlm_pipe2_chunks").value - before, out


def check(lib, img, **kw):
    halves, got = run(lib, img, **kw)
    want = util.oracle_nlmeans(img, P=1, **{k: v for k, v in kw.items() if k != "ieee_div"})
    bad = ~((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want)))
    assert not bad.any(), f"{kw}: {int(bad.sum())} floats differ, first {np.argwhere(bad)[:4].tolist()}"
    return halves


# every patch count here is odd ((2K + 1)^2, or (2K^2 + 2K + 1) decimated): the last pair's twin is itself
@pytest.mark.parametrize("blend", [False, True])
@pytest.mark.parametrize("kw", [dict(K=0), dict(K=1), dict(K=1, decimate=1), dict(K=2), dict(K=3), dict(K=7),
                                dict(K=3, center_weight=-1.0, sharpness=0.01), dict(K=2, norm=(0.7, 1.3, 0.9, 1.0)),
                                dict(K=2, center_weight=0.37, sharpness=0.02, ieee_div=1)],
                         ids=lambda kw: ",".join(f"{k}={v}" for k, v in kw.items()))
def test_half_height_path_equals_oracle(emul, kw, blend):
    """360 x 256 cuts into 64-row chunks; those off the frame's rim take the half-height slots (none at K = 0: one patch)"""
    img = (util.rgba_scene(360, 256, 5, noise=0.02) * 60).astype(np.float32)
    if blend:
        kw = dict(kw, luma=0.8, chroma=0.6)
    halves = check(emul, img, **kw)
    assert (halves > 0) == (kw["K"] > 0)


def test_extreme_pixels_in_half_height_chunks(emul):
    """zeros (weights of exactly 1), subnormals, a saturated patch, infinities and NaN inside the chunks that take the half-height slots"""
    img = (util.rgba_scene(220, 192, 4, noise=0.02) * 60).astype(np.float32)
    img[70:110, 40:100, :3] = 0.0
    img[120:128, 20:60, :3] = 1e-30
    img[80, 100, :3] = (np.inf, 1.0, 2.0)
    img[101, 120, :3] = (np.nan, 1.0, 2.0)
    img[90, 70, :3] = (3e38, -3e38, 1e19)
    img[100, 150, :3] = (-np.inf, 1e-40, 1e-44)
    for kw in (dict(K=3), dict(K=3, center_weight=-1.0, sharpness=0.01), dict(K=2, norm=(0.5, 2.0, 1.5, 1.0), luma=0.5)):
        assert check(emul, img, **kw) > 0


def test_half_height_layout_has_no_bank_conflicts():
    """tools/nlm_pipe_banks.py on the kernel's pitches: every hot access of the half-height path, every shift of K = 7"""
    r = subprocess.run([sys.executable, os.path.join(util.ROOT, "tools", "nlm_pipe_banks.py")], capture_output=True, text=True)
    assert r.returncode == 0 and "no conflicted access" in r.stdout, r.stdout
