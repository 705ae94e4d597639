"""CPU: the phases of the non-local-means group kernel (ansel_b200/csrc/nlm_group.cuh) compiled with g++ and run thread by
thread, phase after phase, against the oracle bit for bit -- the packed fast paths, the scalar edge paths, Markstein's
division and the product's own host-side plan.  What it cannot see is nvcc's code generation (the `-m gpu` tests do).
Test infrastructure only."""
import ctypes as C

import numpy as np
import pytest

import util

SMEM = 232448  # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100 (227 KB)


def same_bits(a, b):
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


@pytest.fixture(scope="module")
def emul():
    return util.emul_nlm()


def emul_nlm(lib, img, *, scattering=0.0, scale=1.0, luma=1.0, chroma=1.0, center_weight=0.1, sharpness=0.005, P=1, K=7, decimate=0,
             norm=(1.0, 1.0, 1.0, 1.0), smem=SMEM, g_cap=8, ieee_div=0, pipe=0):
    h, w = img.shape[:2]
    src = np.ascontiguousarray(img)
    out = np.full_like(src, np.nan)
    G = lib.emul_nlmeans_group(util.fptr(src), util.fptr(out), w, h, C.c_float(scattering), C.c_float(scale), C.c_float(luma), C.c_float(chroma),
                               C.c_float(center_weight), C.c_float(sharpness), P, K, decimate, (C.c_float * 4)(*norm), smem, g_cap, ieee_div, pipe)
    return G, out


# the parameter sets of tests/test_nlm_gpu.py that the group kernel takes (patch radius <= 2, window in shared memory), and more
CONFIGS = [dict(), dict(P=2, K=4, scattering=0.5), dict(K=2, P=1, scattering=1.0, scale=0.7), dict(P=2, K=3), dict(K=5, decimate=1),
           dict(center_weight=-1.0, sharpness=0.01, luma=0.8, chroma=0.6, K=3, P=2), dict(norm=(0.7, 1.3, 0.9, 1.0), K=3),
           dict(norm=(0.7, 1.3, 0.9, 1.0), K=2, P=2, center_weight=-1.0, sharpness=0.02), dict(center_weight=0.37, sharpness=0.02, K=3),
           dict(center_weight=0.0, K=2), dict(center_weight=3.0, sharpness=0.001, K=2, luma=0.5)]


@pytest.mark.parametrize("cfg", range(len(CONFIGS)))
@pytest.mark.parametrize("size", [(200, 150), (73, 61), (145, 121), (17, 9)])
def test_group_kernel_phases_equal_oracle(emul, size, cfg):
    w, h = size
    img = (util.rgba_scene(w, h, 2, noise=0.02) * 60).astype(np.float32)
    kw = CONFIGS[cfg]
    G, got = emul_nlm(emul, img, **kw)
    assert G >= 2
    want = util.oracle_nlmeans(img, **kw)
    bad = ~same_bits(got, want)
    assert not bad.any(), f"G={G}: {int(bad.sum())} floats differ, first {np.argwhere(bad)[:4].tolist()}"


@pytest.mark.parametrize("slots", [1, 2])
@pytest.mark.parametrize("cfg", range(len(CONFIGS)))
@pytest.mark.parametrize("size", [(200, 150), (73, 61), (145, 121), (301, 128), (360, 256), (220, 192)])
def test_pipelined_kernel_phases_equal_oracle(emul, size, cfg, slots):
    """the same phases in the pipelined kernel's order: a patch pair per slot of the ring, 256 accumulating threads with 9 pixel pairs each
    (strip ownership).  slots 1: half-height slots in the 64-row chunks of the frame's interior (heights 256 and 192 cut into such chunks; the
    other sizes, and every chunk on the rim, take the whole-pair slots); slots 2: whole-pair slots everywhere"""
    w, h = size
    img = (util.rgba_scene(w, h, 5, noise=0.02) * 60).astype(np.float32)
    kw = CONFIGS[cfg]
    before = C.c_int.in_dll(emul, "emul_nlm_halves_chunks").value
    G, got = emul_nlm(emul, img, pipe=slots, **kw)
    took_halves = C.c_int.in_dll(emul, "emul_nlm_halves_chunks").value - before
    if G == -1:
        pytest.skip("the pipelined kernel does not take this configuration (wide window or tall chunks)")
    bad = ~same_bits(got, util.oracle_nlmeans(img, **kw))
    assert not bad.any(), f"{int(bad.sum())} floats differ, first {np.argwhere(bad)[:4].tolist()}"
    if slots == 2 or kw.get("P", 1) != 1:
        assert took_halves == 0
    elif size in ((360, 256), (220, 192)) and kw.get("K", 7) <= 7 and not kw.get("scattering"):
        assert took_halves > 0, "no chunk took the half-height slots"


@pytest.mark.parametrize("g_cap,ieee", [(2, 0), (4, 1), (6, 0)])
def test_patches_in_flight_and_division_do_not_matter(emul, g_cap, ieee):
    img = (util.rgba_scene(301, 203, 3, noise=0.02) * 60).astype(np.float32)
    G, got = emul_nlm(emul, img, g_cap=g_cap, ieee_div=ieee)
    assert G == g_cap
    assert same_bits(got, util.oracle_nlmeans(img)).all()


def test_flat_dark_and_extreme_pixels(emul):
    """zeros (weights of exactly 1), a saturated patch, infinities and NaN: the division sequence and the packed lanes
    must leave what the reference leaves"""
    img = (util.rgba_scene(160, 130, 4, noise=0.02) * 60).astype(np.float32)
    img[20:60, 30:90, :3] = 0.0
    img[70:90, 10:50, :3] = 1e-30
    img[100, 100, :3] = (np.inf, 1.0, 2.0)
    img[101, 120, :3] = (np.nan, 1.0, 2.0)
    img[110, 20, :3] = (3e38, -3e38, 1e19)
    img[5, 5, :3] = (1e-40, 1e-44, 0.0)
    for kw in (dict(K=3), dict(K=3, center_weight=-1.0, sharpness=0.01), dict(K=2, P=2, norm=(0.5, 2.0, 1.5, 1.0))):
        G, got = emul_nlm(emul, img, **kw)
        want = util.oracle_nlmeans(img, **kw)
        bad = ~same_bits(got, want)
        assert not bad.any(), f"{kw}: {int(bad.sum())} floats differ, first {np.argwhere(bad)[:4].tolist()}"


def test_plan_refuses_what_does_not_fit(emul):
    img = (util.rgba_scene(100, 80, 2) * 60).astype(np.float32)
    assert emul_nlm(emul, img, P=3, K=2)[0] == 0          # rings of 7 rows: the chunk kernel keeps them
    assert emul_nlm(emul, img, P=0, K=3)[0] == 0          # single-pixel patches: the chunk kernel keeps them
    assert emul_nlm(emul, img, K=7, scattering=1.0)[0] == 0  # shifts of 85 px: no window
    assert emul_nlm(emul, img, smem=48 * 1024)[0] == 0
