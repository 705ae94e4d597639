"""GPU parity: non-local means (exact replay of the reference's accumulation order) against the oracle,
bit for bit; the oracle is bit-identical to the reference's nlmeans_core.c compiled in place."""
import ctypes as C

import numpy as np
import pytest

import util

pytestmark = pytest.mark.gpu


def same_bits(a, b):
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def cuda_nlm(img, *, scattering=0.0, scale=1.0, luma=1.0, chroma=1.0, center_weight=0.1, sharpness=0.005, P=1, K=7, decimate=0,
             norm=(1.0, 1.0, 1.0, 1.0)):
    import torch
    import ansel_b200 as ab
    ab.init()
    h, w = img.shape[:2]
    d_in = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    d_out = torch.zeros_like(d_in)
    ab.check(ab.lib().b200_nlmeans_denoise_dev(d_in.data_ptr(), d_out.data_ptr(), w, h, scattering, scale, luma, chroma, center_weight,
                                               sharpness, P, K, decimate, (C.c_float * 4)(*norm), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return d_out.cpu().numpy()


CONFIGS = [dict(), dict(P=2, K=4, scattering=0.5), dict(center_weight=-1.0, sharpness=0.01, luma=0.8, chroma=0.6, K=3, P=3),
           dict(K=2, P=1, scattering=1.0, scale=0.7), dict(P=4, K=2), dict(P=0, K=3), dict(K=5, decimate=1)]


@pytest.mark.parametrize("cfg", range(len(CONFIGS)))
@pytest.mark.parametrize("size", [(200, 150), (73, 61), (301, 203), (145, 121), (17, 9)])
def test_nlmeans_core_bit_exact(built, size, cfg):
    w, h = size
    img = (util.rgba_scene(w, h, 2, noise=0.02) * 60).astype(np.float32)
    kw = CONFIGS[cfg]
    got = cuda_nlm(img, **kw)
    want = util.oracle_nlmeans(img, **kw)
    bad = ~same_bits(got, want)
    assert not bad.any(), f"{int(bad.sum())} floats differ, first {np.argwhere(bad)[:4].tolist()}"


def run_module(img, data, pipe_type=1, mask_display=0):
    import torch
    import ansel_b200 as ab
    ab.init()
    h, w = img.shape[:2]
    piece = ab.make_piece(w, h, filters=0, channels=4, data=data, devid=0, pipe_type=pipe_type)
    piece.mask_display = mask_display
    d_in = torch.from_numpy(img).cuda()
    d_out = torch.zeros_like(d_in)
    ab.check(ab.lib().b200_denoiseprofile_process_dev(piece, d_in.data_ptr(), d_out.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return d_out.cpu().numpy()


def oracle_module(img, data, pipe_type=1, wb=(2.0, 1.0, 1.5, 0.0), pm=(1.0, 1.0, 1.0, 1.0)):
    h, w = img.shape[:2]
    out = np.zeros_like(img)
    f = util.oracle().orc_denoiseprofile_nlmeans
    f.restype = C.c_int
    assert f(util.fptr(img), util.fptr(out), w, h, C.byref(data), C.c_float(1.0), pipe_type, (C.c_float * 4)(*wb), (C.c_float * 4)(*pm)) == 0
    return out


@pytest.mark.parametrize("new_vst,pipe", [(True, 1), (False, 1), (True, 4)])
def test_denoiseprofile_nlmeans_module_bit_exact(built, new_vst, pipe):
    """SURVEY.md 8d config C3: mode NLMEANS, radius 1, nbhood 7, scattering 0, strength 1, cpw 0.1."""
    import ansel_b200 as ab
    img = util.rgba_scene(900, 600, 5)
    data = ab.denoiseprofile_data(ab.DENOISE_NLMEANS, use_new_vst=new_vst)
    got = run_module(img, data, pipe)
    want = oracle_module(img, data, pipe)
    assert same_bits(got, want).all()
    assert np.abs(np.diff(got[..., 1], axis=1)).mean() < 0.9 * np.abs(np.diff(img[..., 1], axis=1)).mean()


def test_denoiseprofile_nlmeans_keeps_the_alpha_of_a_displayed_mask(built):
    """process_nlmeans_cpu() ends with dt_iop_alpha_copy() when the pipe displays a mask (denoiseprofile.c:1645-1646)."""
    import ansel_b200 as ab
    img = util.rgba_scene(300, 200, 6)
    img[..., 3] = np.random.default_rng(6).random((200, 300), dtype=np.float32)
    data = ab.denoiseprofile_data(ab.DENOISE_NLMEANS)
    shown = run_module(img, data, mask_display=1)
    plain = run_module(img, data)
    assert same_bits(shown[..., 3], img[..., 3]).all()
    assert same_bits(shown[..., :3], plain[..., :3]).all()
    assert same_bits(plain, oracle_module(img, data)).all()


def test_nlmeans_24mp_bit_exact(built):
    w, h = util.SIZE_24MP
    img = (util.rgba_scene(w, h, util.SEEDS[1], noise=0.02) * 60).astype(np.float32)
    got = cuda_nlm(img)
    want = util.oracle_nlmeans(img)
    assert same_bits(got, want).all()


@pytest.mark.parametrize("kw", [dict(), dict(P=2, K=5), dict(center_weight=-1.0, sharpness=0.01, luma=0.8, chroma=0.6, K=4, P=2, norm=(0.7, 1.3, 0.9, 1.0))])
def test_nlmeans_full_width_strip_bit_exact(built, kw):
    """a strip as wide as the 45 MP bench frame: the chunk grid across the row (114 full columns + the 48-px remainder) and the
    group kernel's window at the right edge are the frame's own"""
    w, h = util.SIZE_45MP[0], 600
    img = (util.rgba_scene(w, h, 7, noise=0.02) * 60).astype(np.float32)
    got = cuda_nlm(img, **kw)
    want = util.oracle_nlmeans(img, **kw)
    bad = ~same_bits(got, want)
    assert not bad.any(), f"{int(bad.sum())} floats differ, first {np.argwhere(bad)[:4].tolist()}"


def test_chunk_kernel_is_bit_exact_too(built, monkeypatch):
    """the round-1 kernel (one chunk per CTA, patches one after the other): what runs where the group kernel's window does not fit"""
    monkeypatch.setenv("B200_NLM_CHUNKS", "1")
    for cfg in (0, 1, 4, 6):
        img = (util.rgba_scene(301, 203, 2, noise=0.02) * 60).astype(np.float32)
        kw = CONFIGS[cfg]
        assert same_bits(cuda_nlm(img, **kw), util.oracle_nlmeans(img, **kw)).all(), cfg


def test_extreme_pixels_through_the_group_kernel(built):
    """zeros (weights of exactly 1), infinities, NaN, values next to FLT_MAX and subnormals: Markstein's division, the clamp in
    front of it and the packed lanes must leave what the reference leaves (tests/test_cpu_nlm_emulation.py has the same frame).
    130 rows cut into chunks of 65: too tall for the pipelined kernel (64 rows at most), so this frame runs through the group kernel;
    tests/test_zz_nlm_routes_gpu.py puts the same specials through the pipelined kernel's half-height slots"""
    img = (util.rgba_scene(160, 130, 4, noise=0.02) * 60).astype(np.float32)
    img[20:60, 30:90, :3] = 0.0
    img[70:90, 10:50, :3] = 1e-30
    img[100, 100, :3] = (np.inf, 1.0, 2.0)
    img[101, 120, :3] = (np.nan, 1.0, 2.0)
    img[110, 20, :3] = (3e38, -3e38, 1e19)
    img[5, 5, :3] = (1e-40, 1e-44, 0.0)
    for kw in (dict(K=3), dict(K=3, center_weight=-1.0, sharpness=0.01), dict(K=2, P=2, norm=(0.5, 2.0, 1.5, 1.0))):
        bad = ~same_bits(cuda_nlm(img, **kw), util.oracle_nlmeans(img, **kw))
        assert not bad.any(), f"{kw}: {int(bad.sum())} floats differ, first {np.argwhere(bad)[:4].tolist()}"


def test_window_kernel_is_bit_exact_too(built, monkeypatch):
    """the shared-memory-window variant of the chunk kernel (B200_NLM_WINDOW=1) against the same oracle"""
    monkeypatch.setenv("B200_NLM_WINDOW", "1")
    for cfg in (0, 1, 2, 6):
        img = (util.rgba_scene(301, 203, 2, noise=0.02) * 60).astype(np.float32)
        kw = CONFIGS[cfg]
        assert same_bits(cuda_nlm(img, **kw), util.oracle_nlmeans(img, **kw)).all(), cfg
