"""GPU: every b200_<op>_process_host gives, byte for byte, what b200_<op>_process_dev gives on device copies of the same buffers.
Both outputs start from the same sentinel bytes, so the cases where the module leaves part of its output as it finds it (an unhandled
adaptation of colour calibration, gamma's fourth byte, temperature on non-RGBA pixels, demosaic on frames under 16 px and with PPG) check
that the host entry carries the caller's buffer to the device."""
import ctypes as C
import os

import numpy as np
import pytest

import util

pytestmark = pytest.mark.gpu

W, H = 64, 48
WORK = util.profile_pair(util.REC2020_TO_XYZ_D50)
EXPORT = util.profile_pair(util.SRGB_TO_XYZ_D50)


def _rgba(ab, data):
    return ab.make_piece(W, H, filters=0, channels=4, data=data), util.rgba_test_image(W, H, 4), W * H * 16


def _mosaic(ab, data, w=W, h=H):
    p = ab.make_piece(w, h, data=data)
    p.datatype = ab.TYPE_FLOAT
    return p, util.frame_natural(w, h, 5), w * h * 4


def _struct(piece, data):
    piece.data, piece.data_size = C.addressof(data), C.sizeof(data)
    piece._keepalive = data
    return piece


def cases(ab):
    """name -> (op, piece, input, output bytes, whether sentinel bytes must survive in the output)"""
    conv_in = ab.make_conversion(util.MATRIX_CAM_TO_REC2020)
    enc = util.srgb_encode_lut()
    conv_out = ab.make_conversion(util.MATRIX_REC2020_TO_SRGB, lut_target=enc, coeffs_target=util.fit_unbounded_coeffs(enc))
    blob = np.load(os.path.join(util.GOLDEN_DIR, "filmic_data.npz"))["default_v8"]
    c = {}
    for name, method in (("demosaic", ab.DEMOSAIC_RCD), ("demosaic_ppg", ab.DEMOSAIC_PPG)):
        p, src, n = _mosaic(ab, ab.demosaic_data(method))
        c[name] = ("demosaic", p, src, n * 4, name == "demosaic_ppg")
    p, src, n = _mosaic(ab, ab.demosaic_data(ab.DEMOSAIC_RCD), 12, 12)
    c["demosaic_12x12"] = ("demosaic", p, src, n * 4, True)
    for op, data in (("colorin", ab.colorin_data(conv_in)), ("colorout", ab.colorout_data(conv_out)), ("denoiseprofile", ab.denoiseprofile_data()),
                     ("bilat", ab.bilat_data()), ("diffuse", ab.diffuse_data()), ("nlmeans", ab.nlmeans_data()), ("exposure", ab.exposure_data(0.0, 0.5)),
                     ("flip", ab.FlipData(5)), ("dither", ab.dither_data())):
        c[op] = (op, *_rgba(ab, data), False)
    p, src, n = _rgba(ab, None)
    c["filmicrgb"] = ("filmicrgb", _struct(p, ab.filmic_piece(blob, WORK, EXPORT)), src, n, False)
    p, src, n = _rgba(ab, None)
    c["channelmixerrgb"] = ("channelmixerrgb", _struct(p, ab.channelmixer_piece(WORK)), src, n, False)
    p, src, n = _rgba(ab, None)
    c["channelmixerrgb_unhandled_adaptation"] = ("channelmixerrgb", _struct(p, ab.channelmixer_piece(WORK, adaptation=99)), src, n, True)
    p, src, n = _rgba(ab, None)
    c["gamma"] = ("gamma", p, src, n // 4, True)
    d = ab.rawprepare_data((512,) * 4, (15000,) * 4, 2, 2)
    p = ab.make_piece(W, H, data=d, out_width=W - 2, out_height=H - 2)
    p.datatype = ab.TYPE_UINT16
    raw = np.random.default_rng(6).integers(0, 16384, (H, W), dtype=np.uint16)
    c["rawprepare"] = ("rawprepare", p, raw, (W - 2) * (H - 2) * 4, False)
    c["temperature"] = ("temperature", *_mosaic(ab, ab.temperature_data((2.13, 1.0, 1.57, 1.02))), False)
    p = ab.make_piece(W, H, filters=0, channels=3, data=ab.temperature_data((2.13, 1.0, 1.57, 1.02)))
    c["temperature_3_channels"] = ("temperature", p, util.rgba_test_image(W, H, 4)[..., :3].copy(), W * H * 12, False)
    c["highlights"] = ("highlights", *_mosaic(ab, ab.highlights_data(ab.HIGHLIGHTS_CLIP, 0.8)), False)
    for op in ("finalscale", "initialscale"):
        p = ab.make_piece(W, H, filters=0, channels=4, data=ab.finalscale_data(), out_width=W // 2, out_height=H // 2)
        p.roi_out.scale = 0.5
        c[op] = (op, p, util.rgba_test_image(W, H, 4), (W // 2) * (H // 2) * 16, False)
    return c


CASES = ("demosaic", "demosaic_ppg", "demosaic_12x12", "colorin", "colorout", "denoiseprofile", "filmicrgb", "bilat", "diffuse", "nlmeans",
         "rawprepare", "temperature", "temperature_3_channels", "highlights", "exposure", "gamma", "finalscale", "channelmixerrgb",
         "channelmixerrgb_unhandled_adaptation", "initialscale", "flip", "dither")


@pytest.fixture(scope="module")
def lib(built):
    import ansel_b200 as ab
    ab.init()
    return ab


def test_every_op_has_a_case(lib):
    assert {cases(lib)[name][0] for name in CASES} == set(lib.OPS)


def _dev(call, src, fill):
    """call(d_in, d_out, stream) on device copies of src and fill; -> (rc, output bytes)"""
    import torch
    d_in = torch.from_numpy(np.ascontiguousarray(src).view(np.uint8).reshape(-1).copy()).cuda()
    d_out = torch.from_numpy(fill.copy()).cuda()
    rc = call(d_in.data_ptr(), d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, d_out.cpu().numpy()


@pytest.mark.parametrize("name", CASES)
def test_host_equals_dev(lib, name):
    ab = lib
    L = ab.lib()
    op, piece, src, out_bytes, keeps_sentinel = cases(ab)[name]
    piece.devid = 0
    src = np.ascontiguousarray(src)
    fill = np.random.default_rng(7).integers(0, 256, out_bytes, dtype=np.uint8)
    rc_dev, want = _dev(lambda d_in, d_out, s: getattr(L, f"b200_{op}_process_dev")(C.byref(piece), d_in, d_out, s), src, fill)
    got = fill.copy()
    rc_host = getattr(L, f"b200_{op}_process_host")(C.byref(piece), src.ctypes.data, got.ctypes.data)
    assert rc_dev == 0 and rc_host == 0, L.b200_last_error()
    assert np.array_equal(got, want)
    if keeps_sentinel:
        assert (got == fill).any()


@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_export_convert_host_equals_dev(lib, fmt):
    ab = lib
    L = ab.lib()
    src = util.rgba_test_image(W, H, 4)
    fill = np.random.default_rng(7).integers(0, 256, W * H * (8 if fmt == ab.EXPORT_UINT16 else 4), dtype=np.uint8)
    rc_dev, want = _dev(lambda d_in, d_out, s: L.b200_export_convert_dev(d_in, d_out, W, H, fmt, s), src, fill)
    got = fill.copy()
    assert rc_dev == 0 and L.b200_export_convert_host(src.ctypes.data, got.ctypes.data, W, H, fmt) == 0
    assert np.array_equal(got, want)
