"""CPU tests of the C entry points: every field the tiling callbacks write (the modules that declare no tiling callback of their own
answer with default_tiling_callback, develop/tiling.c:1423-1463; non-local means leaves the OpenCL fields as it found them,
nlmeans.c:400-414), and the host entries of dither and blending refusing to run without a device."""
import ctypes as C

import numpy as np
import pytest

SENTINEL_F, SENTINEL_U = -7.25, 0xDEADBEEF
FIELDS = ("factor", "factor_cl", "maxbuf", "maxbuf_cl", "overhead", "overlap", "xalign", "yalign")

# op -> (overlap: 4 with IOP_FLAGS_TILING_FULL_ROI, placed before demosaic)
DEFAULT_TILING = dict(rawprepare=(4, True), temperature=(0, True), exposure=(0, False), gamma=(0, False), colorin=(0, False),
                      colorout=(0, False), channelmixerrgb=(0, False), dither=(0, False), finalscale=(4, False), initialscale=(4, False))

# (roi_in width, height, roi_out width, height, filters)
PIECES = [(6000, 4000, 6000, 4000, 0x94949494), (6000, 4000, 5990, 3990, 0x94949494), (4000, 3000, 1234, 567, 0x94949494),
          (6000, 4000, 6000, 4000, 9), (6001, 4003, 3000, 2001, 9), (6000, 4000, 6000, 4000, 0), (641, 479, 320, 240, 0)]


def sentinel_tiling(ab):
    t = ab.Tiling()
    t.factor = t.factor_cl = t.maxbuf = t.maxbuf_cl = SENTINEL_F
    t.overhead = t.overlap = t.xalign = t.yalign = SENTINEL_U
    return t


def fields(t):
    return {f: getattr(t, f) for f in FIELDS}


@pytest.mark.parametrize("op", sorted(DEFAULT_TILING))
def test_default_tiling_callback_fields(built, op):
    import ansel_b200 as ab
    L = ab.lib()
    overlap, raw = DEFAULT_TILING[op]
    f32 = np.float32
    for iw, ih, ow, oh, filters in PIECES:
        piece = ab.make_piece(iw, ih, filters=filters, channels=1 if filters else 4, out_width=ow, out_height=oh)
        t = sentinel_tiling(ab)
        getattr(L, f"b200_{op}_tiling")(piece, t)
        factor = f32(1.0) + (f32(ow) * f32(oh)) / (f32(iw) * f32(ih))  # float arithmetic in the order of the C
        align = (3 if filters == 9 else 2) if raw and filters else 1
        want = dict(factor=factor, factor_cl=factor, maxbuf=1.0, maxbuf_cl=1.0, overhead=0, overlap=overlap, xalign=align, yalign=align)
        assert fields(t) == want, (op, iw, ih, ow, oh, hex(filters))


def test_nlmeans_tiling_leaves_the_opencl_fields(built):
    import ansel_b200 as ab
    L = ab.lib()
    for radius, scale, overlap in ((2.0, 1.0, 2 + 7), (3.0, 0.5, 2 + 4), (5.0, 4.0, 10 + 14)):
        piece = ab.make_piece(6000, 4000, filters=0, channels=4, data=ab.nlmeans_data(radius=radius), scale=scale)
        t = sentinel_tiling(ab)
        L.b200_nlmeans_tiling(piece, t)
        want = dict(factor=4.0, factor_cl=SENTINEL_F, maxbuf=1.0, maxbuf_cl=SENTINEL_F, overhead=0, overlap=overlap, xalign=1, yalign=1)
        assert fields(t) == want, (radius, scale)


def test_dither_and_blend_host_entries_fail_loudly_without_a_device(built):
    """refusal with the output (and blending's mask) untouched: nothing computed on the CPU"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import ansel_b200 as ab
    import blend_util as bu
    L = ab.lib()
    rgba, out = np.zeros((64, 64, 4), np.float32), np.full((64, 64, 4), -3.0, np.float32)
    assert L.b200_dither_process_host(ab.make_piece(64, 64, filters=0, channels=4, data=ab.dither_data()), rgba.ctypes.data, out.ctypes.data) != 0
    assert (out == -3.0).all()
    form, mask = np.ones((64, 64), np.float32), np.full((64, 64), -3.0, np.float32)
    pc = ab.make_piece(64, 64, filters=0, channels=4)
    assert L.b200_blend_process_host(C.byref(pc), C.byref(bu.params()), C.c_void_p(rgba.ctypes.data), C.c_void_p(out.ctypes.data),
                                     C.c_void_p(form.ctypes.data), C.c_void_p(mask.ctypes.data)) != 0
    assert (out == -3.0).all() and (mask == -3.0).all()
