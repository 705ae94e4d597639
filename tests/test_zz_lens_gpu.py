"""GPU: lens correction through b200_lens_process_dev / _host and the dt_iop_lens__process / __process_cl adapters, bit for bit against the
oracle (itself pinned to the reference's lines, tests/test_cpu_lens.py) and the reference's committed outputs; a 45 MP frame; repeated
calls byte-identical; the refusals; lens as a node of a device-resident chain between demosaic and colorin."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

import util
import lens_util as lu
from lens_util import same_bits

pytestmark = pytest.mark.gpu


def _dev(img, lp, roi, **kw):
    import torch
    import ansel_b200 as ab
    d_in = torch.from_numpy(img).cuda()
    d_out = torch.from_numpy(lu.fill(roi)).cuda()
    p = lu.piece(roi, lp, **kw)
    rc = ab.lib().b200_lens_process_dev(C.byref(p), d_in.data_ptr(), d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, d_out.cpu().numpy()


def _host(img, lp, roi, **kw):
    import ansel_b200 as ab
    out = lu.fill(roi)
    p = lu.piece(roi, lp, **kw)
    rc = ab.lib().b200_lens_process_host(C.byref(p), img.ctypes.data, out.ctypes.data)
    return rc, out


@pytest.fixture(scope="module", autouse=True)
def _init(built):
    import ansel_b200 as ab
    ab.init()


@pytest.mark.parametrize("dist,tca,vig,inverse", list(itertools.product(lu.DIST, lu.TCA, (False, True), (0, 1))))
def test_both_entry_points_equal_oracle(dist, tca, vig, inverse):
    import ansel_b200 as ab
    for roi in lu.ROIS + ((0, 0, 640, 427, 0, 0, 640, 427, 1.0, 640, 427),):
        img = lu.frame(roi[2], roi[3], 3 * roi[2] + dist)
        for itor in lu.ITORS:
            for nan, mono, mask in lu.FLAGS:
                d = lu.lens_data(dist, tca, vig, inverse, nan, scale=1.02 if inverse else 1.0)
                rc, want = lu.oracle(img, d, itor, roi, mono, mask)
                lp = ab.lens_piece(d, itor)
                for fn in (_dev, _host):
                    rc_g, got = fn(img, lp, roi, monochrome=mono, mask=mask)
                    assert rc_g == rc, (fn.__name__, ab.lib().b200_last_error())
                    assert same_bits(got, want).all(), (fn.__name__, roi[8], itor, nan, mono, mask)


def test_golden_through_entry_points_and_adapters():
    import ansel_b200 as ab
    import ansel_b200.dtsurface as ds
    import torch
    M = ds.modlib()
    g = np.load(os.path.join(util.GOLDEN_DIR, "lens.npz"))
    for k in range(int(g["n"])):
        itor, mono, mask, r = (int(v) for v in g[f"args{k}"])
        d = ab.LensData.from_buffer_copy(g[f"data{k}"].tobytes())
        roi, img, want = lu.ROIS[r], g[f"in{k}"], g[f"out{k}"]
        for fn in (_dev, _host):
            rc, got = fn(img, ab.lens_piece(d, itor), roi, monochrome=mono, mask=mask)
            assert rc == 0 and same_bits(got, want).all(), (k, fn.__name__)
        # the adapters: the data block as the reference commits it, the interpolator from the preference
        C.c_int.in_dll(M, "b200_userpref_warp_interpolator").value = itor
        ix, iy, iw, ih, ox, oy, ow, oh, s, bw, bh = roi
        piece = ds.make_piece_iop("lens", iw, ih, d, channels_in=4, channels_out=4)
        piece.roi_in = ds.Roi(ix, iy, iw, ih, s)
        piece.roi_out = ds.Roi(ox, oy, ow, oh, s)
        piece.buf_in = ds.Roi(0, 0, bw, bh, 1.0)
        pipe = ds.make_pipe(devid=0)
        pipe.mask_display = mask
        pipe.dev.contents.image_storage.flags = ab.IMAGE_MONOCHROME if mono else 0
        out = lu.fill(roi)
        assert M.dt_iop_lens__process(piece.module, C.byref(pipe), C.byref(piece), np.ascontiguousarray(img).ctypes.data, out.ctypes.data) == 0
        assert same_bits(out, want).all(), (k, "process")
        d_in, d_out = torch.from_numpy(np.ascontiguousarray(img)).cuda(), torch.from_numpy(lu.fill(roi)).cuda()
        assert M.dt_iop_lens__process_cl(piece.module, C.byref(pipe), C.byref(piece), d_in.data_ptr(), d_out.data_ptr()) == 1
        torch.cuda.synchronize()
        assert same_bits(d_out.cpu().numpy(), want).all(), (k, "process_cl")
    C.c_int.in_dll(M, "b200_userpref_warp_interpolator").value = ab.INTERPOLATION_MITCHELL
    t = ab.Tiling()
    M.dt_iop_lens__tiling_callback(piece.module, C.byref(pipe), C.byref(piece), C.byref(t))
    assert (t.factor, t.factor_cl, t.maxbuf, t.maxbuf_cl, t.overhead, t.overlap, t.xalign, t.yalign) == (2.0, 2.0, 1.0, 1.0, 0, 4, 1, 1)


def test_45mp_and_repeated_calls():
    import torch
    import ansel_b200 as ab
    w, h = 8256, 5504
    roi = (0, 0, w, h, 0, 0, w, h, 1.0, w, h)
    img = lu.frame(w, h, 45)
    for inverse, tca in ((0, ab.LS_TCA_POLY3), (1, ab.LS_TCA_NONE)):
        d = lu.lens_data(ab.LS_DIST_PTLENS, tca, True, inverse)
        rc, want = lu.oracle(img, d, ab.INTERPOLATION_MITCHELL, roi)
        assert rc == 0
        lp = ab.lens_piece(d)
        p = lu.piece(roi, lp)
        d_in = torch.from_numpy(img).cuda()
        first = None
        for _ in range(10):
            d_out = torch.from_numpy(lu.fill(roi)).cuda()
            assert ab.lib().b200_lens_process_dev(C.byref(p), d_in.data_ptr(), d_out.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
            torch.cuda.synchronize()
            got = d_out.cpu().numpy()
            if first is None:
                first = got
                assert same_bits(got, want).all(), inverse
            else:
                assert np.array_equal(got.view(np.uint32), first.view(np.uint32))


def test_refusals_leave_the_output_untouched():
    import ansel_b200 as ab
    roi = lu.ROIS[0]
    img = lu.frame(roi[2], roi[3], 2)
    small = (0, 0, 2, 5, 0, 0, 2, 5, 1.0, 2, 5)
    copy = (0, 0, 61, 43, 0, 0, 50, 40, 1.0, 61, 43)
    cases = ((lu.lens_data(target_geom=ab.LENS_FISHEYE), roi, img), (lu.lens_data(target_geom=ab.LENS_FISHEYE_THOBY, inverse=1), roi, img),
             (lu.lens_data(), small, lu.frame(2, 5, 3)), (lu.lens_data(ab.LS_DIST_NONE, ab.LS_TCA_NONE, True), copy, img),
             (lu.lens_data(ls_have=0), copy, img))
    for d, r, src in cases:
        for fn in (_dev, _host):
            rc, out = fn(src, ab.lens_piece(d), r)
            assert rc == ab.B200_ERR_UNSUPPORTED, fn.__name__
            assert (out == lu.fill(r)).all()


def test_lens_between_demosaic_and_colorin_in_a_device_resident_chain():
    """demosaic -> lens -> colorin through b200_pixelpipe_process_on_gpu: lens's output in the chain equals the oracle on demosaic's
    device output, and the chain's output equals colorin on that (lanes 0-2: lens leaves lane 3 as the pipe's buffer holds it)"""
    import torch
    import ansel_b200 as ab
    import ansel_b200.dtsurface as ds
    M = ds.modlib()
    w, h = 1203, 811
    mosaic = util.frame_natural(w, h, 8)
    d_lens = lu.lens_data(ab.LS_DIST_PTLENS, ab.LS_TCA_POLY3, True, 0)
    datas = dict(demosaic=ab.demosaic_data(ab.DEMOSAIC_RCD), lens=d_lens, colorin=ab.colorin_data(ab.make_conversion(util.MATRIX_CAM_TO_REC2020)))
    pieces = {"demosaic": ds.make_piece_iop("demosaic", w, h, datas["demosaic"], channels_in=1, channels_out=4, filters=util.BAYER["RGGB"]),
              "lens": ds.make_piece_iop("lens", w, h, d_lens, channels_in=4, channels_out=4),
              "colorin": ds.make_piece_iop("colorin", w, h, datas["colorin"], channels_in=4, channels_out=4)}
    pipe = ds.make_pipe(devid=0)
    order = ("demosaic", "lens", "colorin")
    nodes = (ds.PipeNode * len(order))()
    for k, op in enumerate(order):
        nodes[k].process_cl = C.cast(getattr(M, f"dt_iop_{op}__process_cl"), C.c_void_p)
        nodes[k].module = pieces[op].module
        nodes[k].piece = C.pointer(pieces[op])
    bufs = M.b200_pipe_buffers_new()
    out = np.zeros((h, w, 4), np.float32)
    assert M.b200_pixelpipe_process_on_gpu(C.byref(pipe), nodes, len(order), bufs, mosaic.ctypes.data, out.ctypes.data) == 0
    M.b200_pipe_buffers_free(bufs)

    d_m = torch.from_numpy(mosaic).cuda()
    dem = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    assert M.dt_iop_demosaic__process_cl(pieces["demosaic"].module, C.byref(pipe), C.byref(pieces["demosaic"]), d_m.data_ptr(), dem.data_ptr()) == 1
    torch.cuda.synchronize()
    roi = (0, 0, w, h, 0, 0, w, h, 1.0, w, h)
    rc, lensed = lu.oracle(np.ascontiguousarray(dem.cpu().numpy()), d_lens, ab.INTERPOLATION_MITCHELL, roi)
    assert rc == 0
    d_l = torch.from_numpy(lensed).cuda()
    col = torch.zeros_like(d_l)
    assert M.dt_iop_colorin__process_cl(pieces["colorin"].module, C.byref(pipe), C.byref(pieces["colorin"]), d_l.data_ptr(), col.data_ptr()) == 1
    torch.cuda.synchronize()
    assert same_bits(out[..., :3], col.cpu().numpy()[..., :3]).all()
