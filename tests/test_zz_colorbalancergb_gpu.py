"""GPU: colour balance rgb through b200_colorbalancergb_process_dev / _host and the dt_iop_colorbalancergb__process / __process_cl adapters,
bit for bit against the oracle (itself pinned to the reference's lines, tests/test_cpu_colorbalancergb.py): the whole parameter matrix with
the data blocks and LUTs the reference's commit_params() makes (tests/golden/colorbalancergb_blocks.npz) on three work profiles, and the
reference's committed outputs; a 45 MP frame in each saturation formula; repeated calls byte-identical; the mask-display refusal; colour
balance rgb behind a scene-referred RGB blend node in the default raw edit's device-resident chain, from demosaic to filmic."""
import ctypes as C
import os

import numpy as np
import pytest

import util
import colorbalancergb_util as cu
import ansel_b200 as ab
from colorbalancergb_util import same_bits

pytestmark = pytest.mark.gpu


def _piece(w, h, cp):
    p = ab.make_piece(w, h, filters=0, channels=4, devid=0)
    p.data, p.data_size = C.addressof(cp), C.sizeof(cp)
    p._keepalive = cp
    return p


def _dev(img, cp, fill=-7.0):
    import torch
    h, w = img.shape[:2]
    d_in = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    d_out = torch.full((h, w, 4), fill, dtype=torch.float32, device="cuda")
    rc = ab.lib().b200_colorbalancergb_process_dev(C.byref(_piece(w, h, cp)), d_in.data_ptr(), d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, d_out.cpu().numpy()


def _host(img, cp, fill=-7.0):
    h, w = img.shape[:2]
    out = np.full(img.shape, fill, np.float32)
    rc = ab.lib().b200_colorbalancergb_process_host(C.byref(_piece(w, h, cp)), np.ascontiguousarray(img).ctypes.data, out.ctypes.data)
    return rc, out


@pytest.fixture(scope="module", autouse=True)
def _init(built):
    ab.init()


def _golden():
    g = np.load(os.path.join(util.GOLDEN_DIR, "colorbalancergb.npz"))
    for k in range(int(g["n"])):
        yield g[f"data{k}"], (g[f"work_in{k}"], g[f"work_out{k}"]), g[f"lut{k}"], g[f"in{k}"], g[f"out{k}"]


def test_parameter_matrix_through_both_entries_equals_oracle():
    """every block of the CPU matrix (presets, full-range and sub-range random blocks, both formulas) on three work profiles"""
    g = np.load(os.path.join(util.GOLDEN_DIR, "colorbalancergb_blocks.npz"))
    img = cu.frame(97, 61, 5)
    n = 0
    for j in range(len(g["profiles"])):
        work = (g["work_in"][j], g["work_out"][j])
        for k in range(len(g["names"])):
            data = ab.ColorbalancergbData.from_buffer_copy(g["data"][k].tobytes())
            cp = ab.colorbalancergb_piece(data, work, g["luts"][cu.FORMULAS.index(data.saturation_formula), j])
            rc, want = cu.oracle(img, cp)
            assert rc == 0
            for fn in (_dev, _host):
                rc_g, got = fn(img, cp)
                assert rc_g == 0, ab.lib().b200_last_error()
                assert same_bits(got, want).all(), (fn.__name__, str(g["profiles"][j]), str(g["names"][k]), int((~same_bits(got, want)).sum()))
            n += 1
    assert n == 3 * 165


def test_golden_through_entry_points_and_adapters():
    import torch
    import ansel_b200.dtsurface as ds
    M = ds.modlib()
    for k, (data, work, lut, img, want) in enumerate(_golden()):
        cp = ab.colorbalancergb_piece(data, work, lut)
        for fn in (_dev, _host):
            rc, got = fn(img, cp)
            assert rc == 0 and same_bits(got, want).all(), (k, fn.__name__)
        h, w = img.shape[:2]
        d = cu.adapter_data(cp.data, lut)
        piece = ds.make_piece_iop("colorbalancergb", w, h, d, channels_in=4, channels_out=4)
        piece.data_size = C.sizeof(ab.ColorbalancergbData)
        wp = ds.profile_info(*work)
        pipe = ds.make_pipe(devid=0, work_profile=wp)
        out = np.full(img.shape, -7.0, np.float32)
        assert M.dt_iop_colorbalancergb__process(piece.module, C.byref(pipe), C.byref(piece), np.ascontiguousarray(img).ctypes.data, out.ctypes.data) == 0
        assert same_bits(out, want).all(), (k, "process")
        d_in = torch.from_numpy(np.ascontiguousarray(img)).cuda()
        d_out = torch.full((h, w, 4), -7.0, dtype=torch.float32, device="cuda")
        assert M.dt_iop_colorbalancergb__process_cl(piece.module, C.byref(pipe), C.byref(piece), d_in.data_ptr(), d_out.data_ptr()) == 1
        torch.cuda.synchronize()
        assert same_bits(d_out.cpu().numpy(), want).all(), (k, "process_cl")
    t = ab.Tiling()
    M.dt_iop_colorbalancergb__tiling_callback(piece.module, C.byref(pipe), C.byref(piece), C.byref(t))
    assert (t.factor, t.overlap, t.xalign, t.yalign) == (2.0, 0, 1, 1)


@pytest.mark.parametrize("k", [0, 1])
def test_45mp_and_repeated_calls(k):
    """the golden file's first two blocks (dt UCS: the scene-referred default; JzAzBz: the legacy preset) on a 45 MP frame; the oracle on
    every 61st row (the module is pointwise); ten calls byte-identical"""
    import torch
    data, work, lut, _, _ = list(_golden())[k]
    cp = ab.colorbalancergb_piece(data, work, lut)
    w, h = 8256, 5504
    img = cu.frame(w, h, 45 + k)
    rows = np.arange(0, h, 61)
    rc, want = cu.oracle(np.ascontiguousarray(img[rows]), cp)
    assert rc == 0
    p = _piece(w, h, cp)
    d_in = torch.from_numpy(img).cuda()
    first = None
    for _ in range(10):
        d_out = torch.full((h, w, 4), -7.0, dtype=torch.float32, device="cuda")
        assert ab.lib().b200_colorbalancergb_process_dev(C.byref(p), d_in.data_ptr(), d_out.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0
        torch.cuda.synchronize()
        got = d_out.cpu().numpy()
        if first is None:
            first = got
            assert same_bits(got[rows], want).all()
        else:
            assert np.array_equal(got.view(np.uint32), first.view(np.uint32))


def test_mask_display_is_refused_with_the_output_untouched():
    data = ab.ColorbalancergbData()
    data.mask_display = 1
    cp = ab.colorbalancergb_piece(data, cu.PROFILES["rec2020"], np.ones(360, np.float32))
    img = cu.frame(16, 8, 1)
    for fn in (_dev, _host):
        rc, out = fn(img, cp)
        assert rc == ab.B200_ERR_UNSUPPORTED and (out == -7.0).all(), fn.__name__


def test_default_raw_edit_chain_with_a_blend_node_stays_on_the_device():
    """demosaic -> colorin -> exposure -> channelmixerrgb -> colorbalancergb (the scene-referred default, blended in scene-referred RGB through
    a parametric mask at 80 %) -> filmicrgb through b200_pixelpipe_process_on_gpu equals the same modules called one by one through their
    host entries, with the blend through b200_blend_process_host"""
    import blend_util as bu
    import ansel_b200.dtsurface as ds
    M, L = ds.modlib(), ab.lib()
    L.b200_blend_process_host.argtypes = [C.c_void_p, C.POINTER(bu.BlendParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    w, h = 1203, 811
    mosaic = util.frame_natural(w, h, 8)
    work = cu.PROFILES["rec2020"]
    export = util.profile_pair(util.SRGB_TO_XYZ_D50)
    data, gwork, lut, _, _ = list(_golden())[0]          # the scene-referred default on linear Rec2020
    assert (gwork[0] == work[0]).all()
    d_cb = cu.adapter_data(ab.colorbalancergb_piece(data, work, lut).data, lut)
    conv_in = ab.make_conversion(util.MATRIX_CAM_TO_REC2020)
    blob = np.ascontiguousarray(np.load(os.path.join(util.GOLDEN_DIR, "filmic_data.npz"))["default_v8"], np.uint8)
    datas = dict(demosaic=ab.demosaic_data(ab.DEMOSAIC_RCD), colorin=ab.colorin_data(conv_in),
                 exposure=ab.exposure_data(black=0.002, exposure_ev=0.7), channelmixerrgb=ab.channelmixer_piece(work), colorbalancergb=d_cb,
                 filmicrgb=(C.c_uint8 * blob.size).from_buffer_copy(blob.tobytes()))
    pieces = {op: ds.make_piece_iop(op, w, h, d, channels_in=1 if op == "demosaic" else 4, channels_out=4,
                                    filters=util.BAYER["RGGB"] if op == "demosaic" else 0) for op, d in datas.items()}
    pieces["colorbalancergb"].data_size = C.sizeof(ab.ColorbalancergbData)
    pipe = ds.make_pipe(devid=0, work_profile=ds.profile_info(*work), output_profile=ds.profile_info(*export))
    blend = bu.params(opacity=80.0, mask_mode=bu.MASK_ENABLED | bu.MASK_PARAMETRIC, channels={0: (0.02, 0.1, 0.8, 1.5)})
    order = tuple(datas)
    nodes = (ds.PipeNode * len(order))()
    for k, op in enumerate(order):
        nodes[k].process_cl = C.cast(getattr(M, f"dt_iop_{op}__process_cl"), C.c_void_p)
        nodes[k].module = pieces[op].module
        nodes[k].piece = C.pointer(pieces[op])
    nodes[order.index("colorbalancergb")].blend = C.cast(C.pointer(blend), C.c_void_p)
    bufs = M.b200_pipe_buffers_new()
    out = np.zeros((h, w, 4), np.float32)
    assert M.b200_pixelpipe_process_on_gpu(C.byref(pipe), nodes, len(order), bufs, mosaic.ctypes.data, out.ctypes.data) == 0
    M.b200_pipe_buffers_free(bufs)

    x = mosaic
    for op in order:
        y = np.zeros((h, w, 4), np.float32)
        assert getattr(M, f"dt_iop_{op}__process")(pieces[op].module, C.byref(pipe), C.byref(pieces[op]), np.ascontiguousarray(x).ctypes.data,
                                                   y.ctypes.data) == 0, op
        if op == "colorbalancergb":
            graded = y.copy()
            mask = np.zeros((h, w), np.float32)
            assert L.b200_blend_process_host(C.byref(ab.make_piece(w, h, channels=4, devid=0)), C.byref(blend), np.ascontiguousarray(x).ctypes.data,
                                             y.ctypes.data, None, mask.ctypes.data) == 0
            # the module and the mask both change the frame: the node is neither a copy of its input nor the module alone
            assert (~same_bits(graded[..., :3], x[..., :3])).any() and (~same_bits(y[..., :3], graded[..., :3])).any()
        x = y
    assert same_bits(out[..., :3], x[..., :3]).all()
