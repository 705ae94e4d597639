"""GPU: frequency-domain chroma (FDC, method 1028) on X-Trans sensors through the C ABI and the module adapter, bit for bit against the
oracle's zero-per-tile mode (pinned to iop/demosaic/markesteijn.c compiled in place by tests/test_cpu_fdc.py) and the golden vectors."""
import ctypes as C
import os

import numpy as np
import pytest

import util
import fdc_util as fu
from fdc_util import same_bits
from vng_util import XTRANS

pytestmark = pytest.mark.gpu
FILL = -7.0


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    import ansel_b200 as ab
    ab.init()
    return ab


def piece_for(ab, m, x, y, iso, xover=fu.XOVER, smoothing=0, bare=False):
    h, w = m.shape
    dp = ab.DemosaicPiece()
    dp.data = ab.demosaic_data(ab.DEMOSAIC_FDC)
    dp.data.color_smoothing = smoothing
    dp.fdc_xover_iso = xover
    piece = ab.make_piece(w, h, filters=9, data=dp.data if bare else dp, devid=0, roi_x=x, roi_y=y, exif_iso=iso)
    for i in range(6):
        for j in range(6):
            piece.xtrans[i][j] = int(XTRANS[i][j])
    return piece


def run(ab, piece, m, host=False):
    import torch
    h, w = m.shape
    if host:
        out = np.full((h, w, 4), FILL, np.float32)
        ab.check(ab.lib().b200_demosaic_process_host(C.byref(piece), np.ascontiguousarray(m).ctypes.data, out.ctypes.data))
        return out
    d_in = torch.from_numpy(np.ascontiguousarray(m)).cuda()
    d_out = torch.full((h, w, 4), FILL, device="cuda")
    ab.check(ab.lib().b200_demosaic_process_dev(C.byref(piece), d_in.data_ptr(), d_out.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return d_out.cpu().numpy()


@pytest.mark.parametrize("iso", fu.ISOS)
@pytest.mark.parametrize("name", list(fu.CASES))
def test_fdc_bit_exact_through_both_entry_points(built, name, iso):
    m, x, y = fu.case(name)
    want = fu.oracle(m, x, y, iso, zero_per_tile=1)
    piece = piece_for(built, m, x, y, iso)
    got = run(built, piece, m)
    assert same_bits(got[..., :3], want[..., :3]).all() and (got[..., 3] == FILL).all()   # lane 3 is not a result: kept as found
    assert same_bits(run(built, piece, m, host=True), got).all()
    if name in ("one_tile", "narrow", "small") and iso in (100.0, 3200.0):
        g = np.load(os.path.join(util.GOLDEN_DIR, "fdc.npz"))
        assert same_bits(got[..., :3], g[f"{name}_{int(iso)}"]).all()


def test_fdc_colour_smoothing_and_the_crossover(built):
    m, x, y = fu.case("roi2")
    want = util.oracle_color_smoothing(fu.oracle(m, x, y, 800.0, zero_per_tile=1), 2)
    assert same_bits(run(built, piece_for(built, m, x, y, 800.0, smoothing=2), m)[..., :3], want[..., :3]).all()
    # the crossover is the caller's: ISO 800 is pure FDC above a crossover of 400
    assert same_bits(run(built, piece_for(built, m, x, y, 800.0, xover=400), m)[..., :3], fu.oracle(m, x, y, 800.0, 400)[..., :3]).all()


def test_fdc_refusals(built):
    ab = built
    m, x, y = fu.case("roi")
    with pytest.raises(ab.B200Error) as e:       # a bare data block cannot name the user's crossover
        run(ab, piece_for(ab, m, x, y, 100.0, bare=True), m)
    assert e.value.code == ab.B200_ERR_UNSUPPORTED and "not built" in str(e.value) and "fdc_xover_iso" in str(e.value)
    for (w, h) in ((14, 40), (40, 14)):         # the mirrored border reads out of frames this small in the reference
        s = np.ascontiguousarray(util.frame_natural(w, h, 3), np.float32)
        with pytest.raises(ab.B200Error) as e:
            run(ab, piece_for(ab, s, 0, 0, 100.0), s)
        assert e.value.code == ab.B200_ERR_UNSUPPORTED


def test_fdc_45mp_and_repeated_calls(built):
    ab = built
    w, h = util.SIZE_45MP
    m = np.ascontiguousarray(util.frame_natural(w, h, 9), np.float32)
    piece = piece_for(ab, m, 0, 0, 3200.0)
    first = run(ab, piece, m)
    assert np.isfinite(first[..., :3]).all()
    # a crop whose origin keeps the tile grid (a multiple of 96 and of 6) is the same computation away from the crop's border
    y0, x0, ch, cw = 96 * 7, 96 * 11, 96 * 6, 96 * 7
    crop = np.ascontiguousarray(m[y0:y0 + ch, x0:x0 + cw])
    got = run(ab, piece_for(ab, crop, 0, 0, 3200.0), crop)
    assert same_bits(got[..., :3], fu.oracle(crop, 0, 0, 3200.0)[..., :3]).all()
    inner = (slice(96, ch - 96), slice(96, cw - 96))
    assert same_bits(got[inner][..., :3], first[y0:y0 + ch, x0:x0 + cw][inner][..., :3]).all()
    small, sx, sy = fu.case("multi")
    sp = piece_for(ab, small, sx, sy, 100.0)
    ref = run(ab, sp, small)
    for _ in range(10):
        assert run(ab, sp, small).tobytes() == ref.tobytes()


def test_fdc_module_adapter(built):
    """dt_iop_demosaic__process_cl carries the crossover preference (b200_userpref_fdc_xover_iso) next to a copy of the data block"""
    import torch
    import ansel_b200.dtsurface as ds
    ab = built
    M = ds.modlib()
    m, x, y = fu.case("one_tile")
    h, w = m.shape
    data = ab.demosaic_data(ab.DEMOSAIC_FDC)
    pref = C.c_int.in_dll(M, "b200_userpref_fdc_xover_iso")
    assert pref.value == 1600
    for iso in (1600.0, 3200.0):
        piece = ds.make_piece_iop("demosaic", w, h, data, channels_in=1, channels_out=4, filters=9)
        for k in range(36):
            piece.dsc_in.xtrans[k] = int(XTRANS.ravel()[k])
        pipe = ds.make_pipe(devid=0, stream=torch.cuda.current_stream().cuda_stream, exif_iso=iso)
        d_in = torch.from_numpy(np.ascontiguousarray(m)).cuda()
        d_out = torch.full((h, w, 4), FILL, device="cuda")
        assert M.dt_iop_demosaic__process_cl(piece.module, C.byref(pipe), C.byref(piece), d_in.data_ptr(), d_out.data_ptr()) == 1
        torch.cuda.synchronize()
        assert same_bits(d_out.cpu().numpy()[..., :3], fu.oracle(m, 0, 0, iso)[..., :3]).all(), iso
