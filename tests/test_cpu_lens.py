"""CPU: lens correction (src/iop/lens.c process() over LensSerious's evaluators).  The oracle equals the reference's lines compiled in place
(strict build) bit for bit over distortion model x TCA model x vignetting x direction x interpolator x ROI shift and zoom x the nan checks,
monochrome and mask-display flags, on frames with NaN, +-inf, negative and subnormal pixels; the library's host plan equals the reference's
ls_eval_t field for field; the kernels, compiled with g++ and run thread by thread, equal the oracle; the data block's layout is the
reference's; the kernels' SASS has no local memory and no FFMA outside the IEEE division and square-root sequences."""
import ctypes as C
import itertools
import os
import re
import subprocess

import numpy as np
import pytest

import util
import lens_util as lu
import ansel_b200 as ab
from lens_util import same_bits

SO = os.path.join(util.ROOT, "ansel_b200", "libb200iop.so")


@pytest.fixture(scope="module", autouse=True)
def _build(built):
    subprocess.run(["make", "-s", "-C", util.ORACLE_DIR, "oracle"], check=True)


need_ref = pytest.mark.skipif(not os.path.isdir("/root/reference/src") and lu.ref_lib("strict") is None,
                              reason="oracle/_ref not built (no /root/reference)")

MATRIX = list(itertools.product(lu.DIST, lu.TCA, (False, True), (0, 1)))


def _configs(dist, tca, vig, inverse):
    for roi in lu.ROIS:
        for itor in lu.ITORS:
            for nan, mono, mask in lu.FLAGS:
                yield roi, itor, nan, mono, mask, lu.lens_data(dist, tca, vig, inverse, nan, scale=1.02 if inverse else 1.0)


@need_ref
@pytest.mark.parametrize("dist,tca,vig,inverse", MATRIX)
def test_oracle_and_emulated_kernels_equal_the_strict_reference(dist, tca, vig, inverse):
    fast_diff = total = 0
    for roi, itor, nan, mono, mask, d in _configs(dist, tca, vig, inverse):
        img = lu.frame(roi[2], roi[3], 11 * roi[2] + dist)
        rc, got = lu.oracle(img, d, itor, roi, mono, mask)
        rc_e, emu = lu.emul(img, d, itor, roi, mono, mask)
        assert rc_e == rc
        if rc == ab.B200_ERR_UNSUPPORTED:
            # no geometry to resample, between ROIs of different sizes: the reference copies and vignettes past its output buffer
            assert not (roi[2] == roi[6] and roi[3] == roi[7]) and (got == lu.fill(roi)).all() and (emu == lu.fill(roi)).all()
            continue
        assert rc == 0
        _, want = lu.ref(img, d, itor, roi, mono, mask)
        where = (roi[8], itor, nan, mono, mask)
        assert same_bits(got, want).all(), where
        assert same_bits(emu, got).all(), where
        _, fast = lu.ref(img, d, itor, roi, mono, mask, kind="fast")
        fast_diff += int((~same_bits(fast, want)).sum())
        total += want.size
    print(f"release build differs from the strict one on {fast_diff} of {total} floats")


@pytest.mark.parametrize("w,h", [(61, 43), (150, 104), (6000, 4000), (1, 1)])
@pytest.mark.parametrize("mono", [0, 1])
def test_plan_equals_the_reference_field_for_field(w, h, mono):
    cases = [lu.lens_data(dist, tca, vig, inv, scale=s, focal=f, real_focal=rf)
             for dist, tca, vig, inv in MATRIX for s, f, rf in ((1.0, 28.0, False), (0.97, 18.0, True), (1.02, 70.0, True))]
    cases.append(lu.lens_data(target_geom=ab.LENS_FISHEYE))       # a projection change: resolved, then refused by the kernel entry
    cases.append(lu.lens_data(target_geom=ab.LENS_PANORAMIC))     # not radially expressible: the plan drops the geometry
    cases.append(lu.lens_data(crop=0.0))
    for d in cases:
        p = lu.plans(d, w, h, mono)
        if "ref" not in p:
            pytest.skip("oracle/_ref not built")
        for name in ("lib", "oracle", "emul"):
            assert p[name] == p["ref"], name


@need_ref
def test_data_block_layout_matches_the_reference():
    r = lu.ref_lib("strict")
    r.ref_lens_sizeof.restype = C.c_size_t
    assert r.ref_lens_sizeof(0) == C.sizeof(ab.LensData) == 45144
    assert r.ref_lens_sizeof(1) == C.sizeof(ab.LsLens)
    assert r.ref_lens_sizeof(2) == ab.LensData.ls_lens.offset and r.ref_lens_sizeof(3) == ab.LensData.ls_have.offset
    assert (r.ref_lens_sizeof(4), r.ref_lens_sizeof(5), r.ref_lens_sizeof(6)) == (ab.LsLens.n_tca.offset, ab.LsLens.n_vig.offset,
                                                                                 ab.LsLens.n_real_focal.offset)
    assert r.ref_lens_sizeof(7) == C.sizeof(ab.LensEval) == 632


def test_oracle_and_emulation_equal_golden():
    g = np.load(os.path.join(util.GOLDEN_DIR, "lens.npz"))
    for k in range(int(g["n"])):
        itor, mono, mask, r = (int(v) for v in g[f"args{k}"])
        d = ab.LensData.from_buffer_copy(g[f"data{k}"].tobytes())
        roi = lu.ROIS[r]
        for fn in (lu.oracle, lu.emul):
            rc, got = fn(g[f"in{k}"], d, itor, roi, mono, mask)
            assert rc == 0 and same_bits(got, g[f"out{k}"]).all(), (k, fn.__name__)


def test_refusals_leave_the_output_untouched():
    roi = lu.ROIS[0]
    img = lu.frame(roi[2], roi[3], 1)
    for d in (lu.lens_data(target_geom=ab.LENS_FISHEYE), lu.lens_data(target_geom=ab.LENS_FISHEYE_EQUISOLID, inverse=1)):
        for fn in (lu.oracle, lu.emul):
            rc, out = fn(img, d, ab.INTERPOLATION_MITCHELL, roi)
            assert rc == ab.B200_ERR_UNSUPPORTED and (out == lu.fill(roi)).all()
    small = (0, 0, 2, 5, 0, 0, 2, 5, 1.0, 2, 5)
    rc, out = lu.emul(lu.frame(2, 5, 1), lu.lens_data(), ab.INTERPOLATION_BILINEAR, small)
    assert rc == ab.B200_ERR_UNSUPPORTED and (out == lu.fill(small)).all()


def test_kernels_sass_has_no_local_memory_and_no_contracted_product(built):
    from test_cpu_nlm_sass import functions
    from test_cpu_filmic_sass import stray_ffma
    r = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-300:]
    kernels = {n: i for n, i in functions(r.stdout).items() if re.search(r"lens_(vignette_)?kernel", n)}
    assert len(kernels) == 4
    for name, insns in kernels.items():
        local = [f"{a:#x}: {op}" for a, op, _ in insns if op.split(".")[0] in ("LDL", "STL")]
        assert not local, f"{name}: local-memory traffic {local[:4]}"
        stray, _ = stray_ffma(insns)
        assert not stray, f"{name}: {len(stray)} FFMA outside the IEEE division, reciprocal and square-root sequences, e.g. {stray[:4]}"
