"""CPU: colour balance rgb (src/iop/colorbalancergb.c process()).  The oracle and the kernel compiled with g++ (run thread by thread) equal
the reference's lines compiled in place (strict build) bit for bit over the five presets, 120 random parameter blocks over the full ranges
and 40 over sub-ranges that keep the frame alive x three matrix work profiles (both saturation formulas), on frames with natural pixels, greys, NaN, +-inf, negatives, subnormals and values above 1; the
gamut LUTs come from the reference's own commit_params(), serially, from a defined fill.  Also: hand-made LUTs through the hue wrap, the data
block's layout, the golden file, the mask-display refusal, the adapter's no-op without a work profile, and the kernel's SASS."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import util
import colorbalancergb_util as cu
import ansel_b200 as ab
from colorbalancergb_util import same_bits

SO = os.path.join(util.ROOT, "ansel_b200", "libb200iop.so")


@pytest.fixture(scope="module", autouse=True)
def _build(built):
    subprocess.run(["make", "-s", "-C", util.ORACLE_DIR, "oracle"], check=True)


need_ref = pytest.mark.skipif(not os.path.isdir("/root/reference/src") and cu.ref_lib("strict") is None,
                              reason="oracle/_ref not built (no /root/reference)")


def _luts():
    if "cbrgb_luts" not in util._cache:
        p = cu.defaults()
        luts = {}
        for f in cu.FORMULAS:
            p.saturation_formula = f
            for prof in cu.PROFILES:
                luts[(f, prof)] = cu.commit(p, prof)[1]
        util._cache["cbrgb_luts"] = luts
    return util._cache["cbrgb_luts"]


def _check(img, cp, where):
    rc, want = cu.ref(img, cp)
    assert rc == 0
    rc_o, got = cu.oracle(img, cp)
    rc_e, emu = cu.emul(img, cp)
    assert rc_o == 0 and rc_e == 0
    assert same_bits(got, want).all(), (where, int((~same_bits(got, want)).sum()))
    assert same_bits(emu, want).all(), (where, int((~same_bits(emu, want)).sum()))
    _, fast = cu.ref(img, cp, kind="fast")
    return want, fast


@need_ref
@pytest.mark.parametrize("profile", list(cu.PROFILES))
def test_oracle_and_emulated_kernel_equal_the_strict_reference(profile):
    img = cu.frame(48, 32, 7)
    luts = _luts()
    diff = total = worst = 0
    alive = {"random": [], "moderate": []}
    for name, p in cu.blocks():
        data, _ = cu.commit(p, None)
        cp = cu.piece(data, profile, luts[(p.saturation_formula, profile)])
        want, fast = _check(img, cp, (profile, name))
        kind = name.split()[0]
        if kind in alive:
            alive[kind].append(float((want[..., :3] != 0).any(axis=2).mean()))
        bad = ~same_bits(fast, want)
        diff += int(bad.sum())
        total += want.size
        both = bad & np.isfinite(fast) & np.isfinite(want)
        if both.any():
            worst = max(worst, int(util.ulp_distance(fast[both], want[both]).max()))
    print(f"{profile}: the release (x86-64-v2) build differs from the strict one on {diff} of {total} floats, by up to {worst} ULP")
    full = np.array(alive["random"])
    print(f"{profile}: full-range blocks with an all-black output: {int((full == 0).sum())} of {full.size}, under 5 % non-black: "
          f"{int((full < 0.05).sum())}; mean non-black share {full.mean():.2f}")
    # the sub-range blocks keep most of the frame alive, so that their parity is not that of a black frame
    assert min(alive["moderate"]) > 0.3


@need_ref
@pytest.mark.parametrize("formula", cu.FORMULAS)
def test_hand_made_luts_through_the_hue_wrap(formula):
    """LUTs edited at single entries, 0 and 359 among them, on a frame of saturated colours at every hue: each edit must change the output
    (so the frame reads those entries: lookup_gamut's interpolation between 359 and the wrap to 0, :560-566), and the output must still
    equal the reference's.  For a finite hue x_test stays in [0, 359], so the xi < 0 / xi > 359 branches are reached only through a NaN hue;
    there the result is NaN whichever entry is read (the float-to-int conversion of a NaN gives 0 on the GPU and INT_MIN on x86)."""
    img = cu.hue_frame(96, 64, 11)
    p = cu.presets()[0 if formula == ab.COLORBALANCE_SATURATION_JZAZBZ else -1][1]
    data, _ = cu.commit(p, None)
    base = _luts()[(formula, "rec2020")]
    want0, _ = _check(img, cu.piece(data, "rec2020", base), formula)
    rng = np.random.default_rng(formula)
    edits = [("entry 0", 0), ("entry 359", 359), ("entry 180", 180)]
    for what, idx in edits:
        lut = base.copy()
        lut[idx] *= np.float32(0.5)
        want, _ = _check(img, cu.piece(data, "rec2020", lut), (formula, what))
        assert (~same_bits(want, want0)).any(), (formula, what)
    for lut in (base * rng.uniform(0.5, 1.5, 360).astype(np.float32), np.roll(base, 180)):
        want, _ = _check(img, cu.piece(data, "rec2020", lut.astype(np.float32)), formula)
        assert (~same_bits(want, want0)).any(), formula


@need_ref
def test_lut_march_leaves_no_entry_unwritten_on_these_profiles():
    """the dt UCS branch of commit_params() writes only the entries its 18 000-step march hits (:1295-1347) into an allocation init_pipe
    does not zero; serially, from two fills, every entry is written on the three work profiles here; the JzAzBz branch writes all 360"""
    for f in cu.FORMULAS:
        p = cu.defaults()
        p.saturation_formula = f
        for prof in cu.PROFILES:
            _, a = cu.commit(p, prof, lut_fill=-1.0)
            _, b = cu.commit(p, prof, lut_fill=-2.0)
            unwritten = int((a == -1.0).sum())
            print(f"formula {f}, {prof}: {unwritten} of 360 entries unwritten")
            assert unwritten == int((b == -2.0).sum()) == 0
            assert (a == b).all() and (a > 0).all()


@need_ref
def test_data_block_layout_matches_the_reference():
    r = cu.ref_lib("strict")
    D = ab.ColorbalancergbData
    assert r.ref_colorbalancergb_layout(0) == C.sizeof(D) == 232
    names = ("midtones_Y", "chroma", "saturation", "brilliance", "hue_angle", "white_fulcrum", "checker_color_1", "saturation_formula",
             "checker_size", "mask_display", "lut_inited")
    for k, n in enumerate(names, 1):
        assert r.ref_colorbalancergb_layout(k) == getattr(D, n).offset, n
    assert r.ref_colorbalancergb_layout(12) == C.sizeof(cu.Params)


@need_ref
def test_committed_data_blocks_are_the_references():
    """tests/golden/colorbalancergb_blocks.npz, which the device tests run, holds what the reference's commit_params() makes"""
    g = np.load(os.path.join(util.GOLDEN_DIR, "colorbalancergb_blocks.npz"))
    blocks = cu.blocks()
    assert list(g["names"]) == [n for n, _ in blocks]
    for k, (_, p) in enumerate(blocks):
        assert bytes(cu.commit(p, None)[0]) == g["data"][k].tobytes(), k
    assert (g["luts"] == np.stack([np.stack([_luts()[(f, prof)] for prof in cu.PROFILES]) for f in cu.FORMULAS])).all()


def test_oracle_and_emulation_equal_golden():
    g = np.load(os.path.join(util.GOLDEN_DIR, "colorbalancergb.npz"))
    for k in range(int(g["n"])):
        cp = ab.colorbalancergb_piece(g[f"data{k}"], (g[f"work_in{k}"], g[f"work_out{k}"]), g[f"lut{k}"])
        for fn in (cu.oracle, cu.emul):
            rc, got = fn(g[f"in{k}"], cp)
            assert rc == 0 and same_bits(got, g[f"out{k}"]).all(), (k, fn.__name__)


def test_mask_display_is_refused_with_the_output_untouched():
    data = ab.ColorbalancergbData()
    data.mask_display = 1
    cp = ab.colorbalancergb_piece(data, cu.PROFILES["rec2020"], np.ones(360, np.float32))
    img = cu.frame(8, 4, 1)
    for fn in (cu.oracle, cu.emul):
        rc, out = fn(img, cp)
        assert rc == ab.B200_ERR_UNSUPPORTED and (out == -7.0).all()


def test_adapter_without_work_profile_returns_0_and_writes_nothing(built):
    """process() :592 returns 0 when the pipe has no work profile; the adapter does the same without touching the output or the device"""
    import ansel_b200.dtsurface as ds
    M = ds.modlib()
    lut = np.ones(360, np.float32)
    d = cu.adapter_data(ab.ColorbalancergbData(), lut)
    piece = ds.make_piece_iop("colorbalancergb", 8, 4, d, channels_in=4, channels_out=4)
    piece.data_size = C.sizeof(ab.ColorbalancergbData)
    pipe = ds.make_pipe(devid=0)
    img = cu.frame(8, 4, 1)
    out = np.full_like(img, -7.0)
    assert M.dt_iop_colorbalancergb__process(piece.module, C.byref(pipe), C.byref(piece), img.ctypes.data, out.ctypes.data) == 0
    assert (out == -7.0).all()
    assert M.dt_iop_colorbalancergb__process_cl(piece.module, C.byref(pipe), C.byref(piece), img.ctypes.data, out.ctypes.data) != 0
    assert (out == -7.0).all()


def test_kernel_sass_is_small_has_no_local_memory_and_no_contracted_product(built):
    from test_cpu_nlm_sass import functions
    from test_cpu_filmic_sass import stray_ffma
    r = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-300:]
    kernels = {n: i for n, i in functions(r.stdout).items() if re.search(r"colorbalancergb_kernel", n)}
    assert len(kernels) == 2
    for name, insns in kernels.items():
        local = [f"{a:#x}: {op}" for a, op, _ in insns if op.split(".")[0] in ("LDL", "STL")]
        assert not local, f"{name}: local-memory traffic {local[:4]}"
        stray, _ = stray_ffma(insns)
        assert not stray, f"{name}: {len(stray)} FFMA outside the IEEE division, reciprocal and square-root sequences, e.g. {stray[:4]}"
        # per instance, a little above the first clean build with powf out of line: 2928 (JzAzBz) and 2688 (dt UCS) instructions
        cap = 3000 if "kernelILi0E" in name else 2750
        assert len(insns) <= cap, f"{name}: {len(insns)} instructions, ceiling {cap}"
