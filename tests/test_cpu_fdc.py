"""CPU: frequency-domain chroma (FDC) for X-Trans sensors.  The oracle is pinned bit for bit to iop/demosaic/markesteijn.c
xtrans_fdc_interpolate compiled in place (oracle/fdc.mk): in its carried mode against the reference on one thread, in its zero-per-tile
mode (what the kernel computes) on frames of one tile.  The kernel's stages, compiled with g++ and run thread by thread in either order,
equal the zero-per-tile oracle.  The coefficient tables of the kernel are the reference's, bit for bit.  The kernel's SASS adds no FFMA and
no local memory to what the stages it shares with Markesteijn's one-pass kernel have."""
import os
import re
import subprocess

import numpy as np
import pytest

import util
import fdc_util as fu
from fdc_util import same_bits

need_ref = pytest.mark.skipif(not os.path.isdir("/root/reference/src") and fu.ref_lib() is None, reason="oracle/_ref/libref_fdc_*.so not built")


@pytest.fixture(scope="module", autouse=True)
def _build():
    subprocess.run(["make", "-s", "-C", util.ORACLE_DIR, "oracle"], check=True)


@need_ref
@pytest.mark.parametrize("iso", fu.ISOS)
@pytest.mark.parametrize("name", list(fu.CASES))
def test_oracle_carried_equals_reference_on_one_thread(name, iso):
    m, x, y = fu.case(name)
    for fill in (0x00, 0x55):
        got, want = fu.oracle(m, x, y, iso, zero_per_tile=0, fill=fill), fu.ref(m, x, y, iso, fill=fill)
        assert same_bits(got, want).all(), fill
        assert (got[..., 3] == -7.0).all()          # lane 3 is not written


@need_ref
@pytest.mark.parametrize("iso", (100.0, 3200.0))
def test_oracle_zero_per_tile_equals_reference_on_one_tile(iso):
    for seed, (w, h, x, y) in enumerate(((96, 90, 0, 0), (96, 96, 3, 1), (91, 77, 5, 2), (60, 40, 1, 5))):
        m = np.ascontiguousarray(util.frame_natural(w, h, seed + 11), np.float32)
        m[7, 9], m[20, 30], m[31, 12] = np.inf, -np.inf, np.nan
        assert same_bits(fu.oracle(m, x, y, iso, zero_per_tile=1), fu.ref(m, x, y, iso, fill=0)).all(), (w, h, x, y)


@need_ref
def test_oracle_on_infinite_but_not_nan_frames():
    """isolated ±inf and near-overflow values: the complex products run into NaN + iNaN and libgcc's __mulsc3 recovers infinities"""
    m = np.ascontiguousarray(util.frame_natural(200, 150, 3), np.float32)
    m[60, 70], m[90, 33], m[40, 120], m[41, 121] = np.inf, -np.inf, 1e38, 3e38
    for iso in (100.0, 3200.0):
        assert same_bits(fu.oracle(m, 1, 2, iso, zero_per_tile=0), fu.ref(m, 1, 2, iso)).all()


@need_ref
def test_distances_between_modes_threads_and_builds_are_printed():
    """not asserted: how many pixels the stale scratch bytes reach (fill patterns, zero per tile, thread counts) and how far the release
    build is from the strict one"""
    for name in ("multi", "roi2"):
        m, x, y = fu.case(name)
        base = fu.ref(m, x, y, 100.0, fill=0)
        print(f"{name}: fill 0x55 vs 0xaa {fu.differing(fu.ref(m, x, y, 100.0, fill=0x55), fu.ref(m, x, y, 100.0, fill=0xaa))} px, "
              f"zero per tile vs carried {fu.differing(fu.oracle(m, x, y, 100.0, zero_per_tile=1), base)} px, "
              f"8 threads vs 1 {fu.differing(fu.ref(m, x, y, 100.0, nthreads=8), base)} px, "
              f"release vs strict {fu.differing(fu.ref(m, x, y, 100.0, kind='fast'), base)} px of {m.size}")


@need_ref
def test_kernel_tables_are_the_references():
    import importlib.util
    spec = importlib.util.spec_from_file_location("gen_fdc_tables", os.path.join(util.ROOT, "tools", "gen_fdc_tables.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    text = open(os.path.join(util.ROOT, "ansel_b200", "csrc", "fdc_tables.h")).read()
    lits = re.findall(r"-?0x[0-9a-f.]+p[+-]\d+f", text)
    want = [gen.lit(float(v)) for t in fu.ref_tables() for v in t]
    assert lits == want


def test_oracle_equals_golden():
    g = np.load(os.path.join(util.GOLDEN_DIR, "fdc.npz"))
    for name in ("one_tile", "narrow", "small"):
        m, x, y = fu.case(name)
        for iso in (100.0, 3200.0):
            assert same_bits(fu.oracle(m, x, y, iso, zero_per_tile=1)[..., :3], g[f"{name}_{int(iso)}"]).all(), (name, iso)


@pytest.mark.parametrize("iso", (100.0, 3200.0))
@pytest.mark.parametrize("ascending", [0, 1])
@pytest.mark.parametrize("name", list(fu.CASES))
def test_kernel_stages_equal_oracle(name, ascending, iso):
    m, x, y = fu.case(name)
    assert same_bits(fu.emul(m, x, y, iso, nthreads=96, ascending=ascending), fu.oracle(m, x, y, iso, zero_per_tile=1)).all()


def test_kernel_stages_on_random_geometries():
    rng = np.random.default_rng(28)
    for trial in range(4):
        w, h, x, y = int(rng.integers(15, 330)), int(rng.integers(15, 260)), int(rng.integers(0, 6)), int(rng.integers(0, 6))
        m = np.ascontiguousarray(util.frame_natural(w, h, int(rng.integers(50))), np.float32)
        iso = float(rng.choice(fu.ISOS))
        got = fu.emul(m, x, y, iso, nthreads=int(rng.choice([37, 1024])), ascending=int(rng.integers(2)))
        assert same_bits(got, fu.oracle(m, x, y, iso, zero_per_tile=1)).all(), (trial, w, h, x, y, iso)


def test_fdc_kernel_sass_adds_no_ffma_and_no_local_memory_to_markesteijns():
    """the FDC instance has no FFMA outside the IEEE division sequences Markesteijn's one-pass instance has as well; its stack frame is the one the shared stage of red and blue at the
    solitary greens (mk_solitary, which indexes its candidates at run time) has in Markesteijn's one-pass instance as well"""
    import test_cpu_filmic_sass as fs
    so = os.path.join(util.ROOT, "ansel_b200", "libb200iop.so")
    if not os.path.exists(so):
        pytest.skip("libb200iop.so is not built")
    r = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True)
    funcs = fs.functions(r.stdout)
    fdc = [v for k, v in funcs.items() if "fdc_tiles_kernel" in k]
    mk1 = [v for k, v in funcs.items() if "markesteijn_tiles_kernelILi1E" in k]
    assert len(fdc) == 1 and len(mk1) == 1
    # the classifier knows the reciprocal, square-root and literal-division sequences; the division by 3 of the 2x2 green blocks (mk_div, the
    # IEEE div.rn.ftz.f32 of a register by 3) is the one more sequence, and Markesteijn's kernel has it too: compared with registers erased
    shape = lambda stray: {re.sub(r"R\d+", "R", x.split(": ", 1)[1]) for x in stray}
    stray, _ = fs.stray_ffma(fdc[0])
    assert shape(stray) <= shape(fs.stray_ffma(mk1[0])[0]), sorted(shape(stray) - shape(fs.stray_ffma(mk1[0])[0]))[:4]
    def frame(insns):  # the stack frame the prologue carves out of R1
        return [int(ops[2], 16) & 0xFFFFFFFF for _, op, ops in insns[:8] if op.startswith(("VIADD", "IADD3")) and ops[:2] == ["R1", "R1"]]
    assert frame(fdc[0]) == frame(mk1[0])
