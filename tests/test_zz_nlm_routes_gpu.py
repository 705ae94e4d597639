"""GPU parity of every non-local-means kernel route, bit for bit against the oracle, each case stating the kernel and template
instance it means to run.  Two independent witnesses of the route: the prediction of the product's own host-side planning
(util.nlm_route: grp_plan, grp_pipe_fits, chunk_of, pipe2_takes; the switches B200_NLM_* as the launcher reads them), and the
kernels torch.profiler records on the device.

The 45 MP bench frame runs once through the C3 chain (RCD -> denoiseprofile NLM -> colorin -> filmic) against the oracle chain: the
interior 64-row chunks of that frame are what the half-height slots of nlm_pipe_kernel<1, *, *, *, 0> exist for."""
import ctypes as C
import re

import numpy as np
import pytest

import util

pytestmark = pytest.mark.gpu

NORM = (0.7, 1.3, 0.9, 1.0)
SWITCHES = ("B200_NLM_CHUNKS", "B200_NLM_WINDOW", "B200_NLM_NO_PIPE", "B200_NLM_WHOLE_SLOTS", "B200_NLM_IEEE_DIV", "B200_NLM_G")


def same_bits(a, b):
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _targs(args):
    return tuple(1 if v == "true" else 0 if v == "false" else int(v) for v in re.split(r"\s*,\s*", args.strip()))


def launched_nlm_kernels(run):
    """run() under torch.profiler: the distinct NLM kernels it launched, as (kernel, template arguments) -- nlm_pipe_kernel <R, N1, PR, DC, CFG>,
    nlm_group_kernel <R, WP, N1, PR, DC, KP>, the chunk kernels without -- and what run() returned"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for attempt in range(2):  # a profiling session now and then receives no kernel record at all from CUPTI: then record once more
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = run()
            torch.cuda.synchronize()
        if any("nlm_" in e.name for e in prof.events()):
            break
    seen = set()
    for e in prof.events():
        m = re.search(r"nlm_(chunks_win|chunks|pipe|group)_kernel(?:<([^<>]*)>)?", e.name)
        if m:
            seen.add(({"chunks_win": "window"}.get(m.group(1), m.group(1)), _targs(m.group(2)) if m.group(2) else ()))
            continue
        m = re.search(r"nlm_(chunks_win|chunks|pipe|group)_kernel(?:I((?:L[ib]\d+E)+)E)?", e.name)  # a name the profiler left mangled
        if m:
            seen.add(({"chunks_win": "window"}.get(m.group(1), m.group(1)), tuple(int(v) for v in re.findall(r"L[ib](\d+)E", m.group(2) or ""))))
    return sorted(seen), out


def expected_kernel(route):
    k = route["kernel"]
    if k == "pipe":
        return (k, tuple(route[x] for x in ("R", "N1", "PR", "DC", "CFG")))
    if k == "group":
        return (k, tuple(route[x] for x in ("R", "WP", "N1", "PR", "DC", "KP")))
    return (k, ())


def cuda_nlm(img, **kw):
    import torch
    import ansel_b200 as ab
    ab.init()
    p = dict(scattering=0.0, scale=1.0, luma=1.0, chroma=1.0, center_weight=0.1, sharpness=0.005, P=1, K=7, decimate=0, norm=(1.0, 1.0, 1.0, 1.0))
    p.update(kw)
    h, w = img.shape[:2]
    d_in = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    d_out = torch.zeros_like(d_in)

    def run():
        ab.check(ab.lib().b200_nlmeans_denoise_dev(d_in.data_ptr(), d_out.data_ptr(), w, h, p["scattering"], p["scale"], p["luma"], p["chroma"],
                                                   p["center_weight"], p["sharpness"], p["P"], p["K"], p["decimate"], (C.c_float * 4)(*p["norm"]),
                                                   torch.cuda.current_stream().cuda_stream))
    seen, _ = launched_nlm_kernels(run)
    return seen, d_out.cpu().numpy()


def check_case(monkeypatch, size, kw, env, want, img=None):
    """the route the case means to take (want: kernel, template arguments, chunks on the half-height slots), the route the product's
    planning predicts, the kernel the device ran, and the output against the oracle"""
    for s in SWITCHES:
        monkeypatch.delenv(s, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    w, h = size
    route = util.nlm_route(w, h, **kw)
    for k, v in want.items():
        assert route[k] == v, f"planned route {route}, the case wants {k} = {v}"
    if img is None:
        img = (util.rgba_scene(w, h, 3, noise=0.02) * 60).astype(np.float32)
    seen, got = cuda_nlm(img, **kw)
    assert seen == [expected_kernel(route)], f"launched {seen}, planned {expected_kernel(route)}"
    bad = ~same_bits(got, util.oracle_nlmeans(img, **kw))
    assert not bad.any(), f"{route}: {int(bad.sum())} floats differ, first {np.argwhere(bad)[:4].tolist()}"
    return route


def pipe1(n1, pr, dc, halves, cfg=0):
    return dict(kernel="pipe", R=1, N1=n1, PR=pr, DC=dc, CFG=cfg, halves=halves)


IEEE = {"B200_NLM_IEEE_DIV": "1"}
# 360 x 256 and 220 x 192: chunks of 64 rows (72 / 64 px wide); 8 and 2 of them in the frame's interior at these search radii
# (patch radius + largest shift from the frame's edge).  1000 x 700: 108 of 154.  Every other chunk of these frames is on the rim: the
# whole-pair slots of the same kernel instance.
HALF_SLOT_CASES = {
    "N1-PR-DC": ((360, 256), dict(), {}, pipe1(1, 1, 1, 8)),
    "N0-PR-DC": ((220, 192), dict(norm=NORM, K=3), {}, pipe1(0, 1, 1, 2)),
    "N1-PR-ieee_switch": ((360, 256), dict(K=2), IEEE, pipe1(1, 1, 0, 8)),
    "N0-PR-ieee_switch": ((220, 192), dict(norm=NORM, K=3, luma=0.5), IEEE, pipe1(0, 1, 0, 2)),
    "N1-PR-ieee_range": ((360, 256), dict(K=3, center_weight=3e6, sharpness=0.05), {}, pipe1(1, 1, 0, 8)),  # 1 + cw beyond 2^20
    "N0-PR-ieee_range": ((220, 192), dict(K=2, norm=NORM, center_weight=0.2, sharpness=3e6), {}, pipe1(0, 1, 0, 2)),  # sharpness beyond 2^20
    "N1-P0": ((360, 256), dict(K=3, center_weight=-1.0, sharpness=0.01), {}, pipe1(1, 0, 0, 8)),
    "N0-P0": ((220, 192), dict(K=2, center_weight=-1.0, sharpness=0.01, norm=NORM, luma=0.8, chroma=0.6), {}, pipe1(0, 0, 0, 2)),
    "K1": ((360, 256), dict(K=1), {}, pipe1(1, 1, 1, 8)),
    "K1-P0-N0": ((360, 256), dict(K=1, center_weight=-1.0, sharpness=0.02, norm=NORM), {}, pipe1(0, 0, 0, 8)),
    "K1-decimated": ((360, 256), dict(K=1, decimate=1), {}, pipe1(1, 1, 1, 8)),  # 5 patches: 3 pairs = the six half slots
    "K1-decimated-P0": ((220, 192), dict(K=1, decimate=1, center_weight=-1.0, sharpness=0.01), {}, pipe1(1, 0, 0, 2)),
    "K0": ((360, 256), dict(K=0), {}, pipe1(1, 1, 1, 0)),  # one patch: no pair to split, every chunk on the whole-pair slots
    "K0-P0": ((360, 256), dict(K=0, center_weight=-1.0, sharpness=0.01), {}, pipe1(1, 0, 0, 0)),
    "K7-blend": ((1000, 700), dict(luma=0.8, chroma=0.6), {}, pipe1(1, 1, 1, 108)),
    "K7-P0-N0-blend": ((360, 256), dict(center_weight=-1.0, sharpness=0.01, norm=NORM, luma=0.5, chroma=0.7), {}, pipe1(0, 0, 0, 8)),
}
WHOLE_SLOT_CASES = {
    "64x64": ((64, 64), dict(K=3), {}, pipe1(1, 1, 1, 0)),  # one chunk, the frame's rim on every side
    "rows51-N0-P0": ((300, 150), dict(K=3, center_weight=-1.0, sharpness=0.01, norm=NORM), {}, pipe1(0, 0, 0, 0)),
    "rows60-ieee": ((200, 600), dict(K=3), IEEE, pipe1(1, 1, 0, 0)),
    "rows61-N0-DC": ((150, 61), dict(K=2, norm=NORM), {}, pipe1(0, 1, 1, 0)),
    "R2-N1-PR": ((360, 256), dict(P=2, K=3), {}, dict(kernel="pipe", R=2, N1=1, PR=1, DC=1, CFG=0, halves=0)),
    "R2-N0-P0": ((220, 192), dict(P=2, K=5, norm=NORM, center_weight=-1.0, sharpness=0.01), {}, dict(kernel="pipe", R=2, N1=0, PR=0, CFG=0)),
    "R2-N0-PR": ((300, 150), dict(P=2, K=2, norm=NORM, luma=0.6), {}, dict(kernel="pipe", R=2, N1=0, PR=1, DC=1, CFG=0)),
    "R2-N1-P0": ((360, 256), dict(P=2, K=4, center_weight=-1.0, sharpness=0.01), {}, dict(kernel="pipe", R=2, N1=1, PR=0, CFG=0)),
    "cfg1-R1": ((360, 256), dict(), {"B200_NLM_WHOLE_SLOTS": "1"}, pipe1(1, 1, 1, 0, cfg=1)),
    "cfg1-R2": ((360, 256), dict(P=2, K=3), {"B200_NLM_WHOLE_SLOTS": "1"}, dict(kernel="pipe", R=2, CFG=1, halves=0)),
}
# 400 px: chunks 72 wide.  130 / 203 rows: chunks of 65 / 68 rows, 7 pixel pairs per thread; scattering 0.5 at K=4: a window of 97-128 columns
NOPIPE = {"B200_NLM_NO_PIPE": "1"}
GROUP_CASES = {
    "R1-WP96-KP6": ((400, 256), dict(), NOPIPE, dict(kernel="group", R=1, WP=96, KP=6, N1=1, PR=1, DC=1)),
    "R1-WP96-KP7": ((400, 130), dict(center_weight=-1.0, sharpness=0.01), {}, dict(kernel="group", R=1, WP=96, KP=7, N1=1, PR=0)),
    "R1-WP128-KP6": ((400, 256), dict(K=4, scattering=0.5, norm=NORM), {}, dict(kernel="group", R=1, WP=128, KP=6, N1=0, PR=1, DC=1)),
    "R1-WP128-KP7": ((400, 203), dict(K=4, scattering=0.5), IEEE, dict(kernel="group", R=1, WP=128, KP=7, N1=1, PR=1, DC=0)),
    "R2-WP96-KP6": ((400, 256), dict(P=2, K=5, norm=NORM, center_weight=-1.0, sharpness=0.01), NOPIPE,
                    dict(kernel="group", R=2, WP=96, KP=6, N1=0, PR=0)),
    "R2-WP96-KP7": ((400, 130), dict(P=2, K=5, norm=NORM), IEEE, dict(kernel="group", R=2, WP=96, KP=7, N1=0, PR=1, DC=0)),
    "R2-WP128-KP6": ((400, 256), dict(P=2, K=4, scattering=0.5), {}, dict(kernel="group", R=2, WP=128, KP=6, N1=1, PR=1, DC=1)),
    "R2-WP128-KP7": ((400, 203), dict(P=2, K=4, scattering=0.5, center_weight=-1.0, sharpness=0.01, luma=0.8), {},
                     dict(kernel="group", R=2, WP=128, KP=7, N1=1, PR=0)),
    "R1-WP96-KP7-N0-DC": ((400, 203), dict(K=3, norm=NORM), {}, dict(kernel="group", R=1, WP=96, KP=7, N1=0, PR=1, DC=1)),
    "G2": ((400, 203), dict(K=3), {"B200_NLM_G": "2"}, dict(kernel="group", G=2)),  # 49 patches: the last group is short
    "G4": ((400, 203), dict(K=3, center_weight=-1.0, sharpness=0.01), {"B200_NLM_G": "4"}, dict(kernel="group", G=4)),
    "G6": ((400, 203), dict(K=3, norm=NORM), {"B200_NLM_G": "6"}, dict(kernel="group", G=6)),
}
CHUNK_CASES = {
    "P0": ((300, 203), dict(P=0, K=3), {}, dict(kernel="chunks")),
    "P3": ((300, 203), dict(P=3, K=2), {}, dict(kernel="chunks")),
    "P4": ((300, 203), dict(P=4, K=2), {}, dict(kernel="chunks")),
    "K7-scattered": ((300, 203), dict(K=7, scattering=1.0), {}, dict(kernel="chunks")),  # shifts of 85 px: no window fits
    "chunks_switch": ((360, 256), dict(), {"B200_NLM_CHUNKS": "1"}, dict(kernel="chunks")),
    "window_switch": ((360, 256), dict(), {"B200_NLM_WINDOW": "1"}, dict(kernel="window")),
}


@pytest.mark.parametrize("case", list(HALF_SLOT_CASES))
def test_pipe_kernel_half_slots(built, monkeypatch, case):
    check_case(monkeypatch, *HALF_SLOT_CASES[case])


@pytest.mark.parametrize("case", list(WHOLE_SLOT_CASES))
def test_pipe_kernel_whole_pair_slots(built, monkeypatch, case):
    check_case(monkeypatch, *WHOLE_SLOT_CASES[case])


@pytest.mark.parametrize("case", list(GROUP_CASES))
def test_group_kernel(built, monkeypatch, case):
    check_case(monkeypatch, *GROUP_CASES[case])


@pytest.mark.parametrize("case", list(CHUNK_CASES))
def test_chunk_kernels(built, monkeypatch, case):
    check_case(monkeypatch, *CHUNK_CASES[case])


def test_group_variants_and_pipe_flags_all_covered():
    """the tables above reach all eight group instances (R, WP, KP), each (N1, PR, DC) on the group kernel and, with half-height slots,
    on nlm_pipe_kernel<1, *, *, *, 0>"""
    group = {(w["R"], w["WP"], w["KP"]) for _, _, _, w in GROUP_CASES.values() if "WP" in w}
    assert group == {(r, wp, kp) for r in (1, 2) for wp in (96, 128) for kp in (6, 7)}
    flags = {(1, 0, 0), (0, 0, 0), (1, 1, 1), (0, 1, 1), (1, 1, 0), (0, 1, 0)}
    assert {(w["N1"], w["PR"], w.get("DC", 0)) for _, _, _, w in GROUP_CASES.values() if "N1" in w} == flags
    assert {(w["N1"], w["PR"], w["DC"]) for _, _, _, w in HALF_SLOT_CASES.values() if w["halves"] > 0} == flags


def extreme_frame(w, h):
    """the frame of test_nlm_gpu.test_extreme_pixels_through_the_group_kernel, its specials moved into the interior chunks of a 64-row grid"""
    img = (util.rgba_scene(w, h, 4, noise=0.02) * 60).astype(np.float32)
    img[70:110, 80:140, :3] = 0.0
    img[130:150, 150:190, :3] = 1e-30
    img[100, 100, :3] = (np.inf, 1.0, 2.0)
    img[101, 120, :3] = (np.nan, 1.0, 2.0)
    img[110, 200, :3] = (3e38, -3e38, 1e19)
    img[150, 90, :3] = (-np.inf, 0.5, -1.0)
    img[160, 240, :3] = (1e-40, 1e-44, 0.0)
    img[5, 5, :3] = (1e-40, 1e-44, 0.0)
    return img


EXTREME_CASES = {
    "default": (dict(), pipe1(1, 1, 1, 8)),
    "K3": (dict(K=3), pipe1(1, 1, 1, 8)),
    "P0": (dict(K=3, center_weight=-1.0, sharpness=0.01), pipe1(1, 0, 0, 8)),
    "N0-K3": (dict(K=3, norm=(0.5, 2.0, 1.5, 1.0)), pipe1(0, 1, 1, 8)),
    "R2-N0": (dict(K=2, P=2, norm=(0.5, 2.0, 1.5, 1.0)), dict(kernel="pipe", R=2, N1=0, PR=1, DC=1, CFG=0)),
}


@pytest.mark.parametrize("case", list(EXTREME_CASES))
def test_extreme_pixels_through_the_pipe_kernel(built, monkeypatch, case):
    """zeros, 1e-30, +-inf, NaN, +-3e38 and subnormals inside the half-height-slot chunks of 360 x 256: the min_nan clamp in front of
    Markstein's division, the weights of exactly 1 and 0, NaN through the packed lanes"""
    kw, want = EXTREME_CASES[case]
    check_case(monkeypatch, (360, 256), kw, {}, want, img=extreme_frame(360, 256))


@pytest.mark.parametrize("scale,pipe_type", [(1.0, 1), (0.5, 3)])
def test_nlmeans_module_through_the_half_slots(built, monkeypatch, scale, pipe_type):
    """b200_nlmeans_process_dev: center_weight -1, luma / chroma != 1, its own norm, and the decimated patch list of a preview pipe -- the
    production caller of nlm_pipe_kernel<1, false, false, false, 0> on the half-height slots"""
    import torch
    import ansel_b200 as ab
    for s in SWITCHES:
        monkeypatch.delenv(s, raising=False)
    ab.init()
    w, h = 1000, 700
    img = util.lab_scene(w, h, 3)
    d = ab.nlmeans_data(radius=1.0, strength=50.0, luma=0.5, chroma=0.7)
    # the module's arguments to the core, labglue.cu b200_nlmeans_process_dev
    P, K = int(np.ceil(np.float32(1.0) * np.float32(scale))), int(np.ceil(np.float32(7 * scale)))
    decimate = 1 if pipe_type in (ab.PIPE_PREVIEW, ab.PIPE_THUMBNAIL) else 0
    nL, nC = np.float32(1) / np.float32(120), np.float32(1) / np.float32(512)
    route = util.nlm_route(w, h, scale=scale, luma=0.5, chroma=0.7, center_weight=-1.0, sharpness=float(np.float32(3000) / np.float32(51)), P=P, K=K,
                           decimate=decimate, norm=(float(nL * nL), float(nC * nC), float(nC * nC), 1.0))
    assert (route["kernel"], route["N1"], route["PR"], route["DC"], route["halves"]) == ("pipe", 0, 0, 0, 108)
    piece = ab.make_piece(w, h, filters=0, channels=4, data=d, devid=0, scale=scale, pipe_type=pipe_type)
    d_in = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    d_out = torch.zeros_like(d_in)
    seen, _ = launched_nlm_kernels(lambda: ab.check(ab.lib().b200_nlmeans_process_dev(C.byref(piece), d_in.data_ptr(), d_out.data_ptr(),
                                                                                        torch.cuda.current_stream().cuda_stream)))
    assert seen == [expected_kernel(route)]
    bad = ~same_bits(d_out.cpu().numpy(), util.oracle_nlmeans_iop(img, d, scale, decimate))
    assert not bad.any(), f"{int(bad.sum())} floats differ, first {np.argwhere(bad)[:4].tolist()}"


def test_c3_chain_45mp_bench_frame_bit_exact(built, monkeypatch):
    """C3 on bench.py's own frame (frame_natural(8256, 5504, SEEDS[0])): RCD -> denoiseprofile (NLM, P=1, K=7) -> colorin -> filmic rgb
    against the oracle chain, fed the CUDA demosaic (RCD itself checked on its defined pixels).  9492 of the 86 x 115 chunks of 64 x 72
    px (all but the first and last chunk row and column, the last column being the 48-px remainder) take the half-height slots."""
    import test_chains_gpu as chains
    for s in SWITCHES:
        monkeypatch.delenv(s, raising=False)
    w, h = util.SIZE_45MP
    route = util.nlm_route(w, h, center_weight=0.1, sharpness=float(np.float32(0.045) / np.float32(9)))  # denoiseprofile's arguments at scale 1
    assert (route["kernel"], route["R"], route["N1"], route["PR"], route["DC"], route["CFG"]) == ("pipe", 1, 1, 1, 1, 0)
    assert (route["halves"], route["chunks"]) == (84 * 113, 86 * 115)
    seen, (dev, g, o, _k) = launched_nlm_kernels(lambda: chains._front(w, h, util.SEEDS[0], K=7))
    assert seen == [expected_kernel(route)]
    g, o = chains._filmic(dev, g, o)
    bad = ~same_bits(g.cpu().numpy(), o)
    assert not bad.any(), f"{int(bad.sum())} floats differ, first {np.argwhere(bad)[:4].tolist()}"
