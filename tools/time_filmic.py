"""Time filmic_agx_kernel on the bench frame, one library build against another, by CUDA events around
b200_filmicrgb_process_dev (the v8 defaults with the export profile, as bench.py's C3 step runs it).

The bench frame goes once through RCD -> denoiseprofile (NLM, P = 1, K = 7) -> colorin with the tree's library; each variant
library then tones that same buffer.  Before any timing, every variant's output must be byte-identical to the first one's.
The variants are timed in alternating rounds in one process (median of --calls calls per round, after --warmup calls), and the
card's name, power limit and clocks are printed beside the result.

    python tools/time_filmic.py build NAME SRC      # here: SRC/ansel_b200/csrc/filmic.cu (+ its headers), or a git revision,
                                                    # linked with the tree's other objects into tools/filmic_variants/NAME.so
    python tools/time_filmic.py time [NAME=LIB.so ...] [--rounds 3] [--calls 15] [--warmup 3]
                                                    # on the GPU; no NAME=LIB: the tree's libb200iop.so alone
"""
import argparse
import ctypes as C
import glob
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [os.path.join(ROOT, "tests"), ROOT]
VARIANTS = os.path.join(HERE, "filmic_variants")


def build(name, src):
    """compile filmic.cu of a source tree (a directory holding ansel_b200/csrc and include, or a git revision) with the library's
    flags and link it with the tree's other objects"""
    from ansel_b200 import build as B
    B.build()
    os.makedirs(VARIANTS, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        if not os.path.isdir(src):
            arch = subprocess.run(["git", "-C", ROOT, "archive", src, "ansel_b200/csrc", "include"], capture_output=True, check=True).stdout
            subprocess.run(["tar", "-x", "-C", tmp], input=arch, check=True)
            src = tmp
        obj = os.path.join(tmp, "filmic.o")
        cmd = [B._nvcc()] + [f for f in B.NVCC_FLAGS if f != "-shared"] + ["-I", os.path.join(src, "include"), "-Xptxas=-v", "-c",
                                                                         os.path.join(src, "ansel_b200", "csrc", "filmic.cu"), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True, check=True)
        print(name, *[ln.strip() for ln in r.stderr.splitlines() if "stack frame" in ln or "registers" in ln], sep="\n  ")
        objs = [o for o in sorted(glob.glob(os.path.join(B.HERE, "build", "*.o"))) if os.path.basename(o) != "filmic.o"]
        so = os.path.join(VARIANTS, name + ".so")
        subprocess.run([B._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-cudart", "static", "-Xcompiler", "-fPIC",
                        "-o", so, obj] + objs, check=True)
    print("built", so)


def card(torch):
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[torch.cuda.current_device()] if r.returncode == 0 else torch.cuda.get_device_name()


def time_variants(a):
    import numpy as np
    import torch
    import util
    import ansel_b200 as ab
    assert torch.cuda.is_available(), "needs a GPU"
    variants = [v.split("=", 1) for v in a.variants] or [["tree", ab.LIB_PATH]]
    ab.init()
    L = ab.lib()
    w, h = util.SIZE_45MP
    stream = torch.cuda.current_stream().cuda_stream
    work, export = util.profile_pair(util.REC2020_TO_XYZ_D50), util.profile_pair(util.SRGB_TO_XYZ_D50)
    fblob = np.load(os.path.join(util.GOLDEN_DIR, "filmic_data.npz"))["default_v8"]
    conv_in = ab.make_conversion(util.MATRIX_CAM_TO_REC2020, identity=0x1001)
    datas = [ab.demosaic_data(ab.DEMOSAIC_RCD), ab.denoiseprofile_data(ab.DENOISE_NLMEANS, radius=1, nbhood=7), ab.colorin_data(conv_in)]
    fp = ab.filmic_piece(fblob, work, export)

    def piece_of(data, ch):
        p = ab.make_piece(w, h, filters=util.BAYER["RGGB"] if ch == 1 else 0, channels=ch, devid=0)
        p.data, p.data_size = C.addressof(data), C.sizeof(data)
        return p

    # the bench's C3 frame up to filmic's input
    cur = torch.from_numpy(util.frame_natural(w, h, 20260922)).cuda()
    for op, data, ch in zip(("demosaic", "denoiseprofile", "colorin"), datas, (1, 4, 4)):
        nxt = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
        ab.check(getattr(L, f"b200_{op}_process_dev")(piece_of(data, ch), cur.data_ptr(), nxt.data_ptr(), stream))
        cur = nxt
    fpiece = piece_of(fp, 4)
    out = torch.empty_like(cur)

    calls = []
    for name, path in variants:
        V = C.CDLL(os.path.abspath(path))
        V.b200_filmicrgb_process_dev.argtypes = [C.POINTER(ab.Piece), C.c_void_p, C.c_void_p, C.c_void_p]
        assert V.b200_init(0) == 0, name
        calls.append((name, lambda V=V: ab.check(V.b200_filmicrgb_process_dev(fpiece, cur.data_ptr(), out.data_ptr(), stream))))

    want = None
    for name, call in calls:
        out.zero_()
        call()
        torch.cuda.synchronize()
        got = out.cpu().numpy().view(np.uint32)
        if want is None:
            want = got
        assert np.array_equal(got, want), f"{name}: {int((got != want).sum())} floats differ from {calls[0][0]}"

    med = {name: [] for name, _ in calls}
    for _ in range(a.rounds):
        for name, call in calls:
            for _ in range(a.warmup):
                call()
            torch.cuda.synchronize()
            ts = []
            for _ in range(a.calls):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                call()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            med[name].append(float(np.median(ts)))
    print(f"card: {card(torch)}")
    print(f"{w}x{h} ({w * h / 1e6:.1f} MP), filmic v8 defaults + export profile; outputs of all variants byte-identical")
    print(f"median of {a.calls} calls per round after {a.warmup} warm-up calls, {a.rounds} alternating rounds")
    for name, ms in med.items():
        print(f"  {name:16s} " + "  ".join(f"{m:6.3f}" for m in ms) + f"   ms  (median of rounds {float(np.median(ms)):.3f})")


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    b = sub.add_parser("build")
    b.add_argument("name")
    b.add_argument("src", help="a directory holding ansel_b200/csrc and include, or a git revision")
    t = sub.add_parser("time")
    t.add_argument("variants", nargs="*", metavar="NAME=LIB.so")
    t.add_argument("--rounds", type=int, default=3)
    t.add_argument("--calls", type=int, default=15)
    t.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if a.cmd == "build":
        build(a.name, a.src)
    else:
        time_variants(a)


if __name__ == "__main__":
    main()
