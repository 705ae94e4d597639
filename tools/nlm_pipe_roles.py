"""Where the warps of nlm_pipe_kernel spend their cycles, on the 45 MP bench frame (development tool, not the bench contract).

Builds nlm.cu with -DNLM_PIPE_TIMING into its own library (ansel_b200/build/nlm_pipe_timing/, linked with the product's other
objects; the product libb200iop.so is never touched), runs the bench frame (bench.py's seed) through RCD and the denoise profile
(non-local means P = 1, K = 7) once, and prints each warp's cycle shares by role -- its work, its waits at the FULL / EMPTY /
HANDOVER / GROUP barriers, the window fill with its __syncthreads, the finish, and the drain (idle after its role ends, until the
block's last warp ends) -- as shares of the block's duration, per warp and per scheduler (warp w issues on scheduler w mod 4).

    python tools/nlm_pipe_roles.py            # build if nlm.cu changed, then run on cuda:0
    python tools/nlm_pipe_roles.py --build    # build only (no GPU needed)
"""
from __future__ import annotations

import ctypes as C
import glob
import hashlib
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "ansel_b200", "build", "nlm_pipe_timing")
LIB = os.path.join(OUT, "libb200iop_nlm_timing.so")
os.environ["B200IOP_LIB"] = LIB                  # before ansel_b200 is imported: its C ABI is the instrumented library's
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from ansel_b200 import build as B  # noqa: E402

SEED = 20260922                                   # bench.py's frame
ROLES = ("fill", "work", "FULL", "EMPTY", "HANDOVER", "GROUP", "finish")
NWARPS = 16                                       # pipe_cfg<0>::NT / 32


def _sources_digest() -> str:
    h = hashlib.sha256(" ".join(B.NVCC_FLAGS).encode())
    for f in sorted(glob.glob(os.path.join(B.CSRC, "*"))) + sorted(glob.glob(os.path.join(ROOT, "include", "*.h"))):
        with open(f, "rb") as fh:
            h.update(os.path.basename(f).encode() + fh.read())
    return h.hexdigest()


def build_timing_lib() -> str:
    """the product objects (ansel_b200.build) + nlm.cu compiled with NLM_PIPE_TIMING, rebuilt whenever a source differs"""
    B.build()
    digest = _sources_digest()
    stamp = LIB + ".sha256"
    if os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == digest:
        return LIB
    os.makedirs(OUT, exist_ok=True)
    obj = os.path.join(OUT, "nlm.o")
    flags = [f for f in B.NVCC_FLAGS if f != "-shared"]
    subprocess.run([B._nvcc()] + flags + ["-DNLM_PIPE_TIMING", "-c", os.path.join(B.CSRC, "nlm.cu"), "-o", obj], check=True)
    objs = [o for o in sorted(glob.glob(os.path.join(B.HERE, "build", "*.o"))) if os.path.basename(o) != "nlm.o"] + [obj]
    subprocess.run([B._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-cudart", "static", "-Xcompiler", "-fPIC",
                    "-o", LIB] + objs, check=True)
    with open(stamp, "w") as fh:
        fh.write(digest)
    return LIB


def card() -> str:
    import torch
    name, limit = torch.cuda.get_device_name(0), "power limit unknown"
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        limit = f"{pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0:.0f} W power limit, SM clock max {pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)} MHz"
    except Exception:
        pass
    return f"{name}, {limit}"


def run(lib_path: str):
    import numpy as np
    import torch
    import ansel_b200 as ab
    import util
    assert ab.LIB_PATH == lib_path, "ansel_b200 was imported before the timing library was chosen"
    ab.init()
    L = ab.lib()
    L.b200_nlm_pipe_timing.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    L.b200_kernel_timing_read.argtypes = [C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_int)]
    w, h = util.SIZE_45MP
    mosaic = torch.from_numpy(util.frame_natural(w, h, SEED)).cuda()
    d_dem = ab.demosaic_data(ab.DEMOSAIC_RCD)
    d_dn = ab.denoiseprofile_data(ab.DENOISE_NLMEANS, radius=1, nbhood=7)

    def piece_of(data, ch):
        p = ab.make_piece(w, h, filters=util.BAYER["RGGB"] if ch == 1 else 0, channels=ch, devid=0)
        p.data, p.data_size = C.addressof(data), C.sizeof(data)
        return p

    p_dem, p_dn = piece_of(d_dem, 1), piece_of(d_dn, 4)
    rgb = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
    out = torch.empty_like(rgb)
    stream = torch.cuda.current_stream().cuda_stream
    ab.check(L.b200_demosaic_process_dev(p_dem, mosaic.data_ptr(), rgb.data_ptr(), stream))
    ab.check(L.b200_denoiseprofile_process_dev(p_dn, rgb.data_ptr(), out.data_ptr(), stream))   # warm-up, untimed
    torch.cuda.synchronize()

    words = C.c_int()
    max_blocks = 1 << 16
    L.b200_nlm_pipe_timing(None, C.byref(words))
    buf = torch.zeros(max_blocks * NWARPS * words.value, dtype=torch.int32, device="cuda")
    ab.check(L.b200_nlm_pipe_timing(C.c_void_p(buf.data_ptr()), None))
    L.b200_kernel_timing(1)
    ab.check(L.b200_denoiseprofile_process_dev(p_dn, rgb.data_ptr(), out.data_ptr(), stream))
    torch.cuda.synchronize()
    ksum, kcnt = C.c_double(), C.c_int()
    ab.check(L.b200_kernel_timing_read(b"nlm_kernel", C.byref(ksum), C.byref(kcnt)))
    L.b200_kernel_timing(0)
    ab.check(L.b200_nlm_pipe_timing(None, None))
    t = buf.view(max_blocks, NWARPS, words.value).cpu().numpy().view(np.uint32).astype(np.int64)
    return t, (ksum.value / kcnt.value if kcnt.value else float("nan"))


def report(t, kernel_ms, label):
    import numpy as np
    nr = len(ROLES)
    path = t[:, :, nr + 2]
    print(f"nlm_pipe_kernel role cycles, 45 MP bench frame (RCD -> denoise profile, P = 1, K = 7), {label}")
    print(f"  instrumented kernel: {kernel_ms:.2f} ms")
    for pv, name in ((1, "half-height slots"), (2, "whole-pair slots")):
        blocks = np.nonzero((path == pv).all(axis=1))[0]
        if not len(blocks):
            continue
        b = t[blocks]
        ref = b[:, :1, nr]                                            # warp 0's first clock: every warp of a block shares the SM clock
        start = (b[:, :, nr] - ref) % (1 << 32)
        end = (b[:, :, nr + 1] - ref) % (1 << 32)
        span = end.max(axis=1, keepdims=True) - start.min(axis=1, keepdims=True)
        cyc = np.concatenate([b[:, :, :nr], (end.max(axis=1, keepdims=True) - end)[:, :, None]], axis=2)   # + drain
        share = (cyc / span[:, :, None]).mean(axis=0) * 100.0                                                   # [warp, role]
        cols = ROLES + ("drain",)
        print(f"\n  {name}: {len(blocks)} chunks, mean block {span.mean():.0f} cycles ({span.mean() / 113:.0f} per patch pair at 225 patches)")
        print("  warp sched " + " ".join(f"{c:>8}" for c in cols) + "   (% of the block's cycles)")
        for wi in range(NWARPS):
            print(f"  {wi:4d} {wi % 4:5d} " + " ".join(f"{share[wi, k]:8.1f}" for k in range(len(cols))))
        print("  per scheduler (mean of its four warps):")
        for s in range(4):
            m = share[s::4].mean(axis=0)
            print(f"  {'':4} {s:5d} " + " ".join(f"{m[k]:8.1f}" for k in range(len(cols))))


def main():
    lib_path = build_timing_lib()
    if "--build" in sys.argv:
        print("built", lib_path)
        return
    t, kernel_ms = run(lib_path)
    report(t, kernel_ms, card())


if __name__ == "__main__":
    main()
