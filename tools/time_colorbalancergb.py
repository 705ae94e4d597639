"""Time colour balance rgb at 45 MP (8256 x 5504 RGBA float) on the device: median of 15 calls of b200_colorbalancergb_process_dev between
CUDA events, after a warm-up, in both saturation formulas (the golden file's scene-referred default and legacy preset blocks with their gamut
LUTs), next to filmic rgb's AgX kernel (b200_filmicrgb_process_dev, the v8 defaults with the export profile) on the same frame in the same
run.  Prints the card, its power limit and its SM clock with the numbers.

    PYTHONPATH=.:tests python tools/time_colorbalancergb.py
"""
import ctypes as C
import os
import subprocess

import numpy as np
import torch

import util
import colorbalancergb_util as cu
import ansel_b200 as ab


def _median_ms(call, stream):
    for _ in range(3):
        call()
    ts = []
    for _ in range(15):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        call()
        b.record(stream)
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return np.median(ts), min(ts), max(ts)


def main():
    ab.init()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip())
    w, h = util.SIZE_45MP
    s = torch.cuda.current_stream()
    d_in = torch.from_numpy(cu.frame(w, h, 1)).cuda()
    d_out = torch.empty_like(d_in)
    g = np.load(os.path.join(util.GOLDEN_DIR, "colorbalancergb.npz"))
    keep = []
    cases = []
    for k, name in ((0, "colorbalancergb, darktable UCS (scene-referred default)"), (1, "colorbalancergb, JzAzBz (legacy preset)")):
        cp = ab.colorbalancergb_piece(g[f"data{k}"], (g[f"work_in{k}"], g[f"work_out{k}"]), g[f"lut{k}"])
        p = ab.make_piece(w, h, filters=0, channels=4, devid=0)
        p.data, p.data_size = C.addressof(cp), C.sizeof(cp)
        keep += [cp, p]
        cases.append((name, lambda p=p: ab.check(ab.lib().b200_colorbalancergb_process_dev(C.byref(p), d_in.data_ptr(), d_out.data_ptr(), s.cuda_stream))))
    work, export = util.profile_pair(util.REC2020_TO_XYZ_D50), util.profile_pair(util.SRGB_TO_XYZ_D50)
    fp = ab.filmic_piece(np.load(os.path.join(util.GOLDEN_DIR, "filmic_data.npz"))["default_v8"], work, export)
    pf = ab.make_piece(w, h, filters=0, channels=4, devid=0)
    pf.data, pf.data_size = C.addressof(fp), C.sizeof(fp)
    cases.append(("filmic rgb AgX (filmic_agx_kernel, the yardstick)",
                  lambda: ab.check(ab.lib().b200_filmicrgb_process_dev(C.byref(pf), d_in.data_ptr(), d_out.data_ptr(), s.cuda_stream))))
    for name, call in cases:
        med, lo, hi = _median_ms(call, s)
        print(f"{name}: median {med:.3f} ms (min {lo:.3f}, max {hi:.3f}) at {w}x{h}")
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks_throttle_reasons.active", "--format=csv,noheader"], capture_output=True, text=True)
    print("SM clock and throttle reasons after the runs:", q.stdout.strip())


if __name__ == "__main__":
    main()
