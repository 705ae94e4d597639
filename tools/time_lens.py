"""Time lens correction at 45 MP (8256 x 5504 RGBA float) on the device: median of 15 calls of b200_lens_process_dev between CUDA events,
after a warm-up, for the default interpolator (Mitchell) in the configurations a raw export meets.  Prints the card, its power limit and its
SM clock with the numbers.

    PYTHONPATH=.:tests python tools/time_lens.py
"""
import ctypes as C
import subprocess
import sys

import numpy as np
import torch

import ansel_b200 as ab
import lens_util as lu

W, H = 8256, 5504
CASES = (("distortion + TCA + vignetting, correcting", dict(dist=ab.LS_DIST_PTLENS, tca=ab.LS_TCA_POLY3, vig=True, inverse=0)),
         ("distortion + vignetting (no TCA), correcting", dict(dist=ab.LS_DIST_PTLENS, tca=ab.LS_TCA_NONE, vig=True, inverse=0)),
         ("distortion + TCA + vignetting, reversing", dict(dist=ab.LS_DIST_PTLENS, tca=ab.LS_TCA_POLY3, vig=True, inverse=1)),
         ("vignetting only (copy + vignette)", dict(dist=ab.LS_DIST_NONE, tca=ab.LS_TCA_NONE, vig=True, inverse=0)))


def main():
    ab.init()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip())
    roi = (0, 0, W, H, 0, 0, W, H, 1.0, W, H)
    d_in = torch.from_numpy(lu.frame(W, H, 1, extremes=False)).cuda()
    d_out = torch.empty_like(d_in)
    s = torch.cuda.current_stream()
    for name, kw in CASES:
        lp = ab.lens_piece(lu.lens_data(**kw))
        p = lu.piece(roi, lp)
        call = lambda: ab.check(ab.lib().b200_lens_process_dev(C.byref(p), d_in.data_ptr(), d_out.data_ptr(), s.cuda_stream))
        for _ in range(3):
            call()
        ts = []
        for _ in range(15):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s)
            call()
            b.record(s)
            b.synchronize()
            ts.append(a.elapsed_time(b))
        print(f"{name}: median {np.median(ts):.3f} ms (min {min(ts):.3f}, max {max(ts):.3f}) at {W}x{H}")
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("SM clock after the runs:", q.stdout.strip())
    sys.stdout.flush()


if __name__ == "__main__":
    main()
