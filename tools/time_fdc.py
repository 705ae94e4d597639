"""Timing of frequency-domain chroma (FDC, X-Trans) at 45 MP: the median of 15 calls of b200_demosaic_process_dev, hybrid (ISO 100) and pure
(ISO 3200), next to Markesteijn's one pass, with the card, its SM clock and power limit.  Development tool, not the bench contract."""
import ctypes as C
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "tests"))
sys.path.insert(0, os.path.join(HERE, ".."))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import ansel_b200 as ab  # noqa: E402
import util  # noqa: E402
from vng_util import XTRANS  # noqa: E402


def main():
    ab.init()
    w, h = util.SIZE_45MP
    m = torch.from_numpy(util.frame_natural(w, h, 3)).cuda()
    out = torch.empty((h, w, 4), device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip())
    for label, method, iso in (("FDC hybrid (ISO 100)", ab.DEMOSAIC_FDC, 100.0), ("FDC pure (ISO 3200)", ab.DEMOSAIC_FDC, 3200.0),
                               ("Markesteijn 1-pass", 1025, 100.0)):
        dp = ab.DemosaicPiece()
        dp.data = ab.demosaic_data(method)
        dp.fdc_xover_iso = 1600
        piece = ab.make_piece(w, h, filters=9, data=dp, devid=0, exif_iso=iso)
        for i in range(6):
            for j in range(6):
                piece.xtrans[i][j] = int(XTRANS[i][j])

        def run():
            ab.check(ab.lib().b200_demosaic_process_dev(C.byref(piece), m.data_ptr(), out.data_ptr(), s))
        run()
        torch.cuda.synchronize()
        ts = []
        for _ in range(15):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        print(f"{label}: 45 MP median of 15 calls {np.median(ts):.2f} ms ({w * h / np.median(ts) / 1e3:.0f} MP/s)")
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks_throttle_reasons.active", "--format=csv,noheader"], capture_output=True, text=True)
    print("after: SM clock, throttle reasons:", q.stdout.strip())


if __name__ == "__main__":
    main()
