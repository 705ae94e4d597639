"""Write tests/golden/fdc.npz: FDC's colour lanes on the cases of tests/fdc_util.py at ISO 100 (hybrid chroma) and 3200 (pure FDC), every
tile from a zeroed scratch -- the oracle's mode that tests/test_cpu_fdc.py pins to the reference's own lines on frames of one tile."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import fdc_util as fu  # noqa: E402

GOLDEN = ("one_tile", "narrow", "small")  # kept small: the other cases are pinned to the reference directly
out = {}
for name in GOLDEN:
    m, x, y = fu.case(name)
    for iso in (100.0, 3200.0):
        out[f"{name}_{int(iso)}"] = fu.oracle(m, x, y, iso, zero_per_tile=1)[..., :3]
np.savez_compressed(os.path.join(HERE, "fdc.npz"), **out)
print("wrote tests/golden/fdc.npz")
