"""Write tests/golden/lens.npz: the reference's own process() (oracle/_ref/libref_lens_strict.so, oracle/lens.mk) on synthetic lenses.

    PYTHONPATH=.:tests python tests/golden/make_golden_lens.py

Each case: the input frame, the data block's bytes (dt_iop_lensfun_data_t), the interpolator, monochrome and mask display, the ROIs
and the reference's output over the caller's buffer of lens_util.fill()."""
import os

import numpy as np

import lens_util as lu
import ansel_b200 as ab

# (dist, tca, vig, inverse, nan checks, scale, interpolator, monochrome, mask, roi)
CASES = ((ab.LS_DIST_PTLENS, ab.LS_TCA_POLY3, True, 0, 1, 1.0, ab.INTERPOLATION_MITCHELL, 0, 0, 0),
         (ab.LS_DIST_POLY3, ab.LS_TCA_LINEAR, True, 1, 1, 1.02, ab.INTERPOLATION_BICUBIC, 0, 1, 1),
         (ab.LS_DIST_POLY5, ab.LS_TCA_NONE, False, 0, 0, 1.0, ab.INTERPOLATION_BILINEAR, 1, 0, 1),
         (ab.LS_DIST_PTLENS, ab.LS_TCA_POLY3, True, 1, 0, 1.0, ab.INTERPOLATION_MITCHELL, 0, 1, 0),
         (ab.LS_DIST_NONE, ab.LS_TCA_NONE, True, 0, 1, 1.0, ab.INTERPOLATION_MITCHELL, 0, 0, 0),
         (ab.LS_DIST_NONE, ab.LS_TCA_NONE, True, 1, 1, 1.0, ab.INTERPOLATION_MITCHELL, 0, 0, 0))


def main():
    out = {}
    for k, (dist, tca, vig, inv, nan, scale, itor, mono, mask, r) in enumerate(CASES):
        roi = lu.ROIS[r]
        d = lu.lens_data(dist, tca, vig, inv, nan, scale=scale)
        img = lu.frame(roi[2], roi[3], 100 + k)
        rc, want = lu.ref(img, d, itor, roi, mono, mask)
        assert rc == 0
        out[f"in{k}"], out[f"out{k}"] = img, want
        out[f"data{k}"] = np.frombuffer(bytes(d), np.uint8)
        out[f"args{k}"] = np.array([itor, mono, mask, r], np.int32)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lens.npz")
    np.savez_compressed(path, n=np.int32(len(CASES)), **out)
    print("wrote", path)


if __name__ == "__main__":
    main()
