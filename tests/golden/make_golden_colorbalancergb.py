"""Regenerate tests/golden/colorbalancergb.npz from the reference's own lines (oracle/_ref/libref_colorbalancergb_strict.so): colour balance rgb on
a 40x24 frame for the scene-referred default preset and three random parameter blocks, in both saturation formulas and three work profiles,
with the gamut LUTs of the reference's commit_params().  Also tests/golden/colorbalancergb_blocks.npz: the data blocks the reference's
commit_params() makes for the whole parameter matrix (colorbalancergb_util.blocks(): presets, full-range and sub-range random blocks) and the
gamut LUTs of both formulas on the three work profiles, which the device tests run.  Needs oracle/_ref (built where the reference exists)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import colorbalancergb_util as cu  # noqa: E402


def main():
    rng = np.random.default_rng(20261019)
    blocks = [cu.presets()[-1][1], cu.presets()[0][1]] + [cu.random_params(rng, cu.FORMULAS[k % 2]) for k in range(4)]
    out, n = {}, 0
    for k, p in enumerate(blocks):
        profile = list(cu.PROFILES)[k % 3]
        data, _ = cu.commit(p, None)
        _, lut = cu.commit(p, profile)
        cp = cu.piece(data, profile, lut)
        img = cu.frame(40, 24, 100 + k)
        rc, want = cu.ref(img, cp)
        assert rc == 0
        out.update({f"data{n}": np.frombuffer(bytes(cp.data), np.uint8), f"work_in{n}": cu.PROFILES[profile][0],
                    f"work_out{n}": cu.PROFILES[profile][1], f"lut{n}": lut, f"in{n}": img, f"out{n}": want})
        n += 1
    np.savez_compressed(os.path.join(HERE, "colorbalancergb.npz"), n=n, **out)

    names, datas = [], []
    for name, p in cu.blocks():
        data, _ = cu.commit(p, None)
        names.append(name)
        datas.append(np.frombuffer(bytes(data), np.uint8))
    luts = np.zeros((len(cu.FORMULAS), len(cu.PROFILES), 360), np.float32)
    for i, f in enumerate(cu.FORMULAS):
        p = cu.defaults()
        p.saturation_formula = f
        for j, prof in enumerate(cu.PROFILES):
            luts[i, j] = cu.commit(p, prof)[1]
    np.savez_compressed(os.path.join(HERE, "colorbalancergb_blocks.npz"), names=np.array(names), data=np.stack(datas), luts=luts,
                        profiles=np.array(list(cu.PROFILES)), work_in=np.stack([cu.PROFILES[k][0] for k in cu.PROFILES]),
                        work_out=np.stack([cu.PROFILES[k][1] for k in cu.PROFILES]))


if __name__ == "__main__":
    main()
