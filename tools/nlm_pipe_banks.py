"""Shared-memory bank map of nlm_pipe_kernel's half-height path (development tool, CPU only).

Computes, for every shared-memory access of the half-height path's hot loops and every patch shift of a K = 7 search window, which
banks each warp touches, and reports the accesses that need more wavefronts than their width requires.  The layout is the one at
pipe_cfg / pipe2_fill in ansel_b200/csrc/nlm_group.cuh:
  window  two planes of WP-element rows: f2 {c0, c1} at W01[r * WP + c], c2 at W2[r * WP + c] (W2 = W + 2 * wrows * WP floats)
  slots   f2 {patch a, patch b} at P[row * SP + col] (SP = GRP_SP), P 8-byte aligned
A 32-bit access is conflict-free when the warp's 32 words sit in 32 distinct banks; a 64-bit access is served per half-warp, and a
half-warp is conflict-free when its 16 double-words sit in 16 distinct bank pairs.  Lanes that read the same word are one access.

    python tools/nlm_pipe_banks.py            # WP = 97, SP = 77: the kernel's pitches
    python tools/nlm_pipe_banks.py 98 77      # any other pair
"""
from __future__ import annotations

import sys

WARP = 32


def wavefronts(words: list[int], width: int) -> int:
    """least number of shared-memory wavefronts for one warp-wide access; words: the 4-byte word of each lane's first float"""
    if width == 4:
        groups = [words]
    else:  # 8 bytes: two half-warps, each lane two consecutive banks
        groups = [words[:16], words[16:]]
    n = 0
    for g in groups:
        per_bank: dict[int, set[int]] = {}
        for w in g:
            for k in range(width // 4):
                per_bank.setdefault((w + k) % 32, set()).add(w + k)
        n += max(len(s) for s in per_bank.values())
    return n


def accesses(WP: int, SP: int, wrows: int, shifts):
    """(name, shift, width, [word per lane]) for the warps of every role; word offsets in floats from the start of shared memory"""
    W2 = 2 * wrows * WP
    P = (wrows * 3 * WP + 1) & ~1
    assert P % 2 == 0
    # phase A: scan warp w (0..2), lane = window column t = 32 w + lane; row r of the walk; patch shift s = sr * WP + sc
    for sr, sc in shifts:
        s = sr * WP + sc
        for w in range(3):
            for r in (0, 1, 5):
                cols = [32 * w + l for l in range(WARP)]
                yield "A window f2 (pixel, partner)", (sr, sc), 8, [2 * (r * WP + t + s) for t in cols]
                yield "A window c2 (pixel, partner)", (sr, sc), 4, [W2 + r * WP + t + s for t in cols]
    for w in range(3):
        for r in (0, 1, 31):
            yield "A column sums STS.64", None, 8, [P + 2 * (r * SP + 32 * w + l) for l in range(WARP)]
    # phase B1: warp 3, lane = row of the half, all lanes at the same column j
    for j in range(0, 80):
        yield "B1 column sums / distortions", None, 8, [P + 2 * (l * SP + j) for l in range(WARP)]
    # phase B2: accumulating warp wa (0..7), lane l: column i = l & 7, row pair pr = (wa & 3) + 4 (l >> 3) + 16 (wa >> 2); rows 2 pr, 2 pr + 1
    # of the chunk (window row = chunk row + 8 + shift); strip step k * 8 columns
    for sr, sc in shifts:
        s = sr * WP + sc
        for wa in range(8):
            for k in (0, 4, 8):
                for lo in (0, 1):
                    lanes = range(WARP)
                    pr = [(wa & 3) + 4 * (l >> 3) + 16 * (wa >> 2) for l in lanes]
                    col = [(l & 7) + 8 * k for l in lanes]
                    row = [2 * p + lo for p in pr]
                    o = [(8 + r) * WP + 8 + c + s for r, c in zip(row, col)]
                    yield "B2 window f2", (sr, sc), 8, [2 * x for x in o]
                    yield "B2 window c2", (sr, sc), 4, [W2 + x for x in o]
    for wa in range(8):
        for k in (0, 4, 8):
            for lo in (0, 1):
                lanes = range(WARP)
                pr = [((wa & 3) + 4 * (l >> 3)) for l in lanes]  # row pairs within the half
                yield "B2 distortions {a, b}", None, 8, [P + 2 * ((2 * p + lo) * SP + (l & 7) + 8 * k) for p, l in zip(pr, lanes)]


def main():
    WP = int(sys.argv[1]) if len(sys.argv) > 1 else 97
    SP = int(sys.argv[2]) if len(sys.argv) > 2 else 77
    K = 7
    shifts = [(sr, sc) for sr in range(-K, K + 1) for sc in range(-K, K + 1)]
    wrows = 64 + 2 * (1 + K) + 1
    worst: dict[str, int] = {}
    bad: dict[str, list] = {}
    for name, shift, width, words in accesses(WP, SP, wrows, shifts):
        need = width // 4                       # wavefronts a conflict-free access of this width takes
        n = wavefronts(words, width)
        worst[name] = max(worst.get(name, 0), n - need)
        if n > need:
            bad.setdefault(name, []).append(shift)
    print(f"nlm_pipe_kernel half-height path, WP = {WP}, slot pitch SP = {SP}, every shift of K = {K}")
    for name in worst:
        print(f"  {name:32s} {'conflict-free' if worst[name] == 0 else f'{worst[name]} extra wavefront(s), e.g. shift {bad[name][0]}'}")
    n_bad = sum(len(v) for v in bad.values())
    print("no conflicted access" if not n_bad else f"{n_bad} conflicted accesses")
    return 1 if n_bad else 0


if __name__ == "__main__":
    sys.exit(main())
