#!/usr/bin/env python3
"""CPU model of k_lz<1>'s level-1 parse: how much work a 32-byte window costs, per window that was entered.

    python tools/lz1_model.py [--blocks N]

Replays the kernel's parse on the first N C2 blocks (bench.py's offsets): 4 KiB pieces, a fresh 2048-entry
table per piece pre-seeded with the 2 KiB before it (in the second 32 KiB phase only the 1 KiB of the first phase
that is staged again: the piece at 32768 gets 1 KiB), one probe per position, the 4-byte verify (with at least
4 bytes left before the piece end), the extension by 4 bytes per step up to the 32-byte lane cap, and the greedy
chain "match -> first candidate at or after its end".  Same-hash stores of one window resolve as "highest lane
wins".  Prints, per entered window: lanes that pass the 4-byte check, extension steps (max over the warp and
summed over lanes), matches the chain selects and windows whose last match hits the lane cap.  Those numbers
size the stages tools/lz1_stages.py times.  It also counts the windows in which any lane's match reaches the lane
cap: the windows after which k_lz<1> drains its one-window pipeline (the next window's probe waits for the
selection), on top of every piece's last window.  tests/test_gpu_lz1_model.py checks them against the token-exact
model tests/native/lz1_model.c.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PIECE, PRESEED, CAP, MAX_MATCH, MAX_DIST = 4096, 2048, 32, 258, 32768
PHASE, PHASE_HIST = 32768, 1024


def lz_hash(v):
    return ((v * 0x9E3779B1) & 0xffffffff) >> 21


def window_stats(blocks, any_cap=False):
    """Per-window work of the parse of `blocks` (each 64 KiB of text without NUL bytes), summed.  any_cap: also
    count the entered windows with any lane at the lane cap (key "any_cap")."""
    B = 65536
    tot = dict(windows=0, entered=0, verified=0, ext_steps_warp=0, ext_steps_lanes=0, chain=0, cap=0)
    if any_cap:
        tot["any_cap"] = 0
    for blk in blocks:
        assert len(blk) == B
        d = blk + b"\0" * 400
        w4 = [int.from_bytes(d[p:p + 4], "little") for p in range(B)]
        for pb in range(0, B, PIECE):
            tab = {}
            sbase = PHASE - PHASE_HIST if pb >= PHASE else 0
            for p in range(pb - min(PRESEED, pb - sbase), pb):
                tab[lz_hash(w4[p])] = p
            entry, b1 = pb, pb + PIECE
            for wb in range(pb, b1, 32):
                tot["windows"] += 1
                if entry >= wb + 32:   # the window is skipped: its positions are not inserted
                    continue
                tot["entered"] += 1
                hs = [lz_hash(w4[wb + l]) if wb + l + 4 <= B else None for l in range(32)]
                cand = [tab.get(h, 0xffff) if h is not None else 0xffff for h in hs]
                for l in range(32):
                    if hs[l] is not None:
                        tab[hs[l]] = wb + l
                ms, steps_max = [0] * 32, 0
                for l in range(32):
                    p, c = wb + l, cand[l]
                    lim = min(MAX_MATCH, b1 - p)
                    if c < p and p - c <= MAX_DIST and p >= entry and lim >= 4 and w4[p] == w4[c]:
                        m, steps = 4, 0
                        for k in range(1, CAP // 4):
                            steps += 1
                            x = 0
                            while x < 4 and d[p + 4 * k + x] == d[c + 4 * k + x]:
                                x += 1
                            m += x
                            if x < 4:
                                break
                        tot["ext_steps_lanes"] += steps
                        steps_max = max(steps_max, steps)
                        ms[l] = m if m >= CAP else min(m, lim)
                        tot["verified"] += 1
                tot["ext_steps_warp"] += steps_max
                if any_cap and max(ms) >= CAP:
                    tot["any_cap"] += 1
                l, endw = entry - wb, 0
                while l < 32:
                    if ms[l]:
                        tot["chain"] += 1
                        m = ms[l]
                        if m >= CAP:
                            tot["cap"] += 1
                            p, c = wb + l, cand[l]
                            while m < MAX_MATCH and p + m < b1 and d[p + m] == d[c + m]:
                                m += 1
                        endw = l + m
                        l += m
                    else:
                        l += 1
                entry = wb + max(endw, 32)
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=24)
    args = ap.parse_args()
    from tests import util
    T = util.text_corpus(util.load_corpus())
    tot = window_stats([util.c2_block(T, i) for i in range(args.blocks)], any_cap=True)
    n = tot["entered"]
    print("%d C2 blocks: %d windows, %d entered" % (args.blocks, tot["windows"], n))
    for k in ("verified", "ext_steps_warp", "ext_steps_lanes", "chain", "cap", "any_cap"):
        print("  %-16s %8.3f per entered window" % (k, tot[k] / float(n)))


if __name__ == "__main__":
    main()
