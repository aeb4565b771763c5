"""The level-1 parse (k_lz<1>) where its window loop drains its one-window pipeline, token by token against the CPU
model of tests/test_gpu_lz1_model.py.

k_lz<1> issues window k + 1's probe and table stores alongside window k's selection whenever no lane of window k
reaches the lane cap: then window k's last match ends by wb + 62 and window k + 1 is entered.  A capped lane drains
the pipeline: window k + 1 is probed only after the selection, and only if it is entered (a skipped window inserts
nothing into the table).  The members here are high-entropy bytes (no chance matches) with hand-placed copies:

- lanes: a capped match selected at every lane 0..31 of a window, ending at wb + 63 (the next window is entered
  at its last lane), wb + 64 (it is skipped) and wb + 65 (it is skipped, the one after starts at lane 1);
- unselected: a capped lane covered by a shorter match the chain selects, so that the pipeline drains although
  the next window is entered;
- skips: copies of 258 bytes and more that skip several windows in a row, some ending on a window boundary;
- edges: capped matches in the last window of a batch of 16 and the first of the next, in the last two windows
  of a piece (cut at the piece end), of phase 0 (pieces 7 / 8) and of a member's last, partial chunk;
- repeats: after every skipped run, bytes of the skipped windows occur again, so that a table store from a skipped
  window (which the serial parse never makes) would hand a later probe a different candidate.

The CPU tests show that the members reach these cases; the GPU tests compare the shipped build (the lowest lane of
a store instruction lands) and the ZB_LZ1_RESOLVE_WINNER=1 build (the highest position wins) with the model.
"""
import importlib.util
import os
import pickle
import random
import subprocess
import sys

import numpy as np
import pytest

from tests.test_gpu_lz1_model import (CHUNK, LOWEST, PIECE, ROOT, _VARIANT_SCRIPT, _check_tokens, _high,
                                      compare_tokens, lz_hash, model)  # noqa: F401  (model is a fixture)

CAP = 32


def _hash_at(x, q):
    return lz_hash(int.from_bytes(x[q:q + 4], "little"))


def _copy(x, dst, src, n):
    """x[dst:dst + n] = x[src:src + n] (src + n <= dst), with the bytes just before and just after differing, so
    that the match at dst is exactly n long and no lane before dst matches the same source."""
    assert src + n <= dst
    x[dst:dst + n] = x[src:src + n]
    if x[dst + n] == x[src + n]:
        x[dst + n] = 0x80 | ((x[dst + n] + 1) & 0x7f)
    if x[dst - 1] == x[src - 1]:
        x[dst - 1] = 0x80 | ((x[dst - 1] + 1) & 0x7f)


def _copy_near(x, dst, n, d0):
    """_copy from the first distance d >= max(d0, n) for which no other position from the source's window on to dst
    shares the source's table entry, so that dst's probe finds the source whichever lane of a store lands."""
    for d in range(max(d0, n), max(d0, n) + 64):
        keep = bytes(x[dst - 1:dst + n + 1])
        src = dst - d
        _copy(x, dst, src, n)
        h = _hash_at(x, src)
        if all(_hash_at(x, q) != h for q in range(src & ~31, dst) if q != src):
            return
        x[dst - 1:dst + n + 1] = keep
    raise AssertionError("no clean source for %d" % dst)


def lanes_member(rng):
    """One chunk: for every lane i and end e in (63, 64, 65), a window wb whose lane i starts a copy of e - i bytes
    from about 96 bytes before it.  One case per 256 bytes, 15 per piece, pieces 0..6."""
    x = _high(rng, CHUNK)
    cases = [(i, e) for i in range(32) for e in (63, 64, 65)]
    k = 0
    for b0 in range(0, 7 * PIECE, PIECE):
        for j in range(15):
            if k == len(cases):
                break
            i, e = cases[k]
            wb = b0 + 128 + 256 * j
            _copy_near(x, wb + i, e - i, 96)
            k += 1
    assert k == len(cases)
    return bytes(x)


def unselected_member(rng):
    """One chunk: at window wb, lane 5 starts a copy of 33 bytes from S1 (a capped lane), and lane 3 a copy of 20
    bytes from S2 < S1 that covers lane 5, so the chain selects lane 3, then lane 23 (15 bytes left of the
    first copy): the last match ends at wb + 38 and the next window is entered.  Lane 5 finds S1, the later of
    the two positions with its 4 bytes."""
    x = _high(rng, CHUNK)
    for b0 in range(0, CHUNK, PIECE):
        for wb in range(b0 + 256, b0 + PIECE - 256, 384):
            s2, s1 = wb - 200, wb - 100
            _copy(x, wb + 5, s1, 33)
            x[s2:s2 + 20] = x[wb + 3:wb + 23]
            if x[s2 + 20] == x[wb + 23]:
                x[s2 + 20] = 0x80 | ((x[s2 + 20] + 1) & 0x7f)
            if x[s2 - 1] == x[wb + 2]:
                x[s2 - 1] = 0x80 | ((x[s2 - 1] + 1) & 0x7f)
    return bytes(x)


def skips_member(rng):
    """Two chunks: copies of 300..900 bytes (several 258-byte matches, windows skipped in a row), some ending on a
    window boundary; after each, 8 bytes of every second skipped window occur again further on."""
    x = _high(rng, 2 * CHUNK)
    for b0 in range(0, 2 * CHUNK, PIECE):
        wb = b0 + 1024 + 32 * rng.randrange(4)
        n = rng.choice([300, 516, 774, 900, 32 * 20 - 7, 32 * 24])
        i = rng.randrange(32) if n % 32 else 0
        n = min(n, b0 + PIECE - 600 - (wb + i))
        _copy(x, wb + i, wb + i - 900, n)
        # bytes of the skipped windows again, after the copy: the parse must find them at their source
        at = wb + i + n + 40
        for q in range(wb + 64, wb + i + n - 40, 64):
            if at + 16 > b0 + PIECE - 8:
                break
            x[at:at + 8] = x[q + 3:q + 11]
            at += 24
    return bytes(x)


EDGE_PIECES = (0, 3, 7, 8, 15)


def edge_windows(j):
    """The windows of the j-th of EDGE_PIECES that start a capped match: the last window of a batch of 16 and the
    first of another (15 and 48, or 47 and 16), and one of the piece's last two windows."""
    return (15, 48, 126) if j % 2 == 0 else (16, 47, 127)


def edges_member(rng):
    """Two chunks, the second one 32757 bytes: capped matches at a random lane of edge_windows in EDGE_PIECES of the
    first chunk (piece 15 is the chunk's last; a match in window 126 or 127 goes on past the piece end and is cut
    there), and near the end of the member."""
    n = CHUNK + 32757
    x = _high(rng, n)
    for j, p in enumerate(EDGE_PIECES):
        for w in edge_windows(j):
            dst = p * PIECE + 32 * w + rng.randrange(32 if w < 126 else 24)
            _copy_near(x, dst, 60 if w >= 126 else 40 + rng.randrange(30), 300)
    _copy_near(x, n - 100, 60, 500)
    return bytes(x)


def pipeline_inputs():
    rng = random.Random(0x51BE)
    return [("lanes", lanes_member(rng)), ("unselected", unselected_member(rng)), ("skips", skips_member(rng)),
            ("edges", edges_member(rng))]


@pytest.fixture(scope="module")
def inputs():
    return pipeline_inputs()


def _matches(chunk_tokens, base):
    """(position, length) of every match of one chunk's tokens; base: the chunk's first position."""
    out, p = [], base
    for t in chunk_tokens.tolist():
        if t >= 256:
            out.append((p, t >> 16))
            p += t >> 16
        else:
            p += 1
    return out


# ---------------------------------------------------------------------- CPU: the members reach the drain
def test_members_rebuild(model, inputs):
    for _, x in inputs:
        _check_tokens(x, model.run(x))
        _check_tokens(x, model.run(x, 1, LOWEST))


def test_capped_match_at_every_lane_and_end(model, inputs):
    """A selected match of 32 bytes or more starts at every lane of a window and ends at wb + 63, 64 and 65."""
    x = dict(inputs)["lanes"]
    for flags in (0, LOWEST):
        got = {(p % 32, p % 32 + ln) for p, ln in _matches(model.run(x, 1, flags)[0], 0) if ln >= CAP}
        assert {(i, e) for i in range(32) for e in (63, 64, 65)} <= got, flags


def test_unselected_capped_lanes(model, inputs):
    """Windows with a capped lane whose last selected match stops short of the cap (the pipeline drains, the next
    window is entered) outnumber the windows whose last match is capped."""
    spec = importlib.util.spec_from_file_location("lz1_model_tool", os.path.join(ROOT, "tools", "lz1_model.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    st = tool.window_stats([dict(inputs)["unselected"]], any_cap=True)
    assert st["any_cap"] >= st["cap"] + 100, st


def test_skips_and_edges(model, inputs):
    """Windows skipped in a row, and capped matches in the windows at batch, piece, phase and member ends."""
    cnt = {}
    named = dict(inputs)
    for name in ("skips", "edges"):
        model.run(named[name], 1, 0, cnt)
    assert cnt["skipped"] >= 150 and cnt["m258"] >= 30 and cnt["limit_cut"] >= 3, cnt
    runs = [ln for p, ln in _matches(np.concatenate(model.run(named["skips"])), 0) if ln == 258]
    assert len(runs) >= 30
    x = named["edges"]
    capped = set()
    for k, arr in enumerate(model.run(x)):
        capped |= {p // 32 for p, ln in _matches(arr, k * CHUNK) if ln >= min(CAP, PIECE - p % PIECE)}
    for j, p in enumerate(EDGE_PIECES):
        for w in edge_windows(j):
            assert p * PIECE // 32 + w in capped, (p, w)
    assert (len(x) - 100) // 32 in capped


# ---------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def rw_out(inputs, tmp_path_factory):
    """The members compressed (raw DEFLATE, level 1) by the ZB_LZ1_RESOLVE_WINNER=1 build, in a subprocess: this
    process loads the shipped library."""
    import __graft_entry__ as g
    assert os.path.exists(g.LIB_RW), g.LIB_RW
    d = tmp_path_factory.mktemp("lz1_pipeline")
    with open(d / "in.pkl", "wb") as f:
        pickle.dump(([x for _, x in inputs], [1]), f)
    flags = ["-I"] if sys.flags.isolated else ["-s"] if sys.flags.no_user_site else []
    subprocess.check_call([sys.executable] + flags + ["-c", _VARIANT_SCRIPT, ROOT, g.LIB_RW, str(d / "in.pkl"),
                                                      str(d / "out.pkl")], cwd=ROOT)
    with open(d / "out.pkl", "rb") as f:
        return pickle.load(f)[1]


@pytest.mark.gpu
def test_shipped_build_equals_the_model(model, inputs):
    import zippy_b200 as z
    comp = z.compress_batch([x for _, x in inputs], z.BestSpeed, z.dfDeflate)
    compared, stored, bad = compare_tokens(model, inputs, comp, LOWEST)
    assert not bad, bad[:10]
    assert compared == 6 and stored == 0


@pytest.mark.gpu
def test_resolve_winner_build_equals_the_model(model, inputs, rw_out):
    compared, stored, bad = compare_tokens(model, inputs, rw_out)
    assert not bad, bad[:10]
    assert compared == 6 and stored == 0
