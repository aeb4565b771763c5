"""The rsyncable chunk rule (DESIGN.md section 5 "Rsyncable") as a CPU model: tests/native/rsync_model.c.

The model is a sequential pass over a member.  These tests check it on its own: its gear table is splitmix64's, its
chunk starts equal a direct restatement of the rule in numpy, the starts keep the rule's bounds, and an edit moves only
the starts near it.  tests/test_gpu_rsyncable.py compares the kernel with it.
"""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from tests import util

HERE = os.path.dirname(os.path.abspath(__file__))
MIN, CHUNK, BITS = 16384, 65536, 16
M64 = (1 << 64) - 1


def splitmix64_table():
    out, state = [], 0
    for _ in range(256):
        state = (state + 0x9E3779B97F4A7C15) & M64
        z = state
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        out.append(z ^ (z >> 31))
    return out


GEAR = np.array(splitmix64_table(), dtype=np.uint64)


class Model:
    def __init__(self, so):
        L = self.L = ctypes.CDLL(so)
        for f in (L.rs_model_chunks, L.rs_model_candidates):
            f.restype = ctypes.c_uint64
            f.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint64]
        L.rs_model_gear.argtypes = [ctypes.c_void_p]

    def gear(self):
        g = np.zeros(256, dtype=np.uint64)
        self.L.rs_model_gear(g.ctypes.data)
        return g

    def _list(self, f, buf, cap):
        out = np.zeros(max(cap, 1), dtype=np.uint64)
        n = f(bytes(buf), len(buf), out.ctypes.data, cap)
        assert n <= cap
        return out[:n].copy()

    def chunks(self, buf):
        return self._list(self.L.rs_model_chunks, buf, cap_bound(len(buf)))

    def candidates(self, buf, cap=None):
        return self._list(self.L.rs_model_candidates, buf, len(buf) // 256 + 1024 if cap is None else cap)


def build_model(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("rsync_model") / "librsync_model.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "native", "rsync_model.c")])
    return Model(so)


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return build_model(tmp_path_factory)


def cap_bound(n):
    return 1 if n == 0 else -(-n // CHUNK) + n // MIN


def hashes(buf):
    """h(p) for p = 0..len(buf), from the sum h(p) = sum_{j=1..min(p,64)} G[m[p-j]] << (j-1)."""
    m = np.frombuffer(bytes(buf), dtype=np.uint8)
    g = GEAR[m]
    h = np.zeros(len(m) + 1, dtype=np.uint64)
    for j in range(1, 65):
        if j > len(m):
            break
        h[j:] += g[:len(m) + 1 - j] << np.uint64(j - 1)
    return h


def rule_cuts(cands):
    """accepted cuts: a candidate p >= MIN with no other candidate in (p - MIN, p)"""
    c = np.asarray(cands, dtype=np.int64)
    if c.size == 0:
        return c
    prev = np.concatenate(([-(1 << 62)], c[:-1]))
    return c[(c >= MIN) & (c - prev >= MIN)]


def rule_starts(n, cuts):
    if n == 0:
        return np.zeros(1, dtype=np.uint64)
    pts = [0] + [int(x) for x in cuts] + [n]
    return np.array([s for a, b in zip(pts, pts[1:]) for s in range(a, b, CHUNK)], dtype=np.uint64)


def rule_chunks(buf):
    h = hashes(buf)
    p = np.nonzero((h >> np.uint64(64 - BITS)) == 0)[0]
    cands = p[(p > 0) & (p < len(buf))]
    return rule_starts(len(buf), rule_cuts(cands))


def plant(buf, p):
    """Rewrite buf[p-3:p] so that p becomes a candidate (h(p) >> 48 == 0); needs p >= 3.  Bytes before p - 3 and the
    hash they give stay; the 3 bytes are the first solution in (c, b, a) order."""
    h = 0
    for x in bytes(buf[max(0, p - 67):p - 3]):
        h = ((h << 1) + int(GEAR[x])) & M64
    h0 = np.uint64(h)
    ab = np.arange(65536)
    base = (h0 << np.uint64(3)) + (GEAR[ab >> 8] << np.uint64(2)) + (GEAR[ab & 255] << np.uint64(1))
    for c in range(256):
        hit = np.nonzero(((base + GEAR[c]) >> np.uint64(64 - BITS)) == 0)[0]
        if hit.size:
            k = int(hit[0])
            buf[p - 3:p] = bytes([k >> 8, k & 255, c])
            return
    raise AssertionError("no 3 bytes make %d a candidate" % p)


def test_gear_is_splitmix64(model):
    assert np.array_equal(model.gear(), GEAR)
    # the first output of splitmix64 from state 0 (a published value)
    assert int(GEAR[0]) == 0xE220A8397B1DCDAF


def small_inputs():
    rng = random.Random(7)
    out = [b"", b"x", bytes(63), bytes(64), bytes(65), rng.randbytes(MIN - 1), rng.randbytes(MIN + 1),
           rng.randbytes(300000), bytes(200000), b"ab" * 100000]
    b = bytearray(rng.randbytes(400000))
    for p in (MIN, MIN + 5000, 2 * MIN + 1, 3 * MIN + 4999, 3 * MIN + 5000, len(b) - 1):
        plant(b, p)
    out.append(bytes(b))
    return out


@pytest.mark.parametrize("i", range(11))
def test_model_equals_rule(model, i):
    buf = small_inputs()[i]
    assert np.array_equal(model.chunks(buf), rule_chunks(buf))


def test_planted_candidates(model):
    rng = random.Random(3)
    b = bytearray(rng.randbytes(200000))
    for p in (MIN, MIN + 7000, 2 * MIN + 6999, len(b) - 1):
        plant(b, p)
    cands = set(model.candidates(b).tolist())
    assert {MIN, MIN + 7000, 2 * MIN + 6999, len(b) - 1} <= cands
    cuts = rule_cuts(sorted(cands))
    assert MIN in cuts and (MIN + 7000) not in cuts     # 7000 after another candidate
    assert (2 * MIN + 6999) not in cuts                 # MIN - 1 after another candidate


@pytest.fixture(scope="module")
def corpus():
    return util.load_corpus()


def test_bounds_on_corpus(model, corpus):
    rng = random.Random(11)
    for buf in list(corpus.values()) + [b"".join(corpus.values()), rng.randbytes(4 << 20)]:
        st = model.chunks(buf).astype(np.int64)
        assert st[0] == 0 and len(st) <= cap_bound(len(buf))
        ends = np.append(st[1:], len(buf))
        assert np.all(ends - st <= CHUNK) and (len(buf) == 0 or np.all(ends > st))
        cuts = rule_cuts(model.candidates(buf))
        assert np.all(np.diff(cuts) >= MIN)
        assert set(cuts.tolist()) <= set(st.tolist())


def edits(base, rng):
    n = len(base)
    e = n // 2 + 12345
    yield "insert", e, e, base[:e] + b"\x01INSERTED" + base[e:]
    yield "delete", e, e + 5000, base[:e] + base[e + 5000:]
    yield "overwrite", e, e + 300, base[:e] + rng.randbytes(300) + base[e + 300:]
    yield "prepend", 0, 0, rng.randbytes(7) + base


def check_locality(old_starts, new_starts, old_cuts, new_cuts, e, old_end, new_end):
    """starts up to the edit are kept; from the first cut of the new input at or past new_end + MIN + 64, the starts
    are the old ones shifted by the edit's change in length."""
    delta = new_end - old_end
    assert np.array_equal(old_starts[old_starts <= e], new_starts[new_starts <= e])
    far = new_cuts[new_cuts >= new_end + MIN + 64]
    if far.size == 0:
        return None
    c = int(far[0])
    assert c - delta in set(old_cuts.tolist())
    a = new_starts[new_starts >= c].astype(np.int64)
    b = old_starts[old_starts >= c - delta].astype(np.int64)
    assert np.array_equal(a, b + delta)
    return c


def test_locality(model, corpus):
    rng = random.Random(5)
    T = util.text_corpus(corpus)
    base = bytes(T[:1500000] + rng.randbytes(600000) + T[1500000:2500000])
    old = model.chunks(base)
    old_cuts = rule_cuts(model.candidates(base))
    for name, e, old_end, new in edits(base, rng):
        new_end = old_end + len(new) - len(base)
        c = check_locality(old, model.chunks(new), old_cuts, rule_cuts(model.candidates(new)), e, old_end, new_end)
        assert c is not None and c - new_end < (256 << 10), name
