"""The parse of levels -1 (Default) and 2..9 (k_lz2), token by token, against a CPU model of its rules.

tests/native/lz2_model.c restates the rules of DESIGN.md sections 4 and 5 -- chunks with up to 32 KiB of
history, 8 KiB sub-chunks with their own 4-way tables, direct-mapped static tables of the preceding segments,
the candidate order, the verify / extend budget, the one-step lazy rule and the greedy selection -- as a
sequential program.  The GPU test reads every fixed or dynamic block the kernel wrote (tests/deflate_tokens.py)
and requires the model's tokens exactly; stored chunks have no tokens and are only counted.

The CPU tests check the model on its own: its tokens rebuild the member, respect the sub-chunk and window
limits, round-trip through zlib once packed with fixed codes, and the inputs reach every rule (coverage
counters), so the comparison cannot pass on inputs that never exercise one.
"""
import ctypes
import os
import random
import subprocess
import zlib

import numpy as np
import pytest

from tests import deflate_tokens as dt
from tests import deflate_writer as dw
from tests import util

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "lz2_model.c")

CHUNK, SUB = 65536, 8192
LEVELS = [2, 3, 4, 5, 6, 7, 8, 9, -1]
LAZY = {2: 0, 3: 6, 4: 8, 5: 16, 6: 16, 7: 32, 8: 32, 9: 64, -1: 16}
COUNTERS = ["matches", "lazy_drops", "history", "dist_32768", "cap_ext", "limit_cut", "short_limit",
            "win_window", "win_own", "win_static", "alias", "m258_at_end"]


class Model:
    def __init__(self, so):
        self.L = ctypes.CDLL(so)
        self.L.lz2_model.restype = ctypes.c_int64
        self.L.lz2_model.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint64,
                                     ctypes.c_void_p, ctypes.c_void_p]
        assert self.L.lz2_counter_count() == len(COUNTERS)

    def run(self, member, level, counters=None):
        """-> one array of encoded tokens per chunk (literal b -> b, match -> length << 16 | distance)."""
        n = len(member)
        nch = max(1, -(-n // CHUNK))
        tok = np.zeros(n + 16, dtype=np.uint32)
        per = np.zeros(nch, dtype=np.uint32)
        cnt = np.zeros(len(COUNTERS), dtype=np.uint64)
        got = self.L.lz2_model(bytes(member), n, level, tok.ctypes.data, tok.size, per.ctypes.data, cnt.ctypes.data)
        assert got >= 0
        if counters is not None:
            for k, v in zip(COUNTERS, cnt.tolist()):
                counters[k] = counters.get(k, 0) + v
        bounds = np.concatenate([[0], np.cumsum(per.astype(np.int64))])
        assert bounds[-1] == got
        return [tok[bounds[i]:bounds[i + 1]] for i in range(nch)]


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lz2_model") / "liblz2_model.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, SRC])
    return Model(so)


def encode(tokens):
    return np.array([t if isinstance(t, int) else t[0] << 16 | t[1] for t in tokens], dtype=np.uint32)


def decode(arr):
    return [t if t < 256 else (t >> 16, t & 0xffff) for t in arr.tolist()]


# ---------------------------------------------------------------------- inputs
def _no_a(rng, n):
    """High-entropy bytes without an 'a': 7 random bits per byte, so that a Huffman block beats a stored one
    and the chunk's tokens are written out."""
    b = np.frombuffer(rng.randbytes(n), dtype=np.uint8) | 0x80
    return bytearray(b.tobytes())


def trap_member(in_segment_before=False, n=40017, seed=0x7A):
    """A member whose parse, near its end, turns on the bytes just past it.

    It ends with Q a^L, p0 = n - L the first 'a' (p0 % 32 != 31).  Lane p0's best candidate matches the L
    bytes to the end; lane p0 + 1 matches one byte less at distance 1 -- unless bytes past the member are
    compared as if they were part of it, where a run of 'a's there would make its match look longer and let
    the lazy rule drop lane p0's match.
      * default: an earlier X a^6 Z in the same sub-chunk, 100 bytes before p0 (own-table candidates; L = 6)
      * in_segment_before: a^6 straddling the start S of the segment before p0's, S - 1 the last 'aaaa' of
        the segment before that (static-table candidate, matching 5 bytes; L = 5)."""
    rng = random.Random(seed + in_segment_before)
    x = _no_a(rng, n)
    if in_segment_before:
        L = 5
        S = ((n - L) // SUB - 1) * SUB
        x[S - 2:S + 4] = b"a" * 6
    else:
        L = 6
        r = n - L - 100
        x[r:r + 6] = b"a" * 6
    x[n - L:] = b"a" * L
    assert (n - L) % 32 != 31 and (n - L) // SUB == (n - 1) // SUB
    return bytes(x), n - L, L


def distance_member(rng):
    """Two chunks of random bytes; in chunk 1 a stretch repeats the bytes exactly 32768 back (across the
    joint, into the history) and another stretch the bytes 32769 back (out of reach)."""
    x = bytearray(rng.randbytes(2 * CHUNK + 20000))
    for lo, hi, d in ((CHUNK + 100, CHUNK + 3000, 32768), (CHUNK + 6000, CHUNK + 9000, 32769),
                      (CHUNK + 40000, CHUNK + 40300, 32768), (40000, 40700, 32768)):
        for i in range(lo, hi):
            x[i] = x[i - d]
    return bytes(x)


def runs_member(rng, T):
    """Text with long runs across 8 KiB sub-chunk ends and a chunk end, and 258-byte copies that end exactly
    at sub-chunk ends (random bytes around them, the source near the end of the segment before)."""
    x = bytearray(T[:3 * CHUNK + 4321])
    for c in (SUB * 3, SUB * 5 + 7, CHUNK, CHUNK + SUB * 2 - 1, 2 * CHUNK + 17):
        x[c - 3000:c + 2500] = b"x" * 5500
    for b1 in (SUB * 6, CHUNK + SUB * 5, 2 * CHUNK + SUB * 3):
        x[b1 - 2000:b1 + 200] = rng.randbytes(2200)
        src = b1 - SUB - 300
        x[src - 50:src + 300] = rng.randbytes(350)
        x[b1 - 258:b1] = x[src:src + 258]
    return bytes(x)


def model_inputs(corpus):
    """(name, member) pairs: edge inputs, corpus slices at ragged lengths, members of 2..5 chunks, the
    distance, run and 258-at-the-end members, and the lazy traps."""
    rng = random.Random(0x1A22)
    T = util.text_corpus(corpus)
    urls, html = corpus["urls.10K"], corpus["html"]
    # the edge inputs, without most of the incompressible ones (stored chunks: nothing to compare)
    xs = [("edge%d" % i, x) for i, x in enumerate(util.edge_inputs())
          if (len(x) <= 40000 or len(x) in (65537, 131072)) and (len(x) < 4096 or len(set(x)) < 200)]
    for n in (8191, 8193, 12345, 33000, 65535, 65537):
        o = rng.randrange(len(urls) - n)
        xs.append(("urls%d" % n, urls[o:o + n]))
        o = rng.randrange(len(html) - n)
        xs.append(("html%d" % n, html[o:o + n]))
    for k in (2, 3, 5):
        n = k * CHUNK - 1000 + 777 * k
        o = rng.randrange(len(T) - n)
        xs.append(("text%dchunks" % k, T[o:o + n]))
    xs.append(("kppkn", corpus["kppkn.gtb"][:2 * CHUNK + 5]))
    xs.append(("distances", distance_member(rng)))
    xs.append(("runs", runs_member(rng, T)))
    xs.append(("trap_own", trap_member(False)[0]))
    xs.append(("trap_static", trap_member(True)[0]))
    return xs


# ---------------------------------------------------------------------- CPU: the model on its own
def _check_tokens(member, chunks):
    """Lengths 4..258, distances 1..32768 inside the member, no match across a sub-chunk end, every chunk
    exactly its bytes, and the tokens rebuild the member."""
    blocks = []
    for k, arr in enumerate(chunks):
        c0 = k * CHUNK
        a = arr.astype(np.int64)
        ismatch = a >= 256
        ln = np.where(ismatch, a >> 16, 1)
        d = a & 0xffff
        p = np.concatenate([[0], np.cumsum(ln)[:-1]]) if len(a) else a
        assert int(ln.sum()) == min(CHUNK, len(member) - c0), k
        assert (a[~ismatch] < 256).all()
        lm, dm, pm = ln[ismatch], d[ismatch], p[ismatch]
        assert ((lm >= 4) & (lm <= 258)).all() and ((dm >= 1) & (dm <= 32768)).all(), k
        assert (dm <= c0 + pm).all(), ("distance before the member", k)
        assert (pm // SUB == (pm + lm - 1) // SUB).all(), ("match across a sub-chunk end", k)
        blocks.append(dt.Block(2, False, 0, 0, decode(arr)))
    assert dt.rebuild(blocks) == member


def _fixed_stream(chunks):
    blocks = []
    for k, arr in enumerate(chunks):
        last = k == len(chunks) - 1
        blocks.append(dw.Fixed(decode(arr), final=last))
        if not last:
            blocks.append(dw.Stored(b"", final=False))
    return dw.raw(blocks)


@pytest.fixture(scope="module")
def inputs(corpus):
    return model_inputs(corpus)


@pytest.mark.parametrize("level", LEVELS)
def test_model_tokens_rebuild_the_member(model, inputs, level):
    for name, x in inputs:
        chunks = model.run(x, level)
        _check_tokens(x, chunks)
        if name.startswith(("trap", "distances", "text2", "edge1", "urls8193")):
            raw = _fixed_stream(chunks)
            assert zlib.decompress(raw, -15) == x, name
            assert [list(c.tokens) for c in dt.member_chunks(dt.parse(raw))] == [decode(a) for a in chunks]


def test_model_reaches_every_rule(model, inputs):
    """Every counter is non-zero at every level (lazy drops where the level has a lazy step)."""
    for level in LEVELS:
        cnt = {}
        for _, x in inputs:
            model.run(x, level, cnt)
        for k in COUNTERS:
            if k == "lazy_drops" and LAZY[level] == 0:
                assert cnt[k] == 0
                continue
            assert cnt[k] > 0, (level, k, cnt)


@pytest.mark.parametrize("level", LEVELS)
def test_trap_members_are_armed(model, level):
    """The traps parse as designed: lane p0 keeps its match although lane p0 + 1 has one at distance 1 that
    is one byte shorter (at levels 3.. the lazy rule would drop lane p0's match for a longer one)."""
    x, p0, L = trap_member(False)
    last = decode(model.run(x, level)[-1])[-3:]
    if level in (2, 3, 4):
        # two own ways (levels 2, 3) or a budget of three with good = 4 (level 4) reach the two most recent
        # 'aaaa' positions of the earlier run: 5 bytes from p0 - 99, then the last 'a' as a literal
        assert last[-2:] == [(5, 99), ord("a")], (level, last)
    else:
        assert last[-1] == (6, 100), (level, last)   # the earlier run's first 'a': all 6 bytes
    x, p0, L = trap_member(True)
    S = (p0 // SUB - 1) * SUB
    last = decode(model.run(x, level)[-1])[-3:]
    assert last[-1] == (5, p0 - (S - 1)), (level, last)   # the static entry S - 1 of the segment before S


# ---------------------------------------------------------------------- GPU: model against kernel
@pytest.mark.gpu
@pytest.mark.parametrize("level", LEVELS)
def test_kernel_tokens_equal_the_model(model, inputs, level):
    import zippy_b200 as z
    comp = z.compress_batch([x for _, x in inputs], level, z.dfDeflate)
    compared = stored = 0
    cnt = {}
    bad = []
    for (name, x), c in zip(inputs, comp):
        want = model.run(x, level, cnt)
        got = dt.member_chunks(dt.parse(c))
        assert len(got) == len(want), name
        for k, (g, w) in enumerate(zip(got, want)):
            if g.btype == 0:
                assert bytes(g.tokens) == x[k * CHUNK:(k + 1) * CHUNK], (name, k)
                stored += 1
                continue
            compared += 1
            ga = encode(g.tokens)
            if not np.array_equal(ga, w):
                i = int(np.argmax(ga[:min(len(ga), len(w))] != w[:min(len(ga), len(w))])) if len(ga) and len(w) else 0
                bad.append((name, k, i, decode(ga[max(0, i - 2):i + 3]), decode(w[max(0, i - 2):i + 3])))
    print("level %d: %d chunks compared, %d stored" % (level, compared, stored))
    assert not bad, bad[:10]
    assert compared >= 4 * stored and compared >= 60
    for k in COUNTERS:
        assert cnt[k] > 0 or (k == "lazy_drops" and LAZY[level] == 0), (k, cnt)
