"""Window sizes (include/zippy_b200.h "window size") in the CPU models of the parses, without a GPU.

tests/native/lz1_window_model.c (level 1) and lz2_window_model.c (levels -1 and 2..9, FILTERED's minimum 6 and a
flushed stream's chunk schedule) are the four parse models of lz1_model.c, lz2_model.c, lz2_filtered_model.c and
lz2_schedule_model.c with a distance limit, and count the selected matches at exactly that limit.  At 32768 they give
the tokens of those models.  At 2^n for n = 9..14 their tokens rebuild the member, no distance exceeds 2^n, matches at
exactly 2^n are selected (the edge counter), and the tokens, re-encoded, decode through Python's zlib with
wbits = -n in a loop with a small output limit, which makes zlib copy from its 2^n-byte window.  A hand-built stream
with one distance of 2^n + 1 fails in the same loop, so the loop does detect a violation.  Level 1's matches reach
at most 6 KiB back, so at n = 13 and 14 its tokens are those of n = 15."""
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
from tests.test_gpu_lz1_model import LOWEST
from tests.test_gpu_lz1_model import Model as Lz1Model
from tests.test_gpu_lz2_model import Model as Lz2Model
from tests.test_gpu_lz2_model import decode
from tests.test_gpu_stream_flush import ScheduleModel
from tests.test_strategy_models import Lz2Min

HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = os.path.join(HERE, "native")
CHUNK = 65536
WINDOWS = [9, 10, 11, 12, 13, 14]
LZ2_LEVELS = [2, 4, 6, 9, -1]


# ---------------------------------------------------------------------- shared with tests/test_gpu_window.py
def _high(rng, n):
    """High-entropy bytes with the top bit set: no 4-gram repeats by chance, so a stretch copied from d bytes back
    is the member's only repeat at that place."""
    return bytearray((np.frombuffer(rng.randbytes(n), dtype=np.uint8) | 0x80).tobytes())


def edge_member(n, seed=0x3D):
    """Random bytes over two chunks and a bit, whose only repeats are 200-byte stretches copied from exactly 2^n and
    2^n + 1 bytes back: inside chunk 0 (in one 4 KiB piece, so that level 1 can reach 2^n <= 4096) and across each
    64 KiB chunk joint (the source in the chunk before, history for levels -1 and 2..9)."""
    d = 1 << n
    rng = random.Random(seed + n)
    x = _high(rng, 2 * CHUNK + 9000)
    for p, dist in ((20000, d), (20250, d + 1), (CHUNK + 100, d), (CHUNK + 400, d + 1),
                    (2 * CHUNK + 50, d), (2 * CHUNK + 2600, d + 1)):
        for i in range(p, p + 200):
            x[i] = x[i - dist]
    return bytes(x)


def inflate_small(stream, wbits, step=1):
    """Decode through zlib with at most `step` output bytes per call: every match is copied from zlib's window of
    2^|wbits| bytes (with step 1 exactly: a distance beyond the window fails with "invalid distance too far
    back")."""
    d = zlib.decompressobj(wbits)
    out = [d.decompress(stream, step)]
    while d.unconsumed_tail:
        out.append(d.decompress(d.unconsumed_tail, step))
    out.append(d.flush())
    assert d.eof
    return b"".join(out)


def zlib_header(n):
    """CMF FLG of a zlib member with window 2^n (8 means 9), FLEVEL 0 and no FDICT."""
    cmf = (max(n, 9) - 8) << 4 | 8
    return bytes([cmf, (31 - (cmf << 8) % 31) % 31])


def max_distance(chunks):
    return max([t[1] for c in chunks for t in c if not isinstance(t, int)] or [0])


# ---------------------------------------------------------------------- models
class Windowed:
    """One parse of tests/native/lz1_window_model.c or lz2_window_model.c (kind "lz1", "lz2", "lz2f": FILTERED's
    minimum 6, "lz2s": a flushed stream's schedule), and the same parse through the existing model entry point
    (lz1_model, lz2_model, lz2_model_min, lz2_model_schedule), which has no window."""

    def __init__(self, kind, win_so, ref_so):
        self.kind = kind
        self.L = ctypes.CDLL(win_so)
        P, U64, U32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
        if kind == "lz1":
            self.f = self.L.lz1_window_model
            self.f.argtypes = [ctypes.c_char_p, U64, U32, U32, P, U64, P, P, P]
            self.ref_model = Lz1Model(ref_so)
        else:
            self.f = self.L.lz2_window_model
            self.f.argtypes = [ctypes.c_char_p, U64, ctypes.c_int, ctypes.c_int, U32, P, P, U64, P, U64, P, P, P]
            self.ref_model = {"lz2": Lz2Model, "lz2f": Lz2Min, "lz2s": ScheduleModel}[kind](ref_so)
        self.f.restype = ctypes.c_int64

    def run(self, x, level, d):
        """-> (one array of encoded tokens per chunk, selected matches at exactly distance d)"""
        n = len(x)
        tok = np.zeros(n + 16, dtype=np.uint32)
        cnt = np.zeros(32, dtype=np.uint64)
        edge = ctypes.c_uint64(0)
        if self.kind == "lz1":
            nch = max(1, -(-n // CHUNK))
            per = np.zeros(nch, dtype=np.uint32)
            got = self.f(bytes(x), n, LOWEST, d, tok.ctypes.data, tok.size, per.ctypes.data, cnt.ctypes.data,
                         ctypes.byref(edge))
        else:
            b = h = None
            nch = max(1, -(-n // CHUNK))
            if self.kind == "lz2s":
                bounds, hist_from = schedule(n)
                b, h = np.array(bounds, dtype=np.uint64), np.array(hist_from, dtype=np.uint64)
                nch = len(hist_from)
            per = np.zeros(nch, dtype=np.uint32)
            got = self.f(bytes(x), n, level, 6 if self.kind == "lz2f" else 4, d,
                         b.ctypes.data if b is not None else None, h.ctypes.data if h is not None else None, nch,
                         tok.ctypes.data, tok.size, per.ctypes.data, cnt.ctypes.data, ctypes.byref(edge))
        assert got >= 0, got
        edges = np.concatenate([[0], np.cumsum(per.astype(np.int64))])
        assert edges[-1] == got
        return [tok[edges[i]:edges[i + 1]] for i in range(nch)], edge.value

    def ref(self, x, level):
        m = self.ref_model
        if self.kind == "lz1":
            return m.run(x, 1, LOWEST)
        if self.kind == "lz2s":
            return m.run_schedule(x, level, *schedule(len(x)))
        if self.kind == "lz2f":
            return m.run(x, level, 6)
        return m.run(x, level)


WIN_SRC = {"lz1": "lz1_window_model.c", "lz2": "lz2_window_model.c", "lz2f": "lz2_window_model.c",
           "lz2s": "lz2_window_model.c"}
REF_SRC = {"lz1": "lz1_model.c", "lz2": "lz2_model.c", "lz2f": "lz2_filtered_model.c",
           "lz2s": "lz2_schedule_model.c"}


def _so(tmp_path_factory, src):
    so = str(tmp_path_factory.mktemp(src[:-2]) / ("lib%s.so" % src[:-2]))
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(NATIVE, src)])
    return so


def _windowed(tmp_path_factory, kind):
    return Windowed(kind, _so(tmp_path_factory, WIN_SRC[kind]), _so(tmp_path_factory, REF_SRC[kind]))


@pytest.fixture(scope="module")
def lz1(tmp_path_factory):
    return _windowed(tmp_path_factory, "lz1")


@pytest.fixture(scope="module")
def lz2(tmp_path_factory):
    return _windowed(tmp_path_factory, "lz2")


@pytest.fixture(scope="module")
def lz2f(tmp_path_factory):
    return _windowed(tmp_path_factory, "lz2f")


@pytest.fixture(scope="module")
def lz2s(tmp_path_factory):
    return _windowed(tmp_path_factory, "lz2s")


def schedule(n):
    """A flushed stream's chunks: cuts at 20000 (sync flush), 50000 (full flush: no history before it) and every
    64 KiB after each flush."""
    bounds, hist_from = [0], []
    for lo, hi, h in ((0, 20000, 0), (20000, 50000, 0), (50000, n, 50000)):
        for b in range(lo, hi, CHUNK):
            hist_from.append(h)
            bounds.append(min(hi, b + CHUNK))
    return bounds, hist_from


def runs(w, x, level, d):
    """-> the chunks' tokens of the parse `w` at distance limit d."""
    return w.run(x, level, d)[0]


@pytest.fixture(scope="module")
def members(corpus):
    T = util.text_corpus(corpus)
    rng = random.Random(0x5EED)
    xs = [("alice", corpus["alice29.txt"][:150000]), ("urls", corpus["urls.10K"][:140000]),
          ("html_x_4", corpus["html_x_4"][:140000]), ("kppkn", corpus["kppkn.gtb"][:140000]),
          ("text", T[300000:300000 + 3 * CHUNK + 1234]), ("random", rng.randbytes(70000))]
    return xs


@pytest.mark.parametrize("name", ["lz1", "lz2", "lz2f", "lz2s"])
def test_32768_is_the_existing_model(request, members, name):
    """At 32768 each windowed parse gives the tokens of the existing model entry point, which has no window."""
    w = request.getfixturevalue(name)
    for level in [1] if name == "lz1" else LZ2_LEVELS:
        for mname, x in members + [("edge", edge_member(12))]:
            got, want = runs(w, x, level, 32768), w.ref(x, level)
            assert len(got) == len(want) and all(np.array_equal(a, b) for a, b in zip(got, want)), \
                (name, level, mname)


def _check(x, chunks, n):
    """The tokens rebuild x, every distance is at most 2^n and reaches no byte before the member, and the stream
    decodes through zlib at wbits -n with one output byte per call."""
    blocks = [dt.Block(2, False, 0, 0, decode(c)) for c in chunks]
    assert dt.rebuild(blocks) == x
    assert max_distance([decode(c) for c in chunks]) <= 1 << n
    parts = []
    for k, c in enumerate(chunks):
        parts.append(dw.Fixed(decode(c), final=k == len(chunks) - 1))
        if k != len(chunks) - 1:
            parts.append(dw.Stored(b"", final=False))
    assert inflate_small(dw.raw(parts), -n) == x


@pytest.mark.parametrize("n", WINDOWS)
@pytest.mark.parametrize("name", ["lz1", "lz2", "lz2f", "lz2s"])
def test_windowed_tokens(request, members, name, n):
    w = request.getfixturevalue(name)
    edge = 0
    for level in [1] if name == "lz1" else LZ2_LEVELS:
        for mname, x in members + [("edge", edge_member(n))]:
            chunks, e = w.run(x, level, 1 << n)
            edge += e
            if mname == "edge" or level in (1, 6):   # the zlib loop costs a Python call per byte: one level
                _check(x, chunks, n)
            else:
                assert max_distance([decode(c) for c in chunks]) <= 1 << n
    if name == "lz1" and n >= 13:
        assert edge == 0   # level 1 reaches at most 6 KiB back
    else:
        assert edge > 0, (name, n)


@pytest.mark.parametrize("n", [13, 14])
def test_level1_window_13_and_14_are_window_15(lz1, members, n):
    for mname, x in members + [("edge", edge_member(n))]:
        a = runs(lz1, x, 1, 1 << n)
        b = runs(lz1, x, 1, 32768)
        assert all(np.array_equal(p, q) for p, q in zip(a, b)), mname


def test_small_windows_change_the_parse(lz2, members):
    """The limit is live: at every n < 15 some member parses differently at level 6 than at 32768."""
    for n in WINDOWS:
        differ = 0
        for _, x in members:
            a = runs(lz2, x, 6, 1 << n)
            b = runs(lz2, x, 6, 32768)
            differ += not all(np.array_equal(p, q) for p, q in zip(a, b))
        assert differ, n


@pytest.mark.parametrize("n", [9, 12, 14])
def test_harness_detects_a_distance_beyond_the_window(n):
    """A hand-built stream whose only match is 2^n back decodes at wbits -n; the same stream with the match
    2^n + 1 back fails, and decodes at wbits -(n + 1)."""
    rng = random.Random(n)
    d = 1 << n
    for dist, ok in ((d, True), (d + 1, False)):
        x = bytes(_high(rng, dist + 100))
        toks = list(x) + [(50, dist)]
        stream = dw.raw([dw.Fixed(toks, final=True)])
        want = x + x[len(x) - dist:len(x) - dist + 50]
        if ok:
            assert inflate_small(stream, -n) == want
        else:
            with pytest.raises(zlib.error, match="too far back"):
                inflate_small(stream, -n)
            assert inflate_small(stream, -(n + 1)) == want


def test_zlib_header_bytes():
    """The header the zlib format writes for n = 8..15 (8 means 9) is zlib's own for level 1 (FLEVEL 0)."""
    want = "1819 1819 2815 3811 480d 5809 6805 7801".split()
    for n, h in zip(range(8, 16), want):
        c = zlib.compressobj(1, zlib.DEFLATED, n)
        assert (c.compress(b"") + c.flush())[:2].hex() == h == zlib_header(n).hex(), n
