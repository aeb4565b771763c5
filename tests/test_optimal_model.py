"""The optimal parse (k_opt, zb200_compress_batch_optimal) as a CPU model: tests/native/opt_model.c.

The model restates DESIGN.md's rules -- hash chains over the chunk and its history, the walk / keep limits, the
Pareto candidates, integer bit costs, two cost rounds, the shortest path per 8 KiB sub-chunk and its tie rule -- as
a sequential program.  These tests check the model on its own: its tokens rebuild the input and respect every
limit, a brute-force shortest path under the same costs and candidates reaches the same total cost, the inputs
reach every rule, and the members it stands for are smaller than level 9's (tests/native/lz2_model.c, which
tests/test_gpu_lz2_model.py pins to the kernel) on every corpus file.  tests/test_gpu_optimal.py compares the
kernel with it token by token.
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
CSRC = os.path.join(os.path.dirname(HERE), "zippy_b200", "csrc")
CHUNK, SUB = 65536, 8192
COUNTERS = ["matches", "history", "dist_max", "m258_at_end", "ties", "walk_cut", "keep_cut"]
CORPUS_FILES = ["alice29.txt", "asyoulik.txt", "lcet10.txt", "plrabn12.txt", "urls.10K", "html", "kppkn.gtb",
                "geo.protodata", "paper-100k.pdf"]
TEXT_FILES = ["alice29.txt", "asyoulik.txt", "lcet10.txt", "plrabn12.txt"]


class Model:
    def __init__(self, so):
        L = self.L = ctypes.CDLL(so)
        L.opt_model.restype = ctypes.c_int64
        L.opt_model.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p,
                                ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p]
        L.opt_model_chunk.restype = ctypes.c_uint64
        L.opt_model_chunk.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int, ctypes.c_uint64,
                                      ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.opt_block_bytes.restype = ctypes.c_uint32
        L.opt_block_bytes.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_int]
        assert L.opt_counter_count() == len(COUNTERS)
        self.keep = L.opt_param(1)

    def run(self, buf, hist0=0, window_bits=15, counters=None):
        """Tokens of the len(buf) - hist0 bytes after hist0 bytes of history: one array per chunk (literal b -> b,
        match -> length << 16 | distance)."""
        n = len(buf) - hist0
        nch = max(1, -(-n // CHUNK))
        tok = np.zeros(n + 16, dtype=np.uint32)
        per = np.zeros(nch, dtype=np.uint32)
        cnt = np.zeros(len(COUNTERS), dtype=np.uint64)
        got = self.L.opt_model(bytes(buf), hist0, n, window_bits, tok.ctypes.data, tok.size, per.ctypes.data,
                               cnt.ctypes.data)
        assert got >= 0
        if counters is not None:
            for k, v in zip(COUNTERS, cnt.tolist()):
                counters[k] = counters.get(k, 0) + v
        b = np.concatenate([[0], np.cumsum(per.astype(np.int64))])
        return [tok[b[i]:b[i + 1]] for i in range(nch)]

    def chunk_detail(self, buf, hist0, window_bits, k):
        """-> (literal/length costs, distance costs, candidates per chunk position, last round's path cost)."""
        n = len(buf) - hist0
        ln = min(CHUNK, n - k * CHUNK)
        ll = np.zeros(286, np.uint32)
        dd = np.zeros(30, np.uint32)
        cand = np.zeros(max(ln, 1) * self.keep, np.uint32)
        nc = np.zeros(max(ln, 1), np.uint8)
        total = self.L.opt_model_chunk(bytes(buf), hist0, n, window_bits, k, ll.ctypes.data, dd.ctypes.data,
                                       cand.ctypes.data, nc.ctypes.data)
        cands = [[(int(e) >> 16, int(e) & 0xffff) for e in cand[p * self.keep:p * self.keep + int(nc[p])]] for p in range(ln)]
        return ll.tolist(), dd.tolist(), cands, int(total)

    def member_bytes(self, chunks, n):
        """DEFLATE bytes of the member the library writes for these chunk tokens (k_huff's block choice)."""
        tot = 0
        for k, arr in enumerate(chunks):
            a = np.ascontiguousarray(arr, dtype=np.uint32)
            tot += self.L.opt_block_bytes(a.ctypes.data, len(a), min(CHUNK, n - CHUNK * k), int(k == len(chunks) - 1))
        return tot


def build_model(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("opt_model") / "libopt_model.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-I", CSRC, "-o", so,
                           os.path.join(HERE, "native", "opt_model.c")])
    return Model(so)


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return build_model(tmp_path_factory)


def decode(arr):
    return [t if t < 256 else (t >> 16, t & 0xffff) for t in arr.tolist()]


def encode(tokens):
    return np.array([t if isinstance(t, int) else t[0] << 16 | t[1] for t in tokens], dtype=np.uint32)


# ---------------------------------------------------------------------- inputs
def end_runs_member(rng):
    """Random bytes with runs of 'x' that end exactly at sub-chunk ends and at the chunk end (258-byte matches
    there), and a copy at exactly 2^9 / 2^12 / 2^15 back."""
    x = bytearray(rng.randbytes(2 * CHUNK))
    for b1 in (SUB, 3 * SUB, CHUNK, CHUNK + 5 * SUB):
        x[b1 - 700:b1] = b"x" * 700
    for lo, d in ((CHUNK + 20000, 512), (CHUNK + 30000, 4096), (CHUNK + 40000, 32768), (50000, 32768)):
        x[lo:lo + 400] = x[lo - d:lo - d + 400]
    return bytes(x)


def model_inputs(corpus):
    """(name, buffer, history bytes in front) triples: edge sizes, corpus slices at ragged lengths, multi-chunk
    text, runs at sub-chunk ends, copies at the window distances, and members that follow 1..32767 bytes of
    history."""
    rng = random.Random(0x0B7)
    T = util.text_corpus(corpus)
    urls, html = corpus["urls.10K"], corpus["html"]
    xs = [("empty", b"", 0), ("one", b"a", 0), ("zeros", bytes(CHUNK + 1), 0), ("zeros64k", bytes(CHUNK - 1), 0),
          ("abab", b"ab" * 5000, 0), ("kppkn", corpus["kppkn.gtb"][:CHUNK + 4000], 0)]
    for n in (4, 31, 33, 8191, 8193, 40000, 65535, 65536, 65537):
        o = rng.randrange(len(urls) - n)
        xs.append(("urls%d" % n, urls[o:o + n], 0))
    for n in (12345, 65537):
        o = rng.randrange(len(html) - n)
        xs.append(("html%d" % n, html[o:o + n], 0))
    xs.append(("text3chunks", T[1000:1000 + 3 * CHUNK - 999], 0))
    xs.append(("end_runs", end_runs_member(rng), 0))
    for h in (1, 77, 4096, 20000, 32767):
        o = rng.randrange(len(T) - 50000)
        xs.append(("hist%d" % h, T[o:o + h + 40000], h))
    return xs


@pytest.fixture(scope="module")
def inputs(corpus):
    return model_inputs(corpus)


# ---------------------------------------------------------------------- the model on its own
def check_tokens(buf, hist0, chunks, window_bits):
    """Lengths 4..258, distances 1..2^window_bits inside the member and its history, no match across a sub-chunk
    end, every chunk exactly its bytes, and the tokens rebuild the input."""
    n = len(buf) - hist0
    blocks = [dt.Block(0, False, 0, 0, list(buf[:hist0]))]
    for k, arr in enumerate(chunks):
        c0 = k * CHUNK
        a = arr.astype(np.int64)
        ism = a >= 256
        ln = np.where(ism, a >> 16, 1)
        d = a & 0xffff
        p = np.concatenate([[0], np.cumsum(ln)[:-1]]) if len(a) else a
        assert int(ln.sum()) == min(CHUNK, n - c0), k
        lm, dm, pm = ln[ism], d[ism], p[ism]
        assert ((lm >= 4) & (lm <= 258)).all() and ((dm >= 1) & (dm <= 1 << window_bits)).all(), k
        assert (dm <= hist0 + c0 + pm).all(), ("distance before the history", k)
        assert (pm // SUB == (pm + lm - 1) // SUB).all(), ("match across a sub-chunk end", k)
        blocks.append(dt.Block(2, False, 0, 0, decode(arr)))
    assert dt.rebuild(blocks) == bytes(buf)


@pytest.mark.parametrize("window_bits", [9, 12, 15])
def test_model_tokens_rebuild_the_input(model, inputs, window_bits):
    for name, buf, h in inputs:
        chunks = model.run(buf, h, window_bits)
        check_tokens(buf, h, chunks, window_bits)
        if h == 0 and name in ("zeros", "urls8193", "text3chunks", "end_runs", "one", "empty"):
            blocks = []
            for k, arr in enumerate(chunks):
                last = k == len(chunks) - 1
                blocks.append(dw.Fixed(decode(arr), final=last))
                if not last:
                    blocks.append(dw.Stored(b"", final=False))
            assert zlib.decompress(dw.raw(blocks), -window_bits) == buf, name


def brute_force_cost(buf, hist0, k, ll, dd, cands):
    """Least path cost of chunk k summed over its sub-chunks, by forward relaxation over every (length, distance)
    pair the candidates give (a length maps to the nearest candidate at least that long)."""
    n = len(buf) - hist0
    ln = min(CHUNK, n - k * CHUNK)
    base = hist0 + k * CHUNK

    def lcost(L):
        c = dt.LEN_BASE.index(max(b for b in dt.LEN_BASE if b <= L)) if L != 258 else 28
        return ll[257 + c] + dt.LEN_EXTRA[c]

    def dcost(d):
        c = max(i for i, b in enumerate(dt.DIST_BASE) if b <= d)
        return dd[c] + dt.DIST_EXTRA[c]

    total = 0
    for b0 in range(0, ln, SUB):
        b1 = min(b0 + SUB, ln)
        best = [None] * (b1 - b0 + 1)
        best[0] = 0
        for i in range(b1 - b0):
            if best[i] is None:
                continue
            p = b0 + i
            c = best[i] + ll[buf[base + p]]
            if best[i + 1] is None or c < best[i + 1]:
                best[i + 1] = c
            for L in range(4, 259):
                ds = [d for (m, d) in cands[p] if m >= L]
                if not ds:
                    break
                c = best[i] + lcost(L) + dcost(min(ds))
                if best[i + L] is None or c < best[i + L]:
                    best[i + L] = c
        total += best[b1 - b0]
    return total


def test_shortest_path_matches_brute_force(model):
    """On small random and structured inputs (with and without history, at windows 9 and 15) the model's path
    cost is the least one under its own costs and candidates."""
    rng = random.Random(0x5A7)
    cases = []
    for i in range(24):
        kind = i % 4
        if kind == 0:
            x = rng.randbytes(rng.randrange(1, 600))
        elif kind == 1:
            x = bytes(rng.choice(b"ab") for _ in range(rng.randrange(50, 900)))
        elif kind == 2:
            words = [rng.randbytes(rng.randrange(2, 9)) for _ in range(6)]
            x = b"".join(rng.choice(words) for _ in range(rng.randrange(20, 300)))
        else:
            x = b"z" * rng.randrange(200, 800) + rng.randbytes(30) + b"z" * rng.randrange(5, 400)
        h = rng.choice([0, 0, 13, 300])
        cases.append((rng.randbytes(h) + x if kind == 0 else (x[:h] if h <= len(x) else x) + x, h))
    cases.append((bytes(SUB + 700), 0))   # two sub-chunks
    for buf, h in cases:
        for wb in (9, 15):
            ll, dd, cands, total = model.chunk_detail(buf, h, wb, 0)
            assert brute_force_cost(buf, h, 0, ll, dd, cands) == total, (len(buf), h, wb)


def test_model_reaches_every_rule(model, inputs):
    """History matches, matches at distance 2^window_bits, 258-byte matches ending at a sub-chunk end (the chunk end
    included), cost ties, and walks cut by either limit, at every window size."""
    for wb in (9, 12, 15):
        cnt = {}
        for _, buf, h in inputs:
            model.run(buf, h, wb, cnt)
        for k in COUNTERS:
            assert cnt[k] > 0, (wb, k, cnt)


@pytest.fixture(scope="module")
def lz2(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lz2_for_sizes") / "liblz2.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "native", "lz2_model.c")])
    L = ctypes.CDLL(so)
    L.lz2_model.restype = ctypes.c_int64
    L.lz2_model.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint64,
                            ctypes.c_void_p, ctypes.c_void_p]
    return L


def level9_chunks(lz2, x):
    n = len(x)
    nch = max(1, -(-n // CHUNK))
    tok = np.zeros(n + 16, dtype=np.uint32)
    per = np.zeros(nch, dtype=np.uint32)
    cnt = np.zeros(16, dtype=np.uint64)
    assert lz2.lz2_model(x, n, 9, tok.ctypes.data, tok.size, per.ctypes.data, cnt.ctypes.data) >= 0
    b = np.concatenate([[0], np.cumsum(per.astype(np.int64))])
    return [tok[b[i]:b[i + 1]] for i in range(nch)]


def test_sizes_beat_level9_and_zlib9(model, lz2, corpus):
    """Every corpus file packs smaller than this library's level 9 member, and the text files together smaller
    than zlib -9 (raw DEFLATE bytes on both sides)."""
    opt_text = z9_text = 0
    for name in CORPUS_FILES:
        x = corpus[name]
        opt = model.member_bytes(model.run(x), len(x))
        l9 = model.member_bytes(level9_chunks(lz2, x), len(x))
        assert opt <= l9, (name, opt, l9)
        if name in TEXT_FILES:
            opt_text += opt
            z9_text += len(zlib.compress(x, 9)) - 6
    print("text: optimal %d, zlib -9 %d (%.4f)" % (opt_text, z9_text, opt_text / z9_text))
    assert opt_text <= z9_text
