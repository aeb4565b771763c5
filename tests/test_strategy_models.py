"""CPU models behind the compression strategies (include/zippy_b200.h "compression strategies"), no GPU needed.

- tests/native/rle_model.c, the run-length rule: without the chunk and piece cuts its tokens are zlib's Z_RLE tokens
  (Python zlib at levels 1 / 6 / 9 and memLevels 1 / 8 / 9, read back with deflate_tokens.parse); with the cuts no
  match crosses a 4 KiB piece end, no chunk's first byte is a match, and a piece holds at most 1024 matches -- the
  record capacity of a piece -- which worst_piece() reaches.
- zb_build_codebook (zb_huff.h) with force_type 1 (ZB200_STRATEGY_FIXED) never writes a dynamic block and picks
  the smaller of stored and fixed, ties to stored.
- tests/native/lz2_filtered_model.c (lz2_model.c's parse with a minimum match length) at minimum 6
  (ZB200_STRATEGY_FILTERED) emits no shorter match and still rebuilds its input; at minimum 4 it is lz2_model."""
import ctypes
import os
import random
import subprocess
import zlib

import numpy as np
import pytest

from tests import deflate_tokens as dt
from tests import util
from tests.test_gpu_huff_identity import HOST_UNITS, Host, block_bytes, gen_cases
from tests.test_gpu_lz2_model import decode

HERE = os.path.dirname(os.path.abspath(__file__))
RLE_SRC = os.path.join(HERE, "native", "rle_model.c")
LZ2_SRC = os.path.join(HERE, "native", "lz2_filtered_model.c")
CHUNK, PIECE = 65536, 4096


class Rle:
    def __init__(self, so):
        self.L = ctypes.CDLL(so)
        self.L.rle_model.restype = ctypes.c_int64
        self.L.rle_model.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint64,
                                     ctypes.c_void_p]

    def run(self, member, cuts):
        """-> (all tokens, one array per chunk) in lz2_model's encoding (literal b, match length << 16 | 1)."""
        n = len(member)
        nch = max(1, -(-n // CHUNK))
        tok = np.zeros(n + 16, dtype=np.uint32)
        per = np.zeros(nch, dtype=np.uint32)
        got = self.L.rle_model(bytes(member), n, 1 if cuts else 0, tok.ctypes.data, tok.size, per.ctypes.data)
        assert got >= 0
        tok = tok[:got]
        if not cuts:
            return tok, None
        bounds = np.concatenate([[0], np.cumsum(per.astype(np.int64))])
        assert bounds[-1] == got
        return tok, [tok[bounds[i]:bounds[i + 1]] for i in range(nch)]


@pytest.fixture(scope="module")
def rle(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("rle_model") / "librle_model.so")
    subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-o", so, RLE_SRC])
    return Rle(so)


# ---------------------------------------------------------------------- inputs (the GPU tests use them too)
def runs(rng, n, max_run, symbols):
    """n bytes of runs: each run 1..max_run long, its byte drawn from `symbols`."""
    out = bytearray()
    while len(out) < n:
        out += bytes([rng.choice(symbols)]) * rng.randint(1, max_run)
    return bytes(out[:n])


def sparse_fp16(seed, n_values, density=0.05):
    """A float16 tensor with `density` of its values non-zero, as bytes."""
    g = np.random.default_rng(seed)
    v = np.zeros(n_values, dtype=np.float16)
    k = int(n_values * density)
    v[g.choice(n_values, k, replace=False)] = g.standard_normal(k).astype(np.float16)
    return v.tobytes()


def worst_piece():
    """An 8 KiB member whose second piece holds 1024 matches: a run of 'a' continues 3 bytes into the piece (a match at
    its first byte), then 1023 runs of exactly four bytes (a literal and a 3-byte match each), then one byte."""
    body = bytearray(b"a" * 3)
    for i in range(1023):
        body += bytes([98 + (i & 1)]) * 4
    body += b"z"
    assert len(body) == PIECE
    return b"x" * (PIECE - 1) + b"a" + bytes(body)


def zlib_rle_blocks(data, level, mem_level):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, mem_level, zlib.Z_RLE)
    return dt.parse(c.compress(data) + c.flush())


def assert_zlib_rle(tokens, data, level, mem_level, name):
    """The model's tokens are zlib's, block by block.  A stored block lists its bytes, not the tokens zlib parsed
    them into, so there the model's tokens only have to cover the same bytes."""
    toks, i = decode(tokens), 0
    for b in zlib_rle_blocks(data, level, mem_level):
        if b.btype:
            assert toks[i:i + len(b.tokens)] == b.tokens, (name, level, mem_level)
            i += len(b.tokens)
            continue
        n = 0
        while n < len(b.tokens):
            n += 1 if isinstance(toks[i], int) else toks[i][0]
            i += 1
        assert n == len(b.tokens), (name, level, mem_level)
    assert i == len(toks), (name, level, mem_level)


def model_inputs():
    rng = random.Random(31)
    return {
        "empty": b"", "a": b"a", "aaaa": b"aaaa", "abbbb": b"abbbb", "ab3": b"abbb",
        "short_runs": runs(rng, 200000, 8, b"abcd"),
        "long_runs": runs(rng, 300000, 600, b"xyz"),
        "zeros": bytes(1 << 20),
        "sparse_fp16": sparse_fp16(5, 1 << 18),
        "worst": worst_piece(),
    }


# ---------------------------------------------------------------------- RLE rule
@pytest.mark.parametrize("level,mem_level", [(l, m) for l in (1, 6, 9) for m in (1, 8, 9)])
def test_rle_model_is_zlib_rle(rle, level, mem_level):
    """Without the cuts the rule's tokens are zlib's Z_RLE tokens, on seeded runs, zeros and sparse fp16."""
    for name, data in model_inputs().items():
        tok, _ = rle.run(data, cuts=False)
        assert_zlib_rle(tok, data, level, mem_level, name)


def test_rle_model_is_zlib_rle_on_fixtures(rle):
    """Without the cuts the rule's tokens are zlib's Z_RLE tokens on every decoded golden fixture (level 6, memLevel 8;
    the other level / memLevel pairs run on the seeded inputs above)."""
    for name, data in sorted(util.load_corpus().items()):
        data = data[:1 << 20]
        tok, _ = rle.run(data, cuts=False)
        assert_zlib_rle(tok, data, 6, 8, name)


def _positions(tokens):
    p = 0
    for t in decode(tokens):
        yield p, t
        p += 1 if isinstance(t, int) else t[0]


def test_rle_cuts(rle):
    """With the cuts: the chunks' tokens rebuild the member, no match crosses a piece end, no chunk's first byte is a
    match, every match has distance 1 and length 3..258, and a piece holds at most 1024 matches."""
    rng = random.Random(7)
    inputs = dict(model_inputs())
    inputs["mix"] = runs(rng, 150000, 300, b"ab") + rng.randbytes(70000) + bytes(140000)
    inputs["four_runs"] = runs(rng, 300000, 4, bytes(range(8)))
    for name, data in inputs.items():
        tok, chunks = rle.run(data, cuts=True)
        assert len(chunks) == max(1, -(-len(data) // CHUNK))
        blocks = [dt.Block(1, False, 0, 0, decode(c)) for c in chunks]
        assert dt.rebuild(blocks) == data, name
        for k, c in enumerate(chunks):
            assert sum(1 if t < 256 else t >> 16 for t in c.tolist()) == min(CHUNK, len(data) - k * CHUNK)
        per_piece = {}
        for p, t in _positions(tok):
            if isinstance(t, int):
                continue
            length, dist = t
            assert dist == 1 and 3 <= length <= 258, name
            assert p % CHUNK != 0, (name, p)
            assert p // PIECE == (p + length - 1) // PIECE, (name, p, length)
            per_piece[p // PIECE] = per_piece.get(p // PIECE, 0) + 1
        assert max(per_piece.values(), default=0) <= 1024, name


def test_rle_worst_piece_reaches_record_capacity(rle):
    """The worst case, 3 + 4 x 1023 bytes of matches in one piece, gives exactly 1024 matches, the record capacity
    of a piece (ZB_RECS_PER_SUB / 2); seeded searches around it never give more."""
    tok, _ = rle.run(worst_piece(), cuts=True)
    counts = {}
    for p, t in _positions(tok):
        if not isinstance(t, int):
            counts[p // PIECE] = counts.get(p // PIECE, 0) + 1
    assert counts.get(1) == 1024
    rng = random.Random(11)
    for _ in range(200):
        data = runs(rng, 3 * PIECE, rng.choice([3, 4, 5]), bytes(rng.sample(range(256), rng.randint(2, 4))))
        tok, _ = rle.run(data, cuts=True)
        counts = {}
        for p, t in _positions(tok):
            if not isinstance(t, int):
                counts[p // PIECE] = counts.get(p // PIECE, 0) + 1
        assert max(counts.values(), default=0) <= 1024


# ---------------------------------------------------------------------- FIXED block choice
@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("huff_host_fixed") / "libhost_units.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, HOST_UNITS])
    return Host(so)


def test_fixed_only_codebook(host):
    """force_type 1: never dynamic; stored when its bytes are at most the fixed block's, else fixed; and a fixed
    choice is the same codebook the free choice writes whenever that picked fixed too."""
    rng = np.random.default_rng(2024)
    seen = set()
    for name, h, ln, fin in gen_cases(rng):
        cb = np.frombuffer(host.build(h, ln, fin, 1), dtype=np.uint32)
        btype, total = int(cb[320]), int(cb[331])
        _, fix_bits = host.coded_bits(h)
        npieces = 1 if ln == 0 else -(-ln // 65535)
        stored = ln + 5 * npieces
        fixed = block_bytes(fix_bits, fin)
        assert btype in (0, 1), name
        assert (btype, total) == ((0, stored) if stored <= fixed else (1, fixed)), name
        seen.add(btype)
        free = host.build(h, ln, fin, -1)
        if np.frombuffer(free, dtype=np.uint32)[320] == btype:
            assert free == host.build(h, ln, fin, 1), name
    assert seen == {0, 1}


# ---------------------------------------------------------------------- FILTERED parse model
class Lz2Min:
    def __init__(self, so):
        self.L = ctypes.CDLL(so)
        self.L.lz2_model_min.restype = ctypes.c_int64
        self.L.lz2_model_min.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p,
                                         ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        self.L.lz2_model.restype = ctypes.c_int64
        self.L.lz2_model.argtypes = self.L.lz2_model_min.argtypes[:-1]
        self.ncnt = self.L.lz2_counter_count()

    def run(self, member, level, min_len=None):
        """-> one array of encoded tokens per chunk (lz2_model's encoding); min_len None: lz2_model itself."""
        n = len(member)
        nch = max(1, -(-n // CHUNK))
        tok = np.zeros(n + 16, dtype=np.uint32)
        per = np.zeros(nch, dtype=np.uint32)
        cnt = np.zeros(self.ncnt, dtype=np.uint64)
        args = (bytes(member), n, level, tok.ctypes.data, tok.size, per.ctypes.data, cnt.ctypes.data)
        got = self.L.lz2_model(*args) if min_len is None else self.L.lz2_model_min(*args, min_len)
        assert got >= 0
        bounds = np.concatenate([[0], np.cumsum(per.astype(np.int64))])
        return [tok[bounds[i]:bounds[i + 1]] for i in range(nch)]


@pytest.fixture(scope="module")
def lz2min(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lz2_model_min") / "liblz2_model.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, LZ2_SRC])
    return Lz2Min(so)


def filtered_inputs():
    rng = random.Random(5)
    corpus = util.load_corpus()
    words = [b"ab", b"abc", b"abcd", b"abcde", b"abcdef", b"xyz", b" the ", b"q"]
    return {
        "text": util.text_corpus(corpus)[:200000],
        "short_repeats": b"".join(rng.choice(words) for _ in range(40000)),
        "runs": runs(rng, 150000, 9, b"abc"),
        "random": rng.randbytes(70000),
    }


@pytest.mark.parametrize("level", [2, 3, 4, 5, 6, 7, 8, 9, -1])
def test_lz2_model_min6(lz2min, level):
    """Minimum length 6: no shorter match, the tokens rebuild the input, and the parse differs from minimum 4 on
    inputs with short repeats; minimum 4 is lz2_model itself."""
    differs = False
    for name, data in filtered_inputs().items():
        chunks6 = lz2min.run(data, level, 6)
        blocks = [dt.Block(1, False, 0, 0, decode(c)) for c in chunks6]
        assert dt.rebuild(blocks) == data, name
        for c in chunks6:
            m = c[c >= 256]
            assert (m >> 16).min(initial=6) >= 6, name
        chunks4 = lz2min.run(data, level, 4)
        assert all(np.array_equal(a, b) for a, b in zip(chunks4, lz2min.run(data, level))), name
        differs |= any(not np.array_equal(a, b) for a, b in zip(chunks4, chunks6))
    assert differs
