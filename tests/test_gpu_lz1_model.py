"""The level-1 parse (k_lz<1>), token by token, against a CPU model of its rules; and each chunk's block choice
against the host codebook builder.

tests/native/lz1_model.c restates the rules of DESIGN.md section 4 -- independent 64 KiB chunks, 4 KiB pieces
with a fresh table pre-seeded with what of the 2 KiB before them is staged, one probe per position, the lane cap,
the greedy chain of at most 8 matches per window and the exit match -- as a sequential program.  The one rule
the kernel's code does not fix is which lane lands when lanes of one store instruction write the same table
entry; the model takes it as a parameter.

The CPU tests check the model on its own: its tokens rebuild the member and respect the piece limits, round-trip
through zlib once packed with fixed codes, the inputs reach every rule (coverage counters), and each one-rule
mutant of the model (rule flags) parses the inputs differently -- so equality with the kernel excludes each
mutant.  tools/lz1_model.py's per-window statistics are checked against the model's.

The GPU tests compare with the model token by token both the library built with -DZB_LZ1_RESOLVE_WINNER=1 (the
highest position wins, by construction) and the shipped one (the hardware decides; on the H100 the lowest lane,
i.e. the lowest position, lands).  They check every chunk's block type, size and code lengths against
zb_build_codebook fed with the histograms of the model's tokens.
"""
import ctypes
import importlib.util
import os
import pickle
import random
import subprocess
import sys
import zlib

import numpy as np
import pytest

from tests import deflate_tokens as dt
from tests import deflate_writer as dw
from tests import util

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "native", "lz1_model.c")
HOST_UNITS = os.path.join(HERE, "native", "host_units.cpp")

CHUNK, PHASE, PIECE, SUB = 65536, 32768, 4096, 8192
COUNTERS = ["matches", "collisions", "preseed_hits", "preseed_short", "cap_ext", "m258", "limit_cut", "skipped",
            "win8", "contested_stores", "contested_reads",
            "windows", "entered", "verified", "ext_steps_lanes", "ext_steps_warp"]
FLAGS = {"preseed_2k": 1, "limit3": 2, "two_rounds": 4, "no_exit_ext": 8, "lowest": 16}
LOWEST = FLAGS["lowest"]
N_C2 = 300   # C2 blocks in the arbitration measurement


class Model:
    def __init__(self, so):
        self.L = ctypes.CDLL(so)
        self.L.lz1_model.restype = ctypes.c_int64
        self.L.lz1_model.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_int, ctypes.c_uint32, ctypes.c_void_p,
                                     ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p]
        assert self.L.lz1_counter_count() == len(COUNTERS)

    def run(self, member, mode=1, flags=0, counters=None):
        """-> one array of encoded tokens per chunk (literal b -> b, match -> length << 16 | distance)."""
        n = len(member)
        nch = max(1, -(-n // CHUNK))
        tok = np.zeros(n + 16, dtype=np.uint32)
        per = np.zeros(nch, dtype=np.uint32)
        cnt = np.zeros(len(COUNTERS), dtype=np.uint64)
        got = self.L.lz1_model(bytes(member), n, mode, flags, tok.ctypes.data, tok.size, per.ctypes.data,
                               cnt.ctypes.data)
        assert got >= 0
        if counters is not None:
            for k, v in zip(COUNTERS, cnt.tolist()):
                counters[k] = counters.get(k, 0) + v
        bounds = np.concatenate([[0], np.cumsum(per.astype(np.int64))])
        assert bounds[-1] == got
        return [tok[bounds[i]:bounds[i + 1]] for i in range(nch)]


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lz1_model") / "liblz1_model.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, SRC])
    return Model(so)


def encode(tokens):
    return np.array([t if isinstance(t, int) else t[0] << 16 | t[1] for t in tokens], dtype=np.uint32)


def decode(arr):
    return [t if t < 256 else (t >> 16, t & 0xffff) for t in arr.tolist()]


def preseed_start(b0):
    """First pre-seeded position of the piece at b0: 2 KiB before it, but in the second phase only what of the
    first is staged again (1 KiB)."""
    sbase = PHASE - 1024 if b0 >= PHASE else 0
    return b0 - min(2048, b0 - sbase)


def lz_hash(v):
    return ((v * 0x9E3779B1) & 0xffffffff) >> 21


# ---------------------------------------------------------------------- inputs
def _high(rng, n):
    """High-entropy bytes with the top bit set: 7 random bits per byte, so that a Huffman block beats a stored one
    and the chunk's tokens are written out, and no 4-gram repeats by chance."""
    return bytearray((np.frombuffer(rng.randbytes(n), dtype=np.uint8) | 0x80).tobytes())


def runs_member(rng, T):
    """Text with runs of 'x' across piece ends (lane-cap extensions, 258-byte matches, matches cut at the piece
    end while the run goes on), and 258-byte copies that end exactly at a piece end."""
    x = bytearray(T[:2 * CHUNK + 3000])
    for c in (3 * PIECE, 5 * PIECE + 7, PHASE, 9 * PIECE - 1, CHUNK + 2 * PIECE + 17):
        x[c - 700:c + 600] = b"x" * 1300
    for b1 in (6 * PIECE, 12 * PIECE, CHUNK + 4 * PIECE):
        x[b1 - 1200:b1 + 50] = _high(rng, 1250)
        src = b1 - 1000
        x[b1 - 258:b1] = x[src:src + 258]
    return bytes(x)


def preseed_member(rng):
    """One chunk of high-entropy bytes.  Bytes 32768 + k (k < 400) repeat the bytes 1536 earlier, before the 1 KiB
    that piece 8 has of the first phase; bytes 36864 + k repeat the bytes 1536 earlier, inside piece 9's 2 KiB
    pre-seed; bytes 33768 + k repeat the bytes 1500 earlier, inside piece 8's short pre-seed."""
    x = _high(rng, CHUNK)
    for at, d in ((PHASE, 1536), (9 * PIECE, 1536), (PHASE + 1000, 1500), (3 * PIECE + 100, 1800)):
        for k in range(400):
            x[at + k] = x[at + k - d]
    return bytes(x)


def eight_member(rng):
    """High-entropy bytes with windows made of eight 4-byte matches back to back: each 4-gram occurs once earlier
    just before the window, followed by a byte that does not continue the window."""
    x = _high(rng, 3 * PIECE)
    for wb in (PIECE + 1024, PIECE + 2048 + 64, 2 * PIECE + 512, 2 * PIECE + 1536):
        for i in range(8):
            s = wb - 48 + 5 * i
            x[s:s + 4] = x[wb + 4 * i:wb + 4 * i + 4]
            nxt = x[wb + 4 * i + 4]
            if x[s + 4] == nxt:
                x[s + 4] = 0x80 | ((nxt + 1) & 0x7f)
    return bytes(x)


def collision_member(rng):
    """Pairs of different 4-grams with the same 11-bit hash: one of each pair early in the piece, then both in one
    window (a candidate that fails the 4-byte check, and a contested store of different grams)."""
    x = _high(rng, 2 * PIECE)
    seen, pairs = {}, []
    while len(pairs) < 6:
        g = bytes(_high(rng, 4))
        h = lz_hash(int.from_bytes(g, "little"))
        if h in seen and seen[h] != g:
            pairs.append((seen.pop(h), g))
        else:
            seen[h] = g
    for i, (a, b) in enumerate(pairs):
        s = 256 + 64 * i
        x[s:s + 4] = a
        wb = 2048 + 64 * i
        x[wb + 3:wb + 7] = b
        x[wb + 20:wb + 24] = a
    return bytes(x)


def periodic_member(rng):
    """High-entropy bytes with stretches of period 5, 7, 12 and 20 that start on a window: the period's positions
    share table entries in one store instruction, and the next window reads them."""
    x = _high(rng, 4 * PIECE)
    for i, per in enumerate((5, 7, 12, 20, 7, 12)):
        wb = 512 + 1536 * i
        pat = bytes(_high(rng, per))
        x[wb:wb + 180] = (pat * (180 // per + 1))[:180]
    return bytes(x)


def model_inputs(corpus):
    """(name, member) pairs: C2 blocks, corpus slices whose lengths end around windows, pieces and phases, the
    hand-made members above, multi-chunk members with a stored chunk, tiny members and the empty member."""
    rng = random.Random(0x1A21)
    T = util.text_corpus(corpus)
    urls, html = corpus["urls.10K"], corpus["html"]
    xs = [("c2_%d" % i, util.c2_block(T, i)) for i in range(6)]
    for n in (31, 32, 33, 4095, 4096, 4097, 32767, 32768, 32769, 33791, 33792, 33793, 65537):
        o = rng.randrange(len(urls) - n)
        xs.append(("urls%d" % n, urls[o:o + n]))
        o = rng.randrange(len(html) - n)
        xs.append(("html%d" % n, html[o:o + n]))
    xs.append(("runs", runs_member(rng, T)))
    xs.append(("preseed", preseed_member(rng)))
    xs.append(("eight", eight_member(rng)))
    xs.append(("collisions", collision_member(rng)))
    xs.append(("periodic", periodic_member(rng)))
    o = rng.randrange(len(T) - 3 * CHUNK)
    xs.append(("text3chunks", T[o:o + 3 * CHUNK - 1234]))
    xs.append(("stored_middle", T[:CHUNK] + rng.randbytes(CHUNK) + T[CHUNK:CHUNK + 5000]))
    xs.append(("kppkn", corpus["kppkn.gtb"][:2 * CHUNK + 5]))
    for i, x in enumerate([b"", b"a", b"abcd", b"abcabcabcabc", b"hello, hello, hello world", b"a" * 300,
                           bytes(range(256)) * 3]):
        xs.append(("tiny%d" % i, x))
    return xs


# ---------------------------------------------------------------------- CPU: the model on its own
def _check_tokens(member, chunks):
    """Lengths 4..258, no match across a piece end, every source in its piece or the piece's pre-seed, every chunk
    exactly its bytes, and the tokens rebuild the member."""
    blocks = []
    for k, arr in enumerate(chunks):
        a = arr.astype(np.int64)
        ismatch = a >= 256
        ln = np.where(ismatch, a >> 16, 1)
        d = a & 0xffff
        p = np.concatenate([[0], np.cumsum(ln)[:-1]]) if len(a) else a
        assert int(ln.sum()) == min(CHUNK, len(member) - k * CHUNK), k
        lm, dm, pm = ln[ismatch], d[ismatch], p[ismatch]
        assert ((lm >= 4) & (lm <= 258)).all() and (dm >= 1).all(), k
        b0 = pm // PIECE * PIECE
        assert (b0 == (pm + lm - 1) // PIECE * PIECE).all(), ("match across a piece end", k)
        assert (pm - dm >= np.array([preseed_start(int(b)) for b in b0], dtype=np.int64)).all(), \
            ("source before the piece's pre-seed", k)
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


@pytest.mark.parametrize("mode", [1, 0])
def test_model_tokens_rebuild_the_member(model, inputs, mode):
    for name, x in inputs:
        chunks = model.run(x, mode)
        _check_tokens(x, chunks)
        if mode == 0:
            assert all((a < 256).all() for a in chunks), name
        raw = _fixed_stream(chunks)
        assert zlib.decompress(raw, -15) == x, name
        if not name.startswith(("c2", "urls", "html", "kppkn")):
            assert [list(c.tokens) for c in dt.member_chunks(dt.parse(raw))] == [decode(a) for a in chunks], name


def test_model_reaches_every_rule(model, inputs):
    cnt = {}
    for _, x in inputs:
        model.run(x, 1, 0, cnt)
    for k in COUNTERS:
        assert cnt[k] > 0, (k, cnt)


@pytest.mark.parametrize("flag", sorted(FLAGS))
def test_every_rule_flag_changes_the_parse(model, inputs, flag):
    """Each one-rule mutant of the model parses some input differently, so a kernel equal to the model on these
    inputs is not that mutant."""
    differ = [name for name, x in inputs
              if any(not np.array_equal(a, b) for a, b in zip(model.run(x), model.run(x, 1, FLAGS[flag])))]
    assert differ, flag


def test_statistics_script_agrees_with_the_model(model, corpus):
    """tools/lz1_model.py (an independent Python restatement) gives the model's per-window statistics."""
    spec = importlib.util.spec_from_file_location("lz1_model_tool", os.path.join(ROOT, "tools", "lz1_model.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    T = util.text_corpus(corpus)
    blocks = [util.c2_block(T, i) for i in range(3)]
    got = tool.window_stats(blocks)
    cnt = {}
    for b in blocks:
        model.run(b, 1, 0, cnt)
    want = {"windows": cnt["windows"], "entered": cnt["entered"], "verified": cnt["verified"],
            "ext_steps_warp": cnt["ext_steps_warp"], "ext_steps_lanes": cnt["ext_steps_lanes"],
            "chain": cnt["matches"], "cap": cnt["cap_ext"]}
    assert got == want


# ---------------------------------------------------------------------- the host codebook builder
class Codebook:
    """zb_build_codebook (zb_huff.h, the code k_huff runs) compiled for the CPU, as test_host_units.py does."""

    def __init__(self, so):
        L = ctypes.CDLL(so)
        self.L = L
        self.nbytes = L.t_codebook_size()
        self.lc = np.array([L.t_len_code(n) if n >= 3 else 0 for n in range(259)], dtype=np.int64)
        self.dc = np.array([L.t_dist_code(d) if d else 0 for d in range(32769)], dtype=np.int64)

    def histograms(self, arr):
        """8 x 316 u16: every token counted in the 8 KiB sub-chunk where it starts."""
        a = arr.astype(np.int64)
        ism = a >= 256
        ln = np.where(ism, a >> 16, 1)
        sub = (np.concatenate([[0], np.cumsum(ln)[:-1]]) if len(a) else a) // SUB
        h = np.zeros((8, 316), dtype=np.int64)
        np.add.at(h, (sub[~ism], a[~ism]), 1)
        np.add.at(h, (sub[ism], 257 + self.lc[ln[ism]]), 1)
        np.add.at(h, (sub[ism], 286 + self.dc[a[ism] & 0xffff]), 1)
        return np.ascontiguousarray(h.astype(np.uint16))

    def build(self, arr, chunk_len, is_final):
        """-> (block type, bytes in the stream, literal/length code lengths [286], distance code lengths [30])"""
        h = self.histograms(arr)
        cb = ctypes.create_string_buffer(self.nbytes)
        self.L.t_build_codebook(h.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), chunk_len, int(is_final), -1, cb)
        u32 = np.frombuffer(cb.raw[:4 * 334], dtype=np.uint32)
        return int(u32[320]), int(u32[331]), (u32[:286] >> 16).tolist(), (u32[288:318] >> 16).tolist()


@pytest.fixture(scope="module")
def codebook(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lz1_codebook") / "libhost_units.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, HOST_UNITS])
    return Codebook(so)


def _code_lengths(tab, n):
    """Code lengths of n symbols, read back from a deflate_tokens lookup table (every code fills an entry)."""
    lens = [0] * n
    for e in set(tab):
        if e:
            lens[e >> 4] = e & 15
    return lens


def chunk_layout(raw):
    """-> per chunk of a member's raw stream: (block type, bytes it occupies in the stream with its joint, and
    for a dynamic block the literal/length [286] and distance [30] code lengths of its header)."""
    blocks = dt.parse(raw)
    out, i = [], 0
    for c in dt.member_chunks(blocks):   # also checks the layout
        first = blocks[i]
        if c.btype == 0:
            n = 0
            while True:   # the stored blocks that hold the chunk's bytes
                n += len(blocks[i].tokens)
                i += 1
                if n == len(c.tokens):
                    break
        else:
            i += 1 if first.final else 2   # the block, and the empty stored block of the joint
        assert first.bit_start % 8 == 0, "a chunk starts on a byte boundary"
        lens = None
        if c.btype == 2:
            br = dt._Bits(raw)
            skip = first.bit_start + 3   # to the dynamic header, past BFINAL and BTYPE
            while skip:
                step = min(skip, 32)
                br.get(step)
                skip -= step
            lt, dtab = dt._dynamic_tables(br)
            lens = (_code_lengths(lt, 286), _code_lengths(dtab, 30))
        out.append((c.btype, (blocks[i - 1].bit_end + 7) // 8 - first.bit_start // 8, lens))
    return out


def check_block_choice(codebook, name, member, raw, want):
    """Every chunk of the raw stream `raw` has the block type and size zb_build_codebook gives for the histograms
    of its model tokens `want`, and a dynamic block has the builder's code lengths."""
    got = chunk_layout(raw)
    assert len(got) == len(want), name
    for k, ((gtype, gbytes, glens), w) in enumerate(zip(got, want)):
        n = min(CHUNK, len(member) - k * CHUNK)
        btype, nbytes, ll, dd = codebook.build(w, n, k == len(want) - 1)
        assert gtype == btype, (name, k, gtype, btype)
        assert gbytes == nbytes, (name, k, gbytes, nbytes)
        if btype == 2:
            assert glens[0] == ll, (name, k, "literal/length code lengths")
            assert glens[1] == dd, (name, k, "distance code lengths")


def test_block_choice_check_sees_the_builder(model, codebook, corpus):
    """The check above on a stream made from the builder's own choice: a fixed-code stream of the model's tokens
    is accepted only where the builder picks fixed codes, and its size is what the builder accounts."""
    for x in (b"", b"abc", b"hello, hello, hello world"):
        want = model.run(x)
        check_block_choice(codebook, "tiny", x, _fixed_stream(want), want)
    T = util.text_corpus(corpus)
    x = util.c2_block(T, 0)
    want = model.run(x)
    with pytest.raises(AssertionError):
        check_block_choice(codebook, "c2_0", x, _fixed_stream(want), want)   # text: the builder picks a dynamic block


def test_chunk_layout_reads_dynamic_headers(model, codebook, corpus):
    """chunk_layout reads back the code lengths a dynamic header was written with, and the chunks' byte counts add
    up to the stream."""
    T = util.text_corpus(corpus)
    x = util.c2_block(T, 0) + util.c2_block(T, 1)[:5000]
    want = model.run(x)
    blocks, lens = [], []
    for k, arr in enumerate(want):
        last = k == len(want) - 1
        _, _, ll, dd = codebook.build(arr, min(CHUNK, len(x) - k * CHUNK), last)
        lens.append((ll, dd))
        blocks.append(dw.Dynamic(decode(arr), ll_lens=dw._trim(ll, 257), d_lens=dw._trim(dd, 1), final=last))
        if not last:
            blocks.append(dw.Stored(b"", final=False))
    raw = dw.raw(blocks)
    got = chunk_layout(raw)
    assert [g[0] for g in got] == [2, 2]
    assert [g[2] for g in got] == lens
    assert sum(g[1] for g in got) == len(raw)


# ---------------------------------------------------------------------- GPU
VARIANT_LEVELS = [1, 0, -2, -1]
_VARIANT_SCRIPT = r"""
import pickle, sys
root, lib, path_in, path_out = sys.argv[1:5]
sys.path.insert(0, root)
from zippy_b200 import _native
_native.LIB_PATH = lib          # before the first load
import zippy_b200 as z
members, levels = pickle.load(open(path_in, "rb"))
out = {lv: z.compress_batch(members, lv, z.dfDeflate) for lv in levels}
assert _native.lib()._name == lib
pickle.dump(out, open(path_out, "wb"))
"""


@pytest.fixture(scope="module")
def c2_blocks(corpus):
    T = util.text_corpus(corpus)
    return [("c2_%d" % i, util.c2_block(T, i)) for i in range(6, 6 + N_C2)]


@pytest.fixture(scope="module")
def variant_out(inputs, c2_blocks, tmp_path_factory):
    """The inputs and C2 blocks compressed (raw DEFLATE) by the ZB_LZ1_RESOLVE_WINNER=1 build, in a subprocess:
    this process has the shipped library loaded already."""
    import __graft_entry__ as g
    assert os.path.exists(g.LIB_RW), ("%s is missing: build() in __graft_entry__.py compiles it next to the shipped "
                                      "library (python -c 'import __graft_entry__ as g; g.build()')" % g.LIB_RW)
    d = tmp_path_factory.mktemp("lz1_variant")
    members = [x for _, x in inputs + c2_blocks]
    with open(d / "in.pkl", "wb") as f:
        pickle.dump((members, VARIANT_LEVELS), f)
    flags = ["-I"] if sys.flags.isolated else ["-s"] if sys.flags.no_user_site else []   # as this process runs
    cmd = [sys.executable] + flags + \
        ["-c", _VARIANT_SCRIPT, ROOT, g.LIB_RW, str(d / "in.pkl"), str(d / "out.pkl")]
    subprocess.check_call(cmd, cwd=ROOT)
    with open(d / "out.pkl", "rb") as f:
        return pickle.load(f)


def compare_tokens(model, named, comp, flags=0, per_chunk=None):
    """Chunks of the kernel's streams against the model's tokens.  -> (compared, stored, mismatches); stored
    chunks have their bytes checked.  per_chunk(member, k, tokens) is called for every compared chunk."""
    compared = stored = 0
    bad = []
    for (name, x), c in zip(named, comp):
        want = model.run(x, 1, flags)
        got = dt.member_chunks(dt.parse(c))
        assert len(got) == len(want), name
        for k, (g, w) in enumerate(zip(got, want)):
            if g.btype == 0:
                assert bytes(g.tokens) == x[k * CHUNK:(k + 1) * CHUNK], (name, k)
                stored += 1
                continue
            compared += 1
            ga = encode(g.tokens)
            if per_chunk is not None:
                per_chunk(x, k, ga)
            if not np.array_equal(ga, w):
                n = min(len(ga), len(w))
                i = int(np.argmax(ga[:n] != w[:n])) if n and (ga[:n] != w[:n]).any() else n
                bad.append((name, k, i, decode(ga[max(0, i - 2):i + 3]), decode(w[max(0, i - 2):i + 3])))
    return compared, stored, bad


@pytest.mark.gpu
def test_variant_tokens_equal_the_model(model, inputs, c2_blocks, variant_out):
    """The ZB_LZ1_RESOLVE_WINNER=1 build (highest position wins) writes the model's tokens in every fixed or
    dynamic chunk."""
    named = inputs + c2_blocks
    cnt = {}
    for _, x in inputs:
        model.run(x, 1, 0, cnt)
    compared, stored, bad = compare_tokens(model, named, variant_out[1])
    print("level 1, highest position wins: %d chunks compared, %d stored" % (compared, stored))
    assert not bad, bad[:10]
    assert compared >= 4 * stored and compared >= N_C2
    for k in COUNTERS:
        assert cnt[k] > 0, (k, cnt)


@pytest.mark.gpu
def test_variant_changes_nothing_else(inputs, c2_blocks, variant_out):
    """The switch touches k_lz<1> only: at levels 0, -2 and Default both builds write the same bytes."""
    import zippy_b200 as z
    members = [x for _, x in inputs + c2_blocks]
    for level in (0, -2, -1):
        assert z.compress_batch(members, level, z.dfDeflate) == variant_out[level], level


@pytest.mark.gpu
def test_variant_block_choice_matches_the_codebook(model, codebook, inputs, c2_blocks, variant_out):
    """Every chunk's block type, size and code lengths are zb_build_codebook's for the histograms of the model's
    tokens: a token counted in the wrong sub-chunk, or not at all, changes a code or a size."""
    for (name, x), c in zip(inputs + c2_blocks, variant_out[1]):
        check_block_choice(codebook, name, x, c, model.run(x))


@pytest.mark.gpu
def test_literals_only_level(model, codebook, inputs):
    """Level -2: every non-stored chunk is all literals, and its block type, size and code lengths are the
    builder's for the literal histograms."""
    import zippy_b200 as z
    comp = z.compress_batch([x for _, x in inputs], z.HuffmanOnly, z.dfDeflate)
    huff = 0
    for (name, x), c in zip(inputs, comp):
        want = model.run(x, 0)
        got = dt.member_chunks(dt.parse(c))
        assert len(got) == len(want), name
        for k, (g, w) in enumerate(zip(got, want)):
            if g.btype:
                huff += 1
                assert all(isinstance(t, int) for t in g.tokens) and np.array_equal(encode(g.tokens), w), (name, k)
        check_block_choice(codebook, name, x, c, want)
    assert huff >= 40, huff



@pytest.fixture(scope="module")
def shipped_out(inputs, c2_blocks):
    import zippy_b200 as z
    return z.compress_batch([x for _, x in inputs + c2_blocks], z.BestSpeed, z.dfDeflate)


@pytest.mark.gpu
def test_shipped_build_lets_the_lowest_lane_land(model, inputs, c2_blocks, shipped_out):
    """The shipped build leaves same-entry stores of one instruction to the hardware.  On the H100 the lowest
    lane -- the lowest position -- lands: every chunk equals the model under that rule, also the chunks where a
    probe reads an entry whose last write was contested and the rules part ways."""
    contested = highest = 0

    def tally(x, k, got):
        nonlocal contested, highest
        cnt = {}
        (hi,) = model.run(x[k * CHUNK:(k + 1) * CHUNK], 1, 0, cnt)   # level 1 never refers across a chunk
        contested += cnt["contested_reads"] > 0
        highest += np.array_equal(got, hi)

    compared, stored, bad = compare_tokens(model, inputs + c2_blocks, shipped_out, LOWEST, tally)
    print("level 1, shipped build, lowest position wins: %d chunks compared, %d stored; %d with a contested read; "
          "%d equal to the model under 'highest' too" % (compared, stored, contested, highest))
    assert not bad, bad[:10]
    assert compared >= N_C2 and contested >= compared // 2 and highest < compared // 2


@pytest.mark.gpu
def test_shipped_block_choice_matches_the_codebook(model, codebook, inputs, c2_blocks, shipped_out):
    """test_variant_block_choice_matches_the_codebook for the shipped build, with the model under its rule."""
    for (name, x), c in zip(inputs + c2_blocks, shipped_out):
        check_block_choice(codebook, name, x, c, model.run(x, 1, LOWEST))
