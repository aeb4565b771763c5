"""Compression strategies on the GPU (include/zippy_b200.h "compression strategies"): the run-length parse
(k_lz<2>) against tests/native/rle_model.c, FIXED blocks against the host builder, HUFFMAN_ONLY as level -2, the
FILTERED parse (k_lz2<false, 6>) against tests/native/lz2_filtered_model.c, strategy 0 as the calls without one, and every
strategy x level x format decoded by zlib, the oracle and uncompress, deterministic and independent of batch
neighbours, source alignment, host or device input, and of a stream's write sizes."""
import ctypes
import hashlib
import os
import random
import subprocess
import sys
import zlib

import numpy as np
import pytest

import zippy_b200 as z
from tests import deflate_tokens as dt
from tests import util
from tests.test_gpu_huff_identity import CSRC, ROOT, WORDS, gen_cases
from tests.test_gpu_lz2_model import decode
from tests.test_strategy_models import (CHUNK, Lz2Min, Rle, LZ2_SRC, RLE_SRC, runs, sparse_fp16, worst_piece,
                                        host)  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

FORMATS = [z.dfGzip, z.dfZlib, z.dfDeflate]
STRATEGIES = [z.StrategyDefault, z.StrategyFiltered, z.StrategyHuffmanOnly, z.StrategyRle, z.StrategyFixed]
LEVELS = list(range(-2, 10))
WBITS = {z.dfGzip: 31, z.dfZlib: 15, z.dfDeflate: -15}


def batch(items, level, strategy, fmt, fname_lens=None, ctx=None, cap=None):
    """zb200_compress_batch_strategy -> (rc, [members], statuses)"""
    L = z._native.lib()
    base, offs = z._pack(items)
    n = len(items)
    bound = sum(L.zb200_compress_bound(len(x), fmt) for x in items)
    out = np.zeros((bound if cap is None else cap) + 8, dtype=np.uint8)
    oo = np.zeros(n + 1, dtype=np.uint64)
    st = np.full(max(n, 1), -7, dtype=np.int32)
    fl = np.ascontiguousarray(fname_lens if fname_lens is not None else [0] * n, dtype=np.uint8)
    ctx = ctx or z.default_context()
    rc = L.zb200_compress_batch_strategy(ctx._h, base.ctypes.data, offs.ctypes.data, n, level, strategy, fmt,
                                         fl.ctypes.data, out.ctypes.data, bound if cap is None else cap,
                                         oo.ctypes.data, st.ctypes.data)
    members = [out[int(oo[i]):int(oo[i + 1])].tobytes() for i in range(n)] if rc == 0 else None
    return rc, members, st


def members(items, level, strategy, fmt, **kw):
    rc, m, _ = batch(items, level, strategy, fmt, **kw)
    assert rc == 0, (level, strategy, fmt, rc)
    return m


@pytest.fixture(scope="module")
def inputs():
    rng = random.Random(17)
    T = util.text_corpus(util.load_corpus())
    out = [("text", T[:300001]), ("random", rng.randbytes(100000)), ("zeros", bytes(200000)),
           ("runs", runs(rng, 250000, 40, b"abc")), ("short_runs", runs(rng, 140000, 6, b"wxyz")),
           ("sparse_fp16", sparse_fp16(3, 100000)),
           ("mix", runs(rng, 70000, 300, b"ab") + rng.randbytes(5000) + T[:60000] + bytes(70000)),
           ("worst", worst_piece()), ("worst_x3", worst_piece() * 3)]
    for n in (0, 1, 2, 3, 4, 4095, 4096, 4097, 65535, 65536, 65537):
        out.append(("len%d" % n, (b"aaab" * (n // 4 + 1))[:n]))
    return out


@pytest.fixture(scope="module")
def rle(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("rle_model_gpu") / "librle_model.so")
    subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-o", so, RLE_SRC])
    return Rle(so)


@pytest.fixture(scope="module")
def lz2min(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lz2_model_min_gpu") / "liblz2_model.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, LZ2_SRC])
    return Lz2Min(so)


# ---------------------------------------------------------------------- strategy 0
@pytest.mark.parametrize("fmt", FORMATS)
def test_strategy0_is_the_existing_call(inputs, fmt):
    items = [x for _, x in inputs]
    fl = [i % 26 for i in range(len(items))]
    for level in LEVELS:
        base, offs = z._pack(items)
        out, oo = z.default_context().compress_batch(base, offs, level, fmt, fl)
        want = [out[int(oo[i]):int(oo[i + 1])].tobytes() for i in range(len(items))]
        assert members(items, level, z.StrategyDefault, fmt, fname_lens=fl) == want, level


# ---------------------------------------------------------------------- RLE
def test_rle_tokens_equal_the_model(inputs, rle):
    items = [x for _, x in inputs]
    ref = members(items, 1, z.StrategyRle, z.dfDeflate)
    coded = 0
    for (name, x), c in zip(inputs, ref):
        _, want = rle.run(x, cuts=True)
        got = dt.member_chunks(dt.parse(c))
        assert len(got) == len(want), name
        for k, (g, w) in enumerate(zip(got, want)):
            if g.btype == 0:
                assert bytes(g.tokens) == x[k * CHUNK:(k + 1) * CHUNK], (name, k)
                continue
            coded += 1
            assert g.tokens == decode(w), (name, k)
        assert zlib.decompress(c, -15) == x, name
    assert coded > 10
    # the worst piece (1024 matches) is coded, not stored
    worst = dict(zip([n for n, _ in inputs], ref))["worst"]
    assert dt.member_chunks(dt.parse(worst))[0].btype != 0


def test_rle_levels(inputs):
    items = [x for _, x in inputs]
    for fmt in FORMATS:
        one = members(items, 1, z.StrategyRle, fmt)
        for level in [-1] + list(range(2, 10)):
            assert members(items, level, z.StrategyRle, fmt) == one, (level, fmt)
        for level in (0, -2):
            assert members(items, level, z.StrategyRle, fmt) == members(items, level, z.StrategyDefault, fmt)


# ---------------------------------------------------------------------- FIXED
FIXED_LL = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 6


def fixed_bits(tokens):
    bits = 3 + 7   # header, end-of-block
    for t in tokens:
        if isinstance(t, int):
            bits += FIXED_LL[t]
            continue
        length, dist = t
        lc = max(i for i, b in enumerate(dt.LEN_BASE) if b <= length) if length < 258 else 28
        dc = max(i for i, b in enumerate(dt.DIST_BASE) if b <= dist)
        bits += FIXED_LL[257 + lc] + dt.LEN_EXTRA[lc] + 5 + dt.DIST_EXTRA[dc]
    return bits


@pytest.mark.parametrize("level", [1, -1, 4, 9, -2])
def test_fixed_blocks(inputs, level):
    """Every chunk is fixed or stored, whichever is smaller (ties: stored), and its tokens are DEFAULT's."""
    items = [x for _, x in inputs]
    fx = members(items, level, z.StrategyFixed, z.dfDeflate)
    df = members(items, level, z.StrategyDefault, z.dfDeflate)
    kinds = set()
    for (name, x), a, b in zip(inputs, fx, df):
        assert zlib.decompress(a, -15) == x
        ca, cb = dt.member_chunks(dt.parse(a)), dt.member_chunks(dt.parse(b))
        assert len(ca) == len(cb)
        for k, (ga, gb) in enumerate(zip(ca, cb)):
            assert ga.btype in (0, 1), (name, k)
            kinds.add(ga.btype)
            final = k == len(ca) - 1
            n = len(x[k * CHUNK:(k + 1) * CHUNK])
            stored = n + 5 * max(1, -(-n // 65535))
            if gb.btype != 0:   # DEFAULT coded the chunk: its tokens are the parse
                bits = fixed_bits(gb.tokens)
                fixed = (bits + 7) // 8 if final else (bits + 3 + 7) // 8 + 4
                assert ga.btype == (0 if stored <= fixed else 1), (name, k)
                if ga.btype == 1:
                    assert ga.tokens == gb.tokens, (name, k)
    assert kinds == {0, 1}


@pytest.fixture(scope="module")
def kernel_fixed(tmp_path_factory):
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    so = str(tmp_path_factory.mktemp("huff_warp_fixed") / "libhuff_warp_fixed.so")
    subprocess.check_call([os.environ.get("NVCC", "nvcc")] + g.NVCC_FLAGS +
                          ["-o", so, os.path.join(ROOT, "tests", "native", "huff_warp_strategy.cu")], cwd=CSRC)
    return ctypes.CDLL(so)


def test_k_huff_fixed_equals_host(host, kernel_fixed):  # noqa: F811
    """k_huff's fixed-only choice equals zb_build_codebook's force_type 1 bit for bit, on the histograms of
    test_gpu_huff_identity.py (at level 0 both write stored blocks)."""
    rng = np.random.default_rng(99)
    cases = gen_cases(rng)
    for level, force in ((1, 1), (0, 0)):
        h = np.ascontiguousarray(np.stack([c[1] for c in cases]), dtype=np.uint16)
        ln = np.ascontiguousarray([c[2] for c in cases], dtype=np.uint32)
        fi = np.ascontiguousarray([c[3] for c in cases], dtype=np.int32)
        out = np.zeros(len(cases) * 4 * WORDS, dtype=np.uint8)
        rc = kernel_fixed.t_huff_warp_fixed(h.ctypes.data_as(ctypes.c_void_p), ln.ctypes.data_as(ctypes.c_void_p),
                                            fi.ctypes.data_as(ctypes.c_void_p), len(cases), level,
                                            out.ctypes.data_as(ctypes.c_void_p))
        assert rc == 0
        for i, (name, hh, l_, f_) in enumerate(cases):
            assert out[i * 4 * WORDS:(i + 1) * 4 * WORDS].tobytes() == host.build(hh, l_, f_, force), (name, i)


# ---------------------------------------------------------------------- HUFFMAN_ONLY, FILTERED
def test_huffman_only_is_level_minus2(inputs):
    items = [x for _, x in inputs]
    for fmt in FORMATS:
        want = members(items, -2, z.StrategyDefault, fmt)
        for level in [-1, -2] + list(range(1, 10)):
            assert members(items, level, z.StrategyHuffmanOnly, fmt) == want, (level, fmt)


@pytest.mark.parametrize("level", [2, 3, 4, 5, 6, 7, 8, 9, -1])
def test_filtered_tokens_equal_the_model(inputs, lz2min, level):
    items = [x for _, x in inputs]
    got_all = members(items, level, z.StrategyFiltered, z.dfDeflate)
    compared = 0
    for (name, x), c in zip(inputs, got_all):
        want = lz2min.run(x, level, 6)
        got = dt.member_chunks(dt.parse(c))
        assert len(got) == len(want), name
        for k, (g, w) in enumerate(zip(got, want)):
            if g.btype == 0:
                assert bytes(g.tokens) == x[k * CHUNK:(k + 1) * CHUNK], (name, k)
                continue
            compared += 1
            assert g.tokens == decode(w), (name, level, k)
            assert all(isinstance(t, int) or t[0] >= 6 for t in g.tokens)
    assert compared > 10


def test_filtered_level1_is_level1(inputs):
    items = [x for _, x in inputs]
    for fmt in FORMATS:
        assert members(items, 1, z.StrategyFiltered, fmt) == members(items, 1, z.StrategyDefault, fmt)


# ---------------------------------------------------------------------- every strategy x level x format
@pytest.mark.parametrize("strategy", STRATEGIES[1:])
def test_decodes_and_is_deterministic(inputs, strategy):
    from oracle import oracle as o
    items = [x for _, x in inputs]
    ctx2 = z.Context()
    try:
        for fmt in FORMATS:
            for level in LEVELS:
                fl = [(i * 7) % 26 for i in range(len(items))]
                a = members(items, level, strategy, fmt, fname_lens=fl)
                assert members(items, level, strategy, fmt, fname_lens=fl) == a
                assert members(items, level, strategy, fmt, fname_lens=fl, ctx=ctx2) == a
                for i, (x, m) in enumerate(zip(items, a)):
                    assert zlib.decompress(m, WBITS[fmt]) == x, (level, fmt, i)
                back = z.uncompress_batch(a, fmt)
                assert back == items, (level, fmt)
                if level in (1, -1, 9):
                    for x, m in zip(items[:8], a[:8]):
                        if fmt != z.dfDeflate:
                            assert o.uncompress(m, fmt) == x
                # alone, a member is what it is in the batch
                for i in (0, 3, len(items) - 1):
                    assert members([items[i]], level, strategy, fmt, fname_lens=[fl[i]]) == [a[i]]
    finally:
        ctx2.close()


@pytest.mark.parametrize("strategy", STRATEGIES)
def test_device_input_alignment_and_tight_capacity(inputs, strategy):
    torch = pytest.importorskip("torch")
    items = [x for _, x in inputs if len(x) < 200000]
    L = z._native.lib()
    ctx = z.default_context()
    for fmt in FORMATS:
        for level in (1, -1, 6, -2, 0):
            want = members(items, level, strategy, fmt)
            for shift in (0, 5, 11):
                base, offs = z._pack(items)
                buf = np.zeros(base.size + 16, dtype=np.uint8)
                buf[shift:shift + base.size] = base
                d_src = torch.from_numpy(buf).cuda()
                cap = int(sum(L.zb200_compress_bound(len(x), fmt) for x in items))
                d_dst = torch.empty(cap + 64, dtype=torch.uint8, device="cuda")
                oo = ctx.compress_batch_device(d_src.data_ptr() + shift, offs, level, fmt, d_dst.data_ptr(), cap,
                                               fname_lens=[0] * len(items), strategy=strategy)
                got = d_dst[:int(oo[-1])].cpu().numpy().tobytes()
                assert [got[int(oo[i]):int(oo[i + 1])] for i in range(len(items))] == want, (level, fmt, shift)
            # exactly the bound of each member: every call fits
            for x in items[:12]:
                cap = int(L.zb200_compress_bound(len(x), fmt))
                rc, m, _ = batch([x], level, strategy, fmt, cap=cap)
                assert rc == 0 and len(m[0]) <= cap


# ---------------------------------------------------------------------- streams
@pytest.mark.parametrize("strategy", STRATEGIES[1:])
def test_stream_equals_batch(inputs, strategy):
    rng = random.Random(strategy)
    x = dict(inputs)["mix"] + dict(inputs)["text"][:150000]
    for fmt in FORMATS:
        for level in (1, -1, 4):
            want = members([x], level, strategy, fmt, fname_lens=[3])[0]
            s = z.CompressStream(level, fmt, fname_len=3, strategy=strategy)
            out, off = b"", 0
            while off < len(x):
                n = rng.choice([1, 100, 4096, 65536, 100000])
                out += s.write(x[off:off + n])
                off += n
            out += s.finish()
            s.close()
            assert out == want, (level, fmt)


def _stream(x, level, strategy, cuts, mode, fmt=z.dfDeflate):
    s = z.CompressStream(level, fmt, strategy=strategy)
    out, prev = [], 0
    for c in cuts + [len(x)]:
        out.append(s.write(x[prev:c]))
        if c < len(x):
            out.append(s.flush(mode))
        prev = c
    out.append(s.finish())
    s.close()
    return b"".join(out), [len(b"".join(out[:2 * i + 2])) for i in range(len(cuts))]


def test_rle_stream_flushes(inputs):
    x = dict(inputs)["mix"] + dict(inputs)["runs"]
    cuts = [1000, 70000, 70001, 200000]
    for level in (1, 6):
        a, _ = _stream(x, level, z.StrategyRle, cuts, z.SyncFlush)
        b, ends = _stream(x, level, z.StrategyRle, cuts, z.FullFlush)
        assert a == b
        assert zlib.decompress(a, -15) == x
        for cut, e in zip(cuts, ends):   # a raw inflater started right after a full flush decodes the rest
            d = zlib.decompressobj(-15)
            assert d.decompress(b[e:]) == x[cut:]


def test_filtered_stream_history(inputs):
    x = dict(inputs)["text"]
    cuts = [65536, 131072]
    for level in (-1, 6):
        a, _ = _stream(x, level, z.StrategyFiltered, cuts, z.SyncFlush)
        # sync flushes at chunk multiples keep the history: the batch call's bytes
        assert a == members([x], level, z.StrategyFiltered, z.dfDeflate)[0]
        b, ends = _stream(x, level, z.StrategyFiltered, cuts, z.FullFlush)
        assert b != a and zlib.decompress(b, -15) == x
        d = zlib.decompressobj(-15)
        assert d.decompress(b[ends[-1]:]) == x[cuts[-1]:]


# ---------------------------------------------------------------------- errors
def test_errors(inputs):
    items = [b"abc", b"aaaaaaaa"]
    L = z._native.lib()
    for bad in (-1, 5, 99):
        rc, _, st = batch(items, 1, bad, z.dfGzip)
        assert rc == 22 and (st == -7).all()
        with pytest.raises(z.ZippyError) as e:
            z.compress(b"abc", 1, z.dfZlib, strategy=bad)
        assert e.value.code == 22
        with pytest.raises(z.ZippyError):
            z.CompressStream(1, z.dfZlib, strategy=bad)
        h = ctypes.c_void_p()
        assert L.zb200_compress_stream_begin_strategy(z.default_context()._h, 1, bad, z.dfZlib, 0, ctypes.byref(h)) == 22
    rc, _, st = batch(items, 10, z.StrategyRle, z.dfGzip)
    assert rc == 1 and (st == -7).all()
    with pytest.raises(z.ZippyError):
        z.compress(b"abc", 1, z.dfZlib, dictionary=b"dict", strategy=z.StrategyRle)
    with pytest.raises(z.ZippyError):
        z.CompressStream(1, z.dfZlib, index_span=65536, strategy=z.StrategyFixed)
    assert z.deflate(b"a" * 1000, 1, z.StrategyRle) == members([b"a" * 1000], 1, z.StrategyRle, z.dfDeflate)[0]


# ---------------------------------------------------------------------- ratio
def test_rle_ratio():
    """Run-heavy inputs of 1 MiB and more: the RLE members (64 KiB chunks, no history across chunk starts) total at
    most 1.03 x zlib's Z_RLE at level 6 and less than zlib's level 1; zeros: less than zlib's level 1."""
    rng = random.Random(1)
    cases = {"short_runs": runs(rng, 1 << 20, 8, b"abcd"), "sparse_fp16": sparse_fp16(9, 1 << 19)}
    for name, x in cases.items():
        ours = len(z.compress(x, 1, z.dfDeflate, strategy=z.StrategyRle))
        c = zlib.compressobj(6, zlib.DEFLATED, -15, 8, zlib.Z_RLE)
        zrle = len(c.compress(x) + c.flush())
        c1 = zlib.compressobj(1, zlib.DEFLATED, -15)
        z1 = len(c1.compress(x) + c1.flush())
        assert ours <= 1.03 * zrle and ours < z1, (name, ours, zrle, z1)
    x = bytes(1 << 20)
    c1 = zlib.compressobj(1, zlib.DEFLATED, -15)
    assert len(z.compress(x, 1, z.dfDeflate, strategy=z.StrategyRle)) < len(c1.compress(x) + c1.flush())


# ---------------------------------------------------------------------- C++
def test_cpp_equals_python(tmp_path, inputs):
    exe = str(tmp_path / "cpp_strategy_test")
    libdir = os.path.join(ROOT, "zippy_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "native", "cpp_strategy_test.cpp"),
                           "-L" + libdir, "-l:libzippy_b200.so", "-Wl,-rpath," + libdir])
    data = dict(inputs)["mix"]
    inp = tmp_path / "in.bin"
    inp.write_bytes(data)
    for level, strategy, fmt in ((1, z.StrategyRle, z.dfZlib), (-1, z.StrategyFiltered, z.dfDeflate),
                                 (6, z.StrategyFixed, z.dfGzip), (3, z.StrategyHuffmanOnly, z.dfZlib)):
        o1, o2 = tmp_path / "m.bin", tmp_path / "s.bin"
        subprocess.check_call([exe, str(inp), str(level), str(strategy), str(fmt), "5", "30000", str(o1), str(o2)])
        if fmt != z.dfGzip:
            assert o1.read_bytes() == members([data], level, strategy, fmt)[0]
        s = z.CompressStream(level, fmt, fname_len=5, strategy=strategy)
        m = b""
        for off in range(0, len(data), 30000):
            m += s.write(data[off:off + 30000])
            if off == 0:
                m += s.flush()
        m += s.finish()
        s.close()
        assert o2.read_bytes() == m


# ---------------------------------------------------------------------- full size
def test_full_size_sparse_fp16_rle():
    """1 GiB of sparse fp16 as 16 384 x 64 KiB members at RLE, on the device, round-tripped through
    uncompress_batch_device; the same sha256 over two runs."""
    torch = pytest.importorskip("torch")
    n, size = 16384, 65536
    g = torch.Generator(device="cuda").manual_seed(5)
    v = torch.randn(n * size // 2, device="cuda", generator=g, dtype=torch.float32)
    keep = torch.rand(v.numel(), device="cuda", generator=g) < 0.05
    src = torch.where(keep, v, torch.zeros_like(v)).to(torch.float16).view(torch.uint8)
    del v, keep
    offs = np.arange(n + 1, dtype=np.uint64) * size
    L = z._native.lib()
    cap = int(L.zb200_compress_bound(size, z.dfGzip)) * n
    ctx = z.default_context()
    digests = []
    for _ in range(2):
        d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
        oo = ctx.compress_batch_device(src.data_ptr(), offs, 1, z.dfGzip, d_dst.data_ptr(), cap,
                                       strategy=z.StrategyRle)
        torch.cuda.synchronize()
        digests.append(hashlib.sha256(d_dst[:int(oo[-1])].cpu().numpy().tobytes()).hexdigest())
        assert int(oo[-1]) < n * size // 4
        back = torch.empty(n * size, dtype=torch.uint8, device="cuda")
        lens, st = ctx.uncompress_batch_device(d_dst.data_ptr(), oo, z.dfGzip, back.data_ptr(), offs)
        torch.cuda.synchronize()
        assert (st == 0).all() and (lens == size).all()
        assert torch.equal(back, src)
        del d_dst, back
    assert digests[0] == digests[1]
