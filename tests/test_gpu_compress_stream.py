"""Streaming compression (zb200_compress_stream_*, CompressStream): whatever the sizes of the writes, the
concatenated output is the member compress_batch writes for the whole input, byte for byte.

Contexts with a small batching threshold (ZB200_STREAM_BATCH_BYTES) make a stream launch at nearly every chunk,
so the LZ history, the header flag and the running CRC-32 / Adler-32 / byte count cross many calls."""
import os
import random
import subprocess
import zlib

import numpy as np
import pytest

from tests import util
from tests.test_gpu_lz2_model import trap_member

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CHUNK = 65536
LEVELS = [-2, 0, 1, -1] + list(range(2, 10))
FORMATS = ("gzip", "zlib", "deflate")
WBITS = {"gzip": 31, "zlib": 15, "deflate": -15}


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


def _df(z, fmt):
    return {"gzip": z.dfGzip, "zlib": z.dfZlib, "deflate": z.dfDeflate}[fmt]


@pytest.fixture(scope="module")
def contexts(z):
    """'every': a launch whenever more than one chunk is pending; 'three': launches of about three chunks."""
    mp = pytest.MonkeyPatch()
    ctxs = {}
    try:
        for name, v in (("every", "1"), ("three", str(3 * CHUNK + 5))):
            mp.setenv("ZB200_STREAM_BATCH_BYTES", v)
            ctxs[name] = z.Context()
    finally:
        mp.undo()
    yield ctxs
    for c in ctxs.values():
        c.close()


def _trap(T):
    """A lazy-match trap (test_gpu_lz2_model.trap_member) inside chunk 0, followed by more 'a's and text: the
    writes are cut inside the run of 'a's whose best match the lazy rule weighs."""
    x, p0, L = trap_member(False)
    pre = T[:20000]
    data = pre + x + b"a" * 300 + T[20000:200000]
    cut = len(pre) + p0
    return data, [cut + 2, cut + L + 1]


@pytest.fixture(scope="module")
def inputs(corpus):
    rng = random.Random(0x57)
    T = util.text_corpus(corpus)
    o = rng.randrange(len(T) - 400000)
    text = T[o:o + 300001]
    rnd = rng.randbytes(200003)
    mix = text[:100000] + rng.randbytes(70000) + bytes(90000) + text[100000:170000]
    trap, trap_cuts = _trap(T)
    return {"text": (text, []), "random": (rnd, []), "zeros": (bytes(196608), []), "mix": (mix, []),
            "trap": (trap, trap_cuts)}


def _splits(n, pattern, extra_cuts, seed):
    """Write boundaries for an input of n bytes -> list of (lo, hi) pieces (empty pieces included)."""
    if pattern == "one":
        cuts = [0, n]
    elif pattern in (65535, 65536, 65537):
        cuts = list(range(0, n, pattern)) + [n]
    elif pattern == "random":
        rng = random.Random(seed)
        cuts = sorted({0, n, *extra_cuts, *(rng.randrange(n + 1) for _ in range(12))})
    elif pattern == "empty_between":
        cuts = [0] + [c for c in range(40000, n, 40000) for _ in (0, 1)] + [n, n]   # every piece twice: the
    else:                                                                              # second is empty
        raise ValueError(pattern)
    if pattern != "random":
        cuts = sorted(cuts + [c for c in extra_cuts if c not in cuts])
    return list(zip(cuts[:-1], cuts[1:]))


def _stream(z, ctx, data, level, df, fname_len, pieces):
    out = []
    with z.CompressStream(level, df, fname_len, ctx) as s:
        for lo, hi in pieces:
            out.append(s.write(data[lo:hi]))
        out.append(s.finish())
    return b"".join(out)


def _one_shot(z, ctx, data, level, df, fname_len):
    base, offs = z._pack([data])
    out, oo = ctx.compress_batch(base, offs, level, df, [fname_len])
    return out[:int(oo[1])].tobytes()


def _check_inflates(z, fmt, comp, data):
    from oracle import oracle as o
    assert zlib.decompress(comp, WBITS[fmt]) == data
    assert o.uncompress(comp, {"gzip": o.dfGzip, "zlib": o.dfZlib, "deflate": o.dfDeflate}[fmt]) == data
    assert z.uncompress(comp, _df(z, fmt)) == data


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("level", LEVELS)
def test_stream_equals_one_shot(z, contexts, inputs, level, fmt):
    df = _df(z, fmt)
    bad = []
    for k, (name, (data, cuts)) in enumerate(sorted(inputs.items())):
        fl = (7 * k + level + 2) % 26
        ref = _one_shot(z, z.default_context(), data, level, df, fl)
        _check_inflates(z, fmt, ref, data)
        for pattern in ("one", 65535, 65536, 65537, "random", "empty_between"):
            for cname in (("every", "three") if pattern == "random" else ("every",)):
                got = _stream(z, contexts[cname], data, level, df, fl, _splits(len(data), pattern, cuts, k))
                if got != ref:
                    bad.append((name, pattern, cname))
    # 1-byte writes across a chunk joint, and nothing but finish
    data = inputs["text"][0][:CHUNK + 3000]
    got = _stream(z, contexts["every"], data, level, df, 3, [(i, i + 1) for i in range(len(data))])
    if got != _one_shot(z, z.default_context(), data, level, df, 3):
        bad.append(("text", "bytes", "every"))
    for cname in ("every", "three"):
        got = _stream(z, contexts[cname], b"", level, df, 5, [])
        if got != _one_shot(z, z.default_context(), b"", level, df, 5):
            bad.append(("empty", "finish_only", cname))
    assert not bad, bad


@pytest.mark.gpu
def test_small_writes_launch_nothing(z, corpus):
    """Below the threshold (the built-in 64 MiB) a write only buffers: no kernel runs, nothing is emitted."""
    ctx = z.Context()
    T = util.text_corpus(corpus)
    data = (T * (10 * (1 << 20) // len(T) + 1))[:10 << 20]
    out = []
    with z.CompressStream(z.BestSpeed, z.dfGzip, 4, ctx) as s:
        for i in range(0, len(data), 1 << 20):
            assert s.write(data[i:i + (1 << 20)]) == b""
            assert ctx.timing()["kernel_launches"] == 0
        out.append(s.finish())
        assert ctx.timing()["kernel_launches"] == 5
    assert b"".join(out) == _one_shot(z, ctx, data, z.BestSpeed, z.dfGzip, 4)
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, -1])
def test_interleaved_streams(z, contexts, inputs, level):
    """Two streams on one ctx, with batch calls between their writes, write what each writes alone."""
    ctx = contexts["every"]
    a, b = inputs["text"][0], inputs["mix"][0]
    alone = [_stream(z, ctx, a, level, z.dfGzip, 9, _splits(len(a), 65537, [], 0)),
             _stream(z, ctx, b, level, z.dfZlib, 0, _splits(len(b), 65537, [], 0))]
    s1, s2 = z.CompressStream(level, z.dfGzip, 9, ctx), z.CompressStream(level, z.dfZlib, 0, ctx)
    o1, o2 = [], []
    items = [inputs["zeros"][0], inputs["random"][0][:1000]]
    comp = z._pack([z.compress(x) for x in items])
    for i in range(0, max(len(a), len(b)), 65537):
        o1.append(s1.write(a[i:i + 65537]))
        base, offs = z._pack(items)
        ctx.compress_batch(base, offs, 6, z.dfGzip)
        o2.append(s2.write(b[i:i + 65537]))
        out, do, lens, st = ctx.uncompress_batch(*comp)
        assert list(st) == [0, 0]
    o2.append(s2.finish())
    o1.append(s1.finish())
    s1.close()
    s2.close()
    assert [b"".join(o1), b"".join(o2)] == alone


@pytest.mark.gpu
def test_error_contract(z, contexts, inputs):
    import ctypes
    from zippy_b200 import _native
    L = _native.lib()
    ctx = contexts["every"]
    for args, code in (((10, z.dfGzip, 0), 1), ((-3, z.dfGzip, 0), 1), ((1, z.dfDetect, 0), 2), ((1, 4, 0), 2),
                       ((1, z.dfGzip, 26), 22), ((1, z.dfZlib, -1), 22)):
        with pytest.raises(z.ZippyError) as e:
            z.CompressStream(*args, ctx=ctx)
        assert e.value.code == code, args
    # write / finish after finish
    s = z.CompressStream(1, z.dfZlib, 0, ctx)
    s.write(b"abc")
    s.finish()
    for call in (lambda: s.write(b"x"), s.finish):
        with pytest.raises(z.ZippyError) as e:
            call()
        assert e.value.code == 22
    s.close()
    # a destination too small consumes nothing; the retry with bound() bytes gives the one-shot bytes
    data = inputs["text"][0]
    ref = _one_shot(z, ctx, data, -1, z.dfGzip, 11)
    h = ctypes.c_void_p()
    assert L.zb200_compress_stream_begin(ctx._h, -1, z.dfGzip, 11, ctypes.byref(h)) == 0
    src = np.frombuffer(data, dtype=np.uint8)
    got = []
    n = ctypes.c_size_t(0)
    small = np.empty(16, dtype=np.uint8)
    assert len(data) == 300001
    for lo in range(0, len(data), 100000):
        piece = src[lo:lo + 100000]
        if lo < 300000:   # more than a chunk is pending: these writes launch (the last byte only buffers)
            assert L.zb200_compress_stream_write(h, piece.ctypes.data, piece.size, small.ctypes.data, small.size,
                                                 ctypes.byref(n)) == 19
            assert n.value == 0
            assert L.zb200_compress_stream_write(h, piece.ctypes.data, piece.size, None, 0, ctypes.byref(n)) == 19
        big = np.empty(L.zb200_compress_stream_bound(h, piece.size), dtype=np.uint8)
        assert L.zb200_compress_stream_write(h, piece.ctypes.data, piece.size, big.ctypes.data, big.size,
                                             ctypes.byref(n)) == 0
        got.append(big[:n.value].tobytes())
    assert L.zb200_compress_stream_finish(h, small.ctypes.data, 4, ctypes.byref(n)) == 19
    big = np.empty(L.zb200_compress_stream_bound(h, 0), dtype=np.uint8)
    assert L.zb200_compress_stream_finish(h, big.ctypes.data, big.size, ctypes.byref(n)) == 0
    got.append(big[:n.value].tobytes())
    L.zb200_compress_stream_free(h)
    assert b"".join(got) == ref
    # free without finish, before and after a launch; the ctx goes on working
    for k in (1000, 3 * CHUNK):
        s = z.CompressStream(6, z.dfGzip, 2, ctx)
        s.write(data[:k])
        s.close()
    assert _stream(z, ctx, data, 6, z.dfGzip, 2, [(0, len(data))]) == _one_shot(z, ctx, data, 6, z.dfGzip, 2)


@pytest.mark.gpu
def test_stream_past_4_gib(z, corpus):
    """4 GiB + 1 MiB at level 1 in 256 MiB writes: the trailer CRC and ISIZE of the whole, checked by a streaming
    zlib inflate."""
    T = util.text_corpus(corpus)
    rng = np.random.default_rng(0x4B)
    piece = bytearray((T * ((256 << 20) // len(T) + 1))[:256 << 20])
    flips = rng.integers(0, len(piece), 1 << 16)
    arr = np.frombuffer(piece, dtype=np.uint8)
    arr[flips] = rng.integers(0, 256, len(flips), dtype=np.uint8)
    piece = bytes(piece)
    writes = [piece] * 16 + [piece[:1 << 20]]
    total = sum(map(len, writes))
    assert total == (4 << 30) + (1 << 20)
    crc_in = 0
    d = zlib.decompressobj(31)
    out_len, crc_out, tail = 0, 0, b""

    def take(c):
        nonlocal out_len, crc_out, tail
        if c:
            tail = (tail + c[-8:])[-8:]
            u = d.decompress(c)
            out_len += len(u)
            crc_out = zlib.crc32(u, crc_out)

    with z.CompressStream(z.BestSpeed, z.dfGzip, 0) as s:
        for w in writes:
            crc_in = zlib.crc32(w, crc_in)
            take(s.write(w))
        take(s.finish())
    u = d.flush()
    out_len += len(u)
    crc_out = zlib.crc32(u, crc_out)
    assert d.eof and not d.unused_data
    assert int.from_bytes(tail[:4], "little") == crc_in
    assert int.from_bytes(tail[4:], "little") == total % (1 << 32)
    assert out_len == total and crc_out == crc_in


def _cpp_stream_exe(tmp_path):
    exe = str(tmp_path / "cpp_stream_test")
    libdir = os.path.join(ROOT, "zippy_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(HERE, "native", "cpp_stream_test.cpp"),
                           "-L" + libdir, "-l:libzippy_b200.so", "-Wl,-rpath," + libdir])
    return exe


def test_cpp_stream_compiles_and_links(tmp_path):
    """zippy::CompressStream of include/zippy_b200.hpp builds against the library's stream symbols."""
    import __graft_entry__ as g
    g.build()
    assert os.path.exists(_cpp_stream_exe(tmp_path))


@pytest.mark.gpu
@pytest.mark.parametrize("level,fmt,piece", [(1, "gzip", 65537), (-1, "zlib", 100000), (9, "deflate", 1 << 20)])
def test_cpp_stream_matches_python(z, contexts, inputs, tmp_path, level, fmt, piece):
    exe = _cpp_stream_exe(tmp_path)
    data = inputs["mix"][0]
    src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
    src.write_bytes(data)
    subprocess.check_call([exe, str(src), str(dst), str(level), str(_df(z, fmt)), "13", str(piece)],
                          env=dict(os.environ, ZB200_STREAM_BATCH_BYTES="1"))
    py = _stream(z, contexts["every"], data, level, _df(z, fmt), 13, _splits(len(data), "random", [], 1))
    assert dst.read_bytes() == py == _one_shot(z, z.default_context(), data, level, _df(z, fmt), 13)
