"""Streaming decompression (zb200_decompress_stream_*, DecompressStream): whatever the sizes of the writes, the
concatenated output is uncompress(whole input) byte for byte, and the stream's final status is that call's.

Contexts with a small batching threshold (ZB200_DSTREAM_BATCH_BYTES = 1 / 100 000) make a stream launch at nearly
every write, so its resume point, window, checksum and output count cross many calls.  ZB200_DSTREAM_LOG makes every
launch name its decode path on stderr: joints (k_find_sync), blocks (k_find_blocks) or serial (one open segment)."""
import os
import random
import re
import subprocess
import zlib

import numpy as np
import pytest

from tests import util

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LEVELS = [-2, 0, 1, -1] + list(range(2, 10))
WBITS = {"gzip": 31, "zlib": 15, "deflate": -15}


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


def _df(z, fmt):
    return {"gzip": z.dfGzip, "zlib": z.dfZlib, "deflate": z.dfDeflate, "detect": z.dfDetect}[fmt]


@pytest.fixture(scope="module")
def contexts(z):
    """'every': a launch at every write; 'some': a launch once about 100 000 bytes are pending."""
    mp = pytest.MonkeyPatch()
    ctxs = {}
    try:
        mp.setenv("ZB200_DSTREAM_LOG", "1")
        for name, v in (("every", "1"), ("some", "100000")):
            mp.setenv("ZB200_DSTREAM_BATCH_BYTES", v)
            ctxs[name] = z.Context()
    finally:
        mp.undo()
    yield ctxs
    for c in ctxs.values():
        c.close()


def _stream(z, ctx, data, df, pieces):
    """-> (bytes read, status): the stream fed data[lo:hi] for every piece, then finish."""
    out = []
    try:
        with z.DecompressStream(df, ctx) as s:
            for lo, hi in pieces:
                out.append(s.write(data[lo:hi]))
            out.append(s.finish())
    except z.ZippyError as e:
        return b"".join(out), e.code
    return b"".join(out), 0


def _one_shot(z, data, df):
    try:
        return z.uncompress(data, df), 0
    except z.ZippyError as e:
        return None, e.code


def _pieces(cuts, n):
    cuts = sorted({0, n, *[c for c in cuts if 0 <= c <= n]})
    return list(zip(cuts[:-1], cuts[1:]))


def _splits(n, seed):
    """The write patterns of every identity check -> {name: pieces}"""
    rng = random.Random(seed)
    out = {"one": [(0, n)]}
    for w in (65535, 65536, 65537):
        out[w] = _pieces(range(0, n, w), n)
    out["random"] = _pieces([rng.randrange(n + 1) for _ in range(10)], n)
    cuts = sorted(rng.randrange(n + 1) for _ in range(6))
    out["empty_between"] = [p for lo, hi in _pieces(cuts, n) for p in ((lo, hi), (hi, hi))]
    out["head_tail"] = _pieces(list(range(0, min(n, 40))) + list(range(max(0, n - 12), n)), n)
    return out


def _members(z, corpus):
    """name -> (compressed member, format name, original)"""
    rng = random.Random(0xD5)
    T = util.text_corpus(corpus)
    o = rng.randrange(len(T) - 400000)
    contents = {"text": T[o:o + 300001], "random": rng.randbytes(150001), "zeros": bytes(200000),
                "mix": T[:90000] + rng.randbytes(50000) + bytes(70000) + T[90000:150000]}
    out = {}
    for level in LEVELS:
        for fmt in ("gzip", "zlib", "deflate"):
            for cname, data in contents.items():
                if level not in (1, -1, 9) and cname != "mix":
                    continue
                out["lib_%s_%d_%s" % (fmt, level, cname)] = (z.compress(data, level, _df(z, fmt)), fmt, data)
    text = contents["text"]
    for level in (1, 6, 9):
        out["zlib_%d" % level] = (zlib.compress(text, level), "zlib", text)
        co = zlib.compressobj(level, zlib.DEFLATED, 31)
        parts = [co.compress(text[i:i + 50000]) + co.flush(zlib.Z_SYNC_FLUSH) for i in range(0, len(text), 50000)]
        out["gzip_sync_%d" % level] = (b"".join(parts) + co.flush(), "gzip", text)
    co = zlib.compressobj(6, zlib.DEFLATED, -15, 9, zlib.Z_FIXED)
    out["fixed"] = (co.compress(text) + co.flush(), "deflate", text)
    co = zlib.compressobj(6, zlib.DEFLATED, 15, 1)
    out["memlevel1"] = (co.compress(text) + co.flush(), "zlib", text)
    return out


@pytest.fixture(scope="module")
def members(z, corpus):
    return _members(z, corpus)


@pytest.mark.gpu
def test_identity_members(z, contexts, members):
    """Every member under every write pattern, in both contexts, equals uncompress(whole) and zlib."""
    bad = []
    for k, (name, (comp, fmt, data)) in enumerate(sorted(members.items())):
        assert zlib.decompress(comp, WBITS[fmt]) == data, name
        for dfn in (fmt, "detect") if fmt != "deflate" else (fmt,):
            df = _df(z, dfn)
            ref = _one_shot(z, comp, df)
            assert ref == (data, 0), name
            for pname, pieces in _splits(len(comp), k).items():
                for cname in (("every", "some") if pname in ("random", "head_tail") else ("some",)):
                    got = _stream(z, contexts[cname], comp, df, pieces)
                    if got != ref:
                        bad.append((name, dfn, pname, cname, got[1], len(got[0])))
    assert not bad, bad[:20]


@pytest.mark.gpu
def test_identity_one_byte_writes(z, contexts, members, golden):
    """1-byte writes: members up to 64 KiB with launches every 100 000 bytes, a 3 KiB one launching at every byte."""
    bad = []
    small = [(n, c, f) for n, (c, f, _) in members.items() if len(c) <= 65536]
    small += [(n, c, "detect") for n, (c, _) in golden.items() if len(c) <= 65536]
    assert len(small) >= 8
    for name, comp, fmt in small:
        df = _df(z, fmt)
        if _stream(z, contexts["some"], comp, df, [(i, i + 1) for i in range(len(comp))]) != _one_shot(z, comp, df):
            bad.append(name)
    comp = zlib.compress(b"abcabcabd" * 300 + bytes(range(200)) + random.Random(9).randbytes(2000), 6)
    assert len(comp) < 4096
    if _stream(z, contexts["every"], comp, z.dfZlib, [(i, i + 1) for i in range(len(comp))]) != _one_shot(z, comp, z.dfZlib):
        bad.append("every_byte")
    assert not bad, bad


@pytest.mark.gpu
def test_identity_golden(z, contexts, golden):
    """All fixtures of tests/golden/ under DETECT (fixed.z under ZLIB too), every write pattern."""
    bad = []
    for k, (name, (comp, _)) in enumerate(sorted(golden.items())):
        fmts = [z.dfDetect] + ([z.dfZlib] if name == "fixed.z" else [z.dfGzip])
        for df in fmts:
            ref = _one_shot(z, comp, df)
            for pname, pieces in _splits(len(comp), k).items():
                for cname in ("every", "some"):
                    got = _stream(z, contexts[cname], comp, df, pieces)
                    if got != ref:
                        bad.append((name, df, pname, cname, got[1], ref[1]))
    assert len(golden) == 25
    assert not bad, bad[:20]


@pytest.mark.gpu
def test_each_decode_path(z, contexts, members, capfd):
    """The launch log shows each path taken: joints for this library's members, speculative blocks for a large zlib
    member, the open serial segment for stored random data."""
    T = members["zlib_6"][2]
    cases = {"joints": (members["lib_gzip_-1_text"][0], z.dfGzip, (T,)),
             "blocks": (zlib.compress(T * 4, 6), z.dfZlib, None),
             "serial": (z.compress(os.urandom(1 << 20), 1, z.dfGzip), z.dfGzip, None)}
    for path, (comp, df, _) in cases.items():
        capfd.readouterr()
        got = _stream(z, contexts["some"], comp, df, _pieces(range(0, len(comp), 1 << 20), len(comp)))
        err = capfd.readouterr().err
        assert got == _one_shot(z, comp, df), path
        paths = set(re.findall(r"zb200 dstream: path=(\w+)", err))
        assert path in paths, (path, paths)


@pytest.fixture(scope="module")
def big_member(z, corpus):
    """24 MiB of the C2-style text (64 KiB windows at seeded offsets) as one level-6 gzip member of this library:
    -> (member, original)"""
    T = util.text_corpus(corpus)
    data = b"".join(util.c2_block(T, i) for i in range(384))
    assert len(data) == 24 << 20
    return z.compress(data, 6, z.dfGzip), data


def _decoded_before(comp, end):
    """What zlib decodes from comp[:end]: every stream that has consumed its input past `end` has produced this."""
    return zlib.decompressobj(31).decompress(comp[:end])


@pytest.mark.gpu
def test_progress_before_finish(z, big_member):
    """The member in 1 MiB writes with a 1 MiB threshold, read after every write: the output grows on every write from
    the second on, and after the last write all that is still to come is the output of at most the threshold plus one
    64 KiB chunk of compressed input (plus the held-back trailer)."""
    comp, data = big_member
    thr = 1 << 20
    writes = list(range(0, len(comp), thr))
    assert len(writes) >= 6, len(comp)
    mp = pytest.MonkeyPatch()
    mp.setenv("ZB200_DSTREAM_BATCH_BYTES", str(thr))
    ctx = z.Context()
    mp.undo()
    got = []
    with z.DecompressStream(z.dfGzip, ctx) as s:
        for i in writes:
            got.append(s.write(comp[i:i + thr]))
        before = b"".join(got)
        got.append(s.finish())
    ctx.close()
    assert b"".join(got) == data
    assert data.startswith(before)
    # the first write leaves less than the threshold of payload pending; every later full write launches
    grew = [k for k, u in enumerate(got[:len(writes) - 1]) if u]
    assert grew == list(range(1, len(writes) - 1)), grew
    assert len(before) >= len(_decoded_before(comp, len(comp) - thr - 65536 - 8)) > len(data) // 2


@pytest.mark.gpu
def test_large_write_in_slices(z, contexts, big_member, capfd):
    """One write of the whole member on a context with a 100 000-byte threshold: it is decoded by many launches, each
    staging only a slice of the held input, and returns everything but the last slice's worth."""
    comp, data = big_member
    capfd.readouterr()
    with z.DecompressStream(z.dfGzip, contexts["some"]) as s:
        before = s.write(comp)
        launches = len(re.findall(r"zb200 dstream: path=", capfd.readouterr().err))
        rest = s.finish()
    assert before + rest == data
    assert launches >= len(comp) // 200000, launches
    assert len(before) >= len(_decoded_before(comp, len(comp) - 100000 - 65536 - 8))


def _errors_match(z, ctx, comp, df, pieces, truncated=None, partial=None, what=None):
    got, code = _stream(z, ctx, comp, df, pieces)
    ref, rcode = _one_shot(z, comp, df)
    assert code == rcode, (what, code, rcode, len(got))
    if rcode == 0:
        assert got == ref
    if truncated is not None:
        assert truncated.startswith(got)
    if partial is not None:
        a, b = sorted((got, partial), key=len)
        assert b.startswith(a)
    return code


@pytest.mark.gpu
def test_errors(z, contexts, members):
    from oracle import oracle as o
    rng = random.Random(0xE7)
    for name in ("lib_gzip_1_mix", "lib_zlib_-1_mix", "lib_deflate_9_mix", "zlib_6", "gzip_sync_9", "fixed"):
        comp, fmt, data = members[name]
        df = _df(z, fmt)
        n = len(comp)
        splits = _splits(n, 3)
        # bit flips: the status of the whole, and the shorter of (read, zlib's partial output) prefixes the longer
        for _ in range(16):
            b = bytearray(comp)
            p = rng.randrange(n)
            b[p] ^= 1 << rng.randrange(8)
            b = bytes(b)
            d = zlib.decompressobj(WBITS[fmt])
            try:
                part = d.decompress(b)
            except zlib.error:
                part = b""
            code = _errors_match(z, contexts["some"], b, df, splits["random"], partial=part if part else None,
                                 what=(name, p, comp[p], b[p]))
            try:
                o.uncompress(b, df)
                ocode = 0
            except o.ZippyError as e:
                ocode = e.code
            assert ocode == code, (name, p)
        # truncations inside the header, mid-data, inside the trailer
        for cut in (1, 5, 11, n // 3, n // 2, n - 7, n - 3, n - 1):
            for cname in ("every", "some"):
                _errors_match(z, contexts[cname], comp[:cut], df, _pieces([cut // 2], cut), truncated=data,
                              what=(name, cut, cname))
        # trailing garbage, a wrong ISIZE / checksum
        g = comp + b"garbage!" * 3
        _errors_match(z, contexts["some"], g, df, _pieces(range(0, len(g), 65536), len(g)), what=(name, "garbage"))
        if fmt != "deflate":
            b = bytearray(comp)
            b[-1] ^= 0x40
            assert _errors_match(z, contexts["every"], bytes(b), df, splits["random"], what=(name, "trailer")) in (14, 18)


@pytest.mark.gpu
def test_short_inputs_every_split(z, contexts):
    """Inputs of 0..40 bytes with gzip, zlib and garbage prefixes, under every two-way split and every format."""
    gz = zlib.compress(b"hello hello hello", 9)
    gzip_m = zlib.compressobj(9, zlib.DEFLATED, 31)
    gzip_m = gzip_m.compress(b"hi") + gzip_m.flush()
    rng = random.Random(5)
    bases = [gzip_m + b"\x00" * 20, gz + b"\x00" * 30, bytes(rng.randrange(256) for _ in range(40)),
             b"\x1f\x8b\x08\x08abc\x00" + b"\x00" * 32]
    ctx = contexts["every"]
    for base in bases:
        for n in range(0, 41):
            data = base[:n]
            for df in (z.dfDetect, z.dfGzip, z.dfZlib, z.dfDeflate):
                ref = _one_shot(z, data, df)
                for c in range(0, n + 1):
                    got = _stream(z, ctx, data, df, [(0, c), (c, n)])
                    assert got[1] == ref[1], (base[:4], n, df, c, got, ref)
                    if ref[1] == 0:
                        assert got[0] == ref[0]


@pytest.mark.gpu
def test_contract(z, contexts, members):
    import ctypes
    from zippy_b200 import _native
    L = _native.lib()
    ctx = contexts["every"]
    for df in (4, -1):
        with pytest.raises(z.ZippyError) as e:
            z.DecompressStream(df, ctx)
        assert e.value.code == 2
    comp, fmt, data = members["lib_gzip_1_text"]
    # write / finish after finish
    s = z.DecompressStream(z.dfGzip, ctx)
    out = s.write(comp) + s.finish()
    assert out == data
    for call in (lambda: s.write(b"x"), s.finish):
        with pytest.raises(z.ZippyError) as e:
            call()
        assert e.value.code == 22
    s.close()
    # every call after an error repeats it
    s = z.DecompressStream(z.dfZlib, ctx)
    with pytest.raises(z.ZippyError) as e:
        s.write(b"\x1f\x8b" + bytes(30))
    first = e.value.code
    for call in (lambda: s.write(b"more"), s.finish, lambda: s.write(b"")):
        with pytest.raises(z.ZippyError) as e:
            call()
        assert e.value.code == first
    s.close()
    # read with a small dst_cap drains the output in pieces
    h = ctypes.c_void_p()
    assert L.zb200_decompress_stream_begin(ctx._h, z.dfGzip, ctypes.byref(h)) == 0
    src = np.frombuffer(comp, dtype=np.uint8)
    avail = ctypes.c_size_t(0)
    assert L.zb200_decompress_stream_write(h, src.ctypes.data, src.size, ctypes.byref(avail)) == 0
    assert L.zb200_decompress_stream_finish(h, ctypes.byref(avail)) == 0
    assert avail.value == len(data)
    buf = np.empty(1000, dtype=np.uint8)
    n = ctypes.c_size_t(0)
    got = []
    while True:
        assert L.zb200_decompress_stream_read(h, buf.ctypes.data, 777, ctypes.byref(n)) == 0
        if not n.value:
            break
        got.append(buf[:n.value].tobytes())
    L.zb200_decompress_stream_free(h)
    assert b"".join(got) == data and max(map(len, got)) == 777
    # freeing unfinished streams, before and after a launch; the ctx goes on working
    for k in (10, 1000, len(comp) // 2):
        s = z.DecompressStream(z.dfGzip, ctx)
        s.write(comp[:k])
        s.close()
    assert _stream(z, ctx, comp, z.dfGzip, [(0, len(comp))]) == (data, 0)


@pytest.mark.gpu
def test_interleaved_streams(z, contexts, members):
    """Two streams on one ctx, with batch calls between their writes, read what each reads alone."""
    ctx = contexts["every"]
    a, b = members["lib_gzip_-1_text"], members["zlib_9"]
    s1, s2 = z.DecompressStream(z.dfGzip, ctx), z.DecompressStream(z.dfZlib, ctx)
    o1, o2 = [], []
    items = [b"abc" * 1000, os.urandom(5000)]
    comp = z._pack([z.compress(x) for x in items])
    step = 65537
    for i in range(0, max(len(a[0]), len(b[0])), step):
        o1.append(s1.write(a[0][i:i + step]))
        base, offs = z._pack(items)
        ctx.compress_batch(base, offs, 6, z.dfGzip)
        o2.append(s2.write(b[0][i:i + step]))
        _, _, _, st = ctx.uncompress_batch(*comp)
        assert list(st) == [0, 0]
    o2.append(s2.finish())
    o1.append(s1.finish())
    s1.close()
    s2.close()
    assert b"".join(o1) == a[2] and b"".join(o2) == b[2]


@pytest.mark.gpu
def test_stream_past_4_gib(z, corpus):
    """A 4 GiB + 1 MiB Default-level gzip member written by CompressStream, decoded in 256 MiB writes: its sha256 equals
    streaming zlib's, and the CRC / ISIZE (mod 2^32) checks pass."""
    import hashlib
    T = util.text_corpus(corpus)
    rng = np.random.default_rng(0x4C)
    piece = bytearray((T * ((256 << 20) // len(T) + 1))[:256 << 20])
    flips = rng.integers(0, len(piece), 1 << 16)
    arr = np.frombuffer(piece, dtype=np.uint8)
    arr[flips] = rng.integers(0, 256, len(flips), dtype=np.uint8)
    piece = bytes(piece)
    writes = [piece] * 16 + [piece[:1 << 20]]
    total = sum(map(len, writes))
    comp = []
    with z.CompressStream(z.DefaultCompression, z.dfGzip, 0) as s:
        for w in writes:
            comp.append(s.write(w))
        comp.append(s.finish())
    comp = b"".join(comp)
    want = hashlib.sha256()
    for w in writes:
        want.update(w)
    d = zlib.decompressobj(31)
    zh = hashlib.sha256()
    for i in range(0, len(comp), 256 << 20):
        zh.update(d.decompress(comp[i:i + (256 << 20)]))
    zh.update(d.flush())
    assert zh.digest() == want.digest()
    assert int.from_bytes(comp[-4:], "little") == total % (1 << 32)
    gh = hashlib.sha256()
    n = 0
    with z.DecompressStream(z.dfGzip) as s:
        for i in range(0, len(comp), 256 << 20):
            u = s.write(comp[i:i + (256 << 20)])
            n += len(u)
            gh.update(u)
        u = s.finish()
        n += len(u)
        gh.update(u)
    assert n == total and gh.digest() == want.digest()


def _cpp_dstream_exe(tmp_path):
    exe = str(tmp_path / "cpp_dstream_test")
    libdir = os.path.join(ROOT, "zippy_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(HERE, "native", "cpp_dstream_test.cpp"),
                           "-L" + libdir, "-l:libzippy_b200.so", "-Wl,-rpath," + libdir])
    return exe


def test_cpp_dstream_compiles_and_links(tmp_path):
    """zippy::DecompressStream of include/zippy_b200.hpp builds against the library's stream symbols."""
    import __graft_entry__ as g
    g.build()
    assert os.path.exists(_cpp_dstream_exe(tmp_path))


@pytest.mark.gpu
@pytest.mark.parametrize("name,piece", [("lib_gzip_-1_mix", 65537), ("zlib_6", 100000), ("fixed", 1 << 20)])
def test_cpp_dstream_matches_python(z, contexts, members, tmp_path, name, piece):
    exe = _cpp_dstream_exe(tmp_path)
    comp, fmt, data = members[name]
    src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
    src.write_bytes(comp)
    subprocess.check_call([exe, str(src), str(dst), str(_df(z, fmt)), str(piece)],
                          env=dict(os.environ, ZB200_DSTREAM_BATCH_BYTES="1"))
    py = _stream(z, contexts["every"], comp, _df(z, fmt), _pieces(range(0, len(comp), 50000), len(comp)))
    assert dst.read_bytes() == py[0] == data and py[1] == 0
