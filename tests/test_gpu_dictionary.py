"""Preset dictionaries on the GPU (zb200_*_dict, dictionary= in Python): compressed bytes against the
stream-after-flush definition, interop with zlib's zdict both ways, verdicts against the CPU oracle's verdict on
stored(W) || S, and large batches through both host pipelines."""
import random
import zlib

import numpy as np
import pytest

from oracle import oracle as o
from tests import deflate_writer as dw
from tests import util
from tests.test_dictionary_rules import stored, window

pytestmark = pytest.mark.gpu

LEVELS = [-2, 0, 1, -1] + list(range(2, 10))
LZ_LEVELS = [-1] + list(range(2, 10))
WINDOWS = [1, 100, 8191, 8193, 32767, 32768, 100000]


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


@pytest.fixture(scope="module")
def text():
    return util.text_corpus(util.load_corpus())


def _msg(kind, n, rng, text):
    if kind == "text":
        a = rng.randrange(len(text) - n - 1)
        return text[a:a + n]
    if kind == "random":
        return rng.randbytes(n)
    if kind == "zeros":
        return bytes(n)
    if kind == "trap":  # short repeats just past matches of the window: lazy-match decisions
        unit = b"abcabcabd" + bytes([rng.randrange(256)])
        return (unit * (n // len(unit) + 1))[:n]
    out = bytearray()  # mix
    while len(out) < n:
        out += text[rng.randrange(100000):][:rng.randrange(1, 3000)] if rng.random() < 0.5 else rng.randbytes(rng.randrange(1, 500))
    return bytes(out[:n])


def _dict_for(text, dlen, rng):
    a = rng.randrange(len(text) - dlen - 1)
    return text[a:a + dlen]


def _stream_after_flush(z, level, w, m):
    """The definition of the blocks: a raw compress stream fed W, sync-flushed, then M."""
    cs = z.CompressStream(level, z.dfDeflate)
    cs.write(w)
    cs.flush(z.SyncFlush)
    out = cs.write(m) + cs.finish()
    cs.close()
    return out


def _abi(z, fn, *args):
    return getattr(z._native.lib(), fn)(*args)


def test_empty_dictionary_is_no_dictionary(z, text):
    rng = random.Random(1)
    items = [_msg(k, n, rng, text) for k in ("text", "random", "mix") for n in (0, 1, 4095, 70000)]
    ctx = z.default_context()
    base, offs = z._pack(items)
    for fmt in (z.dfZlib, z.dfDeflate):
        for level in LEVELS:
            ref, ro = ctx.compress_batch(base, offs, level, fmt)
            out = np.empty(ref.size + 4096, np.uint8)
            oo = np.zeros(len(items) + 1, np.uint64)
            st = np.zeros(len(items), np.int32)
            d = np.zeros(1, np.uint8)
            rc = _abi(z, "zb200_compress_batch_dict", ctx._h, base.ctypes.data, offs.ctypes.data, len(items), level, fmt,
                      d.ctypes.data, 0, out.ctypes.data, out.size, oo.ctypes.data, st.ctypes.data)
            assert rc == 0 and np.array_equal(oo, ro) and bytes(out[:int(oo[-1])]) == bytes(ref), (fmt, level)
        # decode side: same outputs and statuses, corrupted members included
        comp = z.compress_batch(items, 6, fmt) + [b"\x78\x20\0\0\0\0\x03\0\0\0\0\1", b"\x00\x01", b""]
        cb, co = z._pack(comp)
        d = np.zeros(1, np.uint8)
        s0, t0 = ctx.uncompressed_sizes(cb, co, fmt)
        s1 = np.zeros(len(comp), np.uint64)
        t1 = np.zeros(len(comp), np.int32)
        assert _abi(z, "zb200_uncompress_sizes_dict", ctx._h, cb.ctypes.data, co.ctypes.data, len(comp), fmt,
                    d.ctypes.data, 0, s1.ctypes.data, t1.ctypes.data) == 0
        assert np.array_equal(t0, t1) and np.array_equal(np.where(t0 == 0, s0, 0), np.where(t1 == 0, s1, 0))
        assert [r if isinstance(r, bytes) else r.code for r in z.uncompress_batch(comp, fmt)] == \
               [r if isinstance(r, bytes) else r.code for r in z.uncompress_batch(comp, fmt, dictionary=b"")]


@pytest.mark.parametrize("dlen", WINDOWS)
def test_compressed_bytes_definition(z, text, dlen):
    rng = random.Random(dlen)
    d = _dict_for(text, dlen, rng)
    w = window(d)
    sizes = [0, 1, 100, 4095, 65535, 65536, 65537, 1 << 20]
    kinds = ["text", "random", "zeros", "mix", "trap"]
    items = [_msg(kinds[i % len(kinds)], n, rng, text) for i, n in enumerate(sizes)]
    items += [d[-min(len(d), 5000):] + _msg("text", 3000, rng, text)]  # matches straight into W
    for level in LEVELS:
        raw = z.compress_batch(items, level, z.dfDeflate, dictionary=d)
        zl = z.compress_batch(items, level, z.dfZlib, dictionary=d)
        plain = z.compress_batch(items, level, z.dfDeflate) if level in (0, 1, -2) else None
        for i, m in enumerate(items):
            want = plain[i] if plain is not None else _stream_after_flush(z, level, w, m)
            assert raw[i] == want, (level, i)
            assert zl[i] == b"\x78\x20" + zlib.adler32(d).to_bytes(4, "big") + want + zlib.adler32(m).to_bytes(4, "big")
            assert zlib.decompressobj(-15, zdict=d).decompress(raw[i]) == m
            assert zlib.decompressobj(15, zdict=d).decompress(zl[i]) == m
        back = z.uncompress_batch(zl, z.dfZlib, dictionary=d)
        assert back == items, level
        assert z.uncompress_batch(raw, z.dfDeflate, dictionary=d) == items
    with pytest.raises(z.ZippyError) as e:
        z.compress(b"abc", 6, z.dfGzip, dictionary=d)
    assert e.value.code == 2


@pytest.mark.parametrize("wbits", [15, -15])
def test_decodes_zlib_zdict_output(z, text, wbits):
    rng = random.Random(wbits & 0xff)
    fmt = z.dfZlib if wbits > 0 else z.dfDeflate
    for dlen in (100, 32768, 100000):
        d = _dict_for(text, dlen, rng)
        comps, msgs = [], []
        for level, mem, strat in ((1, 8, zlib.Z_DEFAULT_STRATEGY), (6, 8, zlib.Z_DEFAULT_STRATEGY),
                                  (9, 9, zlib.Z_DEFAULT_STRATEGY), (6, 8, zlib.Z_FIXED), (6, 1, zlib.Z_DEFAULT_STRATEGY)):
            for flush in (None, zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH):
                m = _msg("mix", rng.randrange(1, 200000), rng, text)
                co = zlib.compressobj(level, zlib.DEFLATED, wbits, mem, strat, zdict=d)
                c = co.compress(m[:len(m) // 2]) + (co.flush(flush) if flush else b"") + co.compress(m[len(m) // 2:]) + co.flush()
                comps.append(c)
                msgs.append(m)
        assert z.uncompress_batch(comps, fmt, dictionary=d) == msgs
        sizes, st = z.uncompressed_sizes(comps, fmt, dictionary=d)
        assert list(st) == [0] * len(comps) and list(sizes) == [len(m) for m in msgs]
        for c, m in zip(comps[:4], msgs[:4]):
            assert z.uncompress(c, fmt, dictionary=d) == m
    if wbits > 0:  # DETECT: FDICT members next to plain zlib and gzip members
        d = text[:5000]
        co = zlib.compressobj(6, zlib.DEFLATED, 15, zdict=d)
        mixed = [co.compress(b"x" * 100 + d[:300]) + co.flush(), zlib.compress(b"plain"), zlib.compress(b"gz", wbits=31)]
        assert z.uncompress_batch(mixed, z.dfDetect, dictionary=d) == [b"x" * 100 + d[:300], b"plain", b"gz"]


def _expected(member, fmt, d):
    """The verdict and output the definition gives: the oracle on stored(W) || payload (zlib: header rules first,
    the Adler-32 of the output last)."""
    w = window(d)
    if fmt == "zlib":
        if len(member) < 6:
            return 3, None
        cmf, flg = member[0], member[1]
        if cmf & 15 != 8:
            return 10, None
        if cmf >> 4 > 7:
            return 11, None
        if (cmf * 256 + flg) % 31:
            return 12, None
        if flg & 0x20:
            if len(member) < 10:
                return 3, None
            if int.from_bytes(member[2:6], "big") != zlib.adler32(d):
                return 23, None
            payload = member[6:]
        else:
            try:
                return 0, o.uncompress(member, o.dfZlib)
            except o.ZippyError as e:
                return e.code, None
    else:
        payload = member
    try:
        out = o.uncompress(stored(w) + payload, o.dfDeflate)[len(w):]
    except o.ZippyError as e:
        return e.code, None
    if fmt == "zlib" and zlib.adler32(out) != int.from_bytes(member[-4:], "big"):
        return 14, None
    return 0, out


@pytest.mark.parametrize("fmt", ["deflate", "zlib"])
def test_corrupted_members_follow_definition(z, text, fmt):
    rng = random.Random(5 if fmt == "zlib" else 6)
    d = _dict_for(text, 40000, rng)
    df = z.dfZlib if fmt == "zlib" else z.dfDeflate
    srcs = [_msg("mix", rng.randrange(1, 20000), rng, text) for _ in range(30)]
    good = z.compress_batch(srcs, 6, df, dictionary=d)
    members = []
    for k in range(1500):
        b = bytearray(good[k % len(good)])
        kind = k % 3
        if kind == 0:
            for _ in range(rng.randrange(1, 3)):
                i = rng.randrange(len(b) * 8)
                b[i // 8] ^= 1 << (i % 8)
        elif kind == 1:
            b = b[:rng.randrange(len(b))]
        else:
            b += rng.randbytes(rng.randrange(1, 9))
        members.append(bytes(b))
    got = z.uncompress_batch(members, df, dictionary=d)
    for mbr, g in zip(members, got):
        st, out = _expected(mbr, fmt, d)
        if st == 0:
            assert g == out
        else:
            assert isinstance(g, z.ZippyError) and g.code == st, (st, g)
    for mbr in members[:150]:
        st, out = _expected(mbr, fmt, d)
        try:
            assert z.uncompress(mbr, df, dictionary=d) == out
        except z.ZippyError as e:
            assert e.code == st


def test_wrong_and_missing_dictionary(z, text):
    d = text[1000:41000]
    m = text[50000:60000]
    c = z.compress(m, 6, z.dfZlib, dictionary=d)
    for bad in (d[:-1] + bytes([d[-1] ^ 1]), d + b"x"):
        r = z.uncompress_batch([c], z.dfZlib, dictionary=bad)[0]
        assert isinstance(r, z.ZippyError) and r.code == 23
        with pytest.raises(z.ZippyError) as e:
            z.uncompress(c, z.dfZlib, dictionary=bad)
        assert e.value.code == 23
    assert z.uncompress_batch([c], z.dfZlib)[0].code == 13
    assert z.uncompress_batch([c[:9]], z.dfZlib, dictionary=d)[0].code == 3
    assert z._native.lib().zb200_strerror(23) != z._native.lib().zb200_strerror(99)


@pytest.mark.parametrize("wlen", [5, 32768])
def test_hand_built_distances(z, text, wlen):
    d = text[:wlen]
    lits = list(b"hello")
    if wlen < 32768:
        cases = [
            (lits + [(3, len(lits) + wlen)], True),        # reaches the first byte of W
            (lits + [(3, len(lits) + wlen + 1)], False),   # one byte before W
        ]
    else:  # a full window: the longest distance DEFLATE has reaches W's first byte from the output's start
        cases = [([(3, 32768)], True), (lits + [(3, 32768)], True)]
    if wlen >= 300:
        cases.append(([(258, 1000)], True))              # a 258-byte match inside W
    cases.append(([(10, 3)], True))                       # straddles the end of W (3 bytes of W, then its own output)
    cases.append(([(20, 2)], True))                       # overlapping, starting in W
    for tokens, ok in cases:
        s = dw.raw([dw.Fixed(tokens, final=True)])
        st, out = _expected(s, "deflate", d)
        assert (st == 0) == ok, tokens
        r = z.uncompress_batch([s], z.dfDeflate, dictionary=d)[0]
        if ok:
            assert r == out == zlib.decompressobj(-15, zdict=d).decompress(s)
            assert z.uncompress(s, z.dfDeflate, dictionary=d) == out
        else:
            assert isinstance(r, z.ZippyError) and r.code == st


@pytest.mark.parametrize("gated", ["0", "1"])
@pytest.mark.parametrize("group", ["1", "3"])
def test_large_batch(z, text, gated, group, monkeypatch):
    monkeypatch.setenv("ZB200_UNC_GATED", gated)
    monkeypatch.setenv("ZB200_GROUP_CHUNKS", group)
    ctx = z.Context()
    try:
        d = text[:32768]
        n, size = 65536, 4096
        rng = np.random.default_rng(9)
        starts = rng.integers(32768, len(text) - size, n)
        tarr = np.frombuffer(text, np.uint8)
        base = np.concatenate([tarr[s:s + size] for s in starts])
        offs = np.arange(n + 1, dtype=np.uint64) * size
        comp, co = ctx.compress_batch(base, offs, -1, z.dfZlib, dictionary=d)
        for i in range(0, n, 4099):
            assert zlib.decompressobj(15, zdict=d).decompress(bytes(comp[int(co[i]):int(co[i + 1])])) == \
                bytes(base[int(offs[i]):int(offs[i + 1])])
        sizes, st = ctx.uncompressed_sizes(comp, co, z.dfZlib, dictionary=d)
        assert (st == 0).all() and (sizes == size).all()
        for pinned in (False, True):
            src = comp
            if pinned:
                import torch
                src = torch.from_numpy(comp.copy()).pin_memory().numpy()
            out, do, lens, st = ctx.uncompress_batch(src, co, z.dfZlib, dictionary=d)
            assert (st == 0).all() and (lens == size).all()
            assert np.array_equal(out, base)
    finally:
        ctx.close()


def test_streams_with_dictionary(z, text):
    d = text[:50000]
    m = text[60000:60000 + 300000]
    for level in (-1, 1, 6):
        for fmt in (z.dfZlib, z.dfDeflate):
            want = z.compress(m, level, fmt, dictionary=d)
            rng = random.Random(level)
            cs = z.CompressStream(level, fmt, dictionary=d)
            out, i = b"", 0
            while i < len(m):
                k = rng.randrange(1, 70000)
                out += cs.write(m[i:i + k])
                i += k
            out += cs.finish()
            cs.close()
            assert out == want, (level, fmt)
    # a full flush drops the dictionary: a raw inflater started right after it decodes the rest
    cs = z.CompressStream(6, z.dfDeflate, dictionary=d)
    head = cs.write(m[:1000]) + cs.flush(z.FullFlush)
    tail = cs.write(d[-2000:] + m[:5000]) + cs.finish()
    assert zlib.decompressobj(-15).decompress(tail) == d[-2000:] + m[:5000]
    assert zlib.decompressobj(-15, zdict=d).decompress(head + tail) == m[:1000] + d[-2000:] + m[:5000]


def test_large_member_single_decode(z, text):
    d = text[:32768]
    m = (text * 20)[:24 << 20]
    c = z.compress(m, -1, z.dfZlib, dictionary=d)
    assert z.uncompress(c, z.dfZlib, dictionary=d) == m
    bad = bytearray(c)
    bad[-1] ^= 1
    with pytest.raises(z.ZippyError) as e:
        z.uncompress(bytes(bad), z.dfZlib, dictionary=d)
    assert e.value.code == 14


def _message_sets():
    corpus = util.load_corpus()
    out = {}
    for name in ("urls.10K", "alice29.txt", "html_x_4"):
        data = corpus[name]
        out[name] = (data[:32768], [data[i:i + 1024] for i in range(32768, len(data) - 1023, 1024)])
    return out


def test_ratio_against_zlib_zdict(z):
    """Every LZ level is smaller with the dictionary.  At Default, urls.10K and alice29.txt are within 1.10 x zlib
    level 6 with the same zdict.  html_x_4 is not (1.12, DESIGN 8 (j)): its messages are almost all matches into W,
    where k_lz2 looks at one candidate per 8 KiB segment of history, a search about as deep as zlib's short chains at
    levels 2-4 (the totals of all three sets lie between zlib 2 and 4), while zlib 6 walks up to 128 links; on this
    set zlib 3 is itself 1.09 x zlib 6.  So html_x_4 is held to zlib level 2 with the same zdict."""
    for name, (d, msgs) in _message_sets().items():
        zl = {6: 0, 2: 0}
        for m in msgs:
            for lv in zl:
                co = zlib.compressobj(lv, zlib.DEFLATED, 15, zdict=d)
                zl[lv] += len(co.compress(m) + co.flush())
        for level in LZ_LEVELS:
            a = sum(map(len, z.compress_batch(msgs, level, z.dfZlib)))
            b = sum(map(len, z.compress_batch(msgs, level, z.dfZlib, dictionary=d)))
            assert b < a, (name, level)
            if level == -1 and name == "html_x_4":
                assert b <= zl[2], (name, b, zl)
            elif level == -1:
                assert b <= 1.10 * zl[6], (name, b, zl[6], b / zl[6])


def _dstream(z, data, fmt, d, cuts=None, drain=False):
    s = z.DecompressStream(fmt, dictionary=d)
    out = b""
    pos = 0
    for c in (cuts or [len(data)]) + [len(data)]:
        out += s.write(data[pos:c])
        if drain:
            out += s.drain()
        pos = max(pos, c)
    out += s.finish()
    s.close()
    return out


@pytest.mark.parametrize("fmt", ["zlib", "deflate"])
def test_decompress_stream_with_dictionary(z, text, fmt):
    df = z.dfZlib if fmt == "zlib" else z.dfDeflate
    wbits = 15 if fmt == "zlib" else -15
    for dlen in (100, 32768, 100000):
        d = text[7 * dlen % 100000:][:dlen]
        m = d[-500:] + text[300000:300000 + 200000]
        c = z.compress(m, 6, df, dictionary=d)
        want = z.uncompress(c, df, dictionary=d)
        assert want == m
        # one-byte writes, with and without drains
        small = z.compress(m[:3000], -1, df, dictionary=d)
        assert _dstream(z, small, df, d, cuts=list(range(1, len(small)))) == m[:3000]
        assert _dstream(z, small, df, d, cuts=list(range(1, len(small), 7)), drain=True) == m[:3000]
        # a cut at every byte of the header and DICTID
        for k in range(11):
            assert _dstream(z, c, df, d, cuts=[k]) == m, (dlen, k)
        # zlib's zdict output with sync flushes: a drain after each flush yields everything up to it
        co = zlib.compressobj(6, zlib.DEFLATED, wbits, zdict=d)
        parts, sent = [], b""
        for i in range(5):
            piece = m[i * 20000:(i + 1) * 20000]
            parts.append(co.compress(piece) + co.flush(zlib.Z_SYNC_FLUSH))
        parts.append(co.flush())
        s = z.DecompressStream(df, dictionary=d)
        got = b""
        for i, p in enumerate(parts[:-1]):
            got += s.write(p) + s.drain()
            sent += m[i * 20000:(i + 1) * 20000]
            if fmt == "deflate" or i > 0:
                assert got == sent, (dlen, i)
        got += s.write(parts[-1]) + s.finish()
        s.close()
        assert got == m[:100000]
    # verdicts: the stream's status is uncompress's
    d = text[:40000]
    c = z.compress(text[50000:90000], 6, df, dictionary=d)
    for bad_d, code in ((d[:-1] + b"?", 23 if fmt == "zlib" else None), (None, 13 if fmt == "zlib" else None)):
        if code is None:
            continue
        s = z.DecompressStream(df, dictionary=bad_d)
        with pytest.raises(z.ZippyError) as e:
            s.write(c)
            s.finish()
        assert e.value.code == code
    bad = bytearray(c)
    bad[len(bad) // 2] ^= 0x10
    try:
        want = z.uncompress(bytes(bad), df, dictionary=d)
        assert _dstream(z, bytes(bad), df, d) == want
    except z.ZippyError as e:
        with pytest.raises(z.ZippyError) as e2:
            _dstream(z, bytes(bad), df, d)
        assert e2.value.code == e.code


def test_large_member_takes_parallel_path(z, text):
    d = text[:32768]
    m = (text * 40)[:64 << 20]
    c = z.compress(m, -1, z.dfZlib, dictionary=d)
    ctx = z.default_context()
    assert ctx.decode_one(c, z.dfZlib, dictionary=d) == m
    big = ctx.timing()["kernel_launches"]
    small = z.compress(m[:100000], -1, z.dfZlib, dictionary=d)
    assert ctx.decode_one(small, z.dfZlib, dictionary=d) == m[:100000]
    serial = ctx.timing()["kernel_launches"]
    # the serial decode is one inflate launch and its checks; the joint path adds the sync search, the segment
    # passes and the window resolve
    assert big >= serial + 3, (big, serial)


def test_cpp_reads_and_writes_python_bytes(z, text, tmp_path):
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "cpp_dict_test")
    libdir = os.path.join(root, "zippy_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(root, "tests", "native", "cpp_dict_test.cpp"),
                           "-L" + libdir, "-l:libzippy_b200.so", "-Wl,-rpath," + libdir])
    d = text[:50000]
    m = text[60000:60000 + 400000]
    for fmt in (z.dfZlib, z.dfDeflate):
        for level in (1, -1, 9):
            py = z.compress(m, level, fmt, dictionary=d)
            paths = {k: tmp_path / ("%s_%d_%d.bin" % (k, fmt, level)) for k in ("in", "dict", "member", "cpp", "data")}
            paths["in"].write_bytes(m)
            paths["dict"].write_bytes(d)
            paths["member"].write_bytes(py)
            subprocess.check_call([exe, str(paths["in"]), str(paths["dict"]), str(level), str(fmt), str(paths["member"]),
                                   str(paths["cpp"]), str(paths["data"])])
            assert paths["cpp"].read_bytes() == py
            assert paths["data"].read_bytes() == m
            assert zlib.decompressobj(15 if fmt == z.dfZlib else -15, zdict=d).decompress(py) == m
