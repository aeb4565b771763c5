"""Random access into one member (zippy_b200.Index): the access points against a CPU model built from
tests/deflate_tokens.py, ranges against uncompress, the launch economy and the per-range verdicts."""
import os
import random
import zlib

import numpy as np
import pytest

from tests import deflate_tokens as dt

pytestmark = pytest.mark.gpu

z = pytest.importorskip("zippy_b200")

ERR_UNCOMPRESS, ERR_CHECKSUM, ERR_ARG, ERR_INVALID_FORMAT = 3, 14, 22, 2


def _payload_start(data, fmt):
    """Where the raw DEFLATE payload starts (the header zippy_b200 and Python write: no FEXTRA / FCOMMENT)."""
    if fmt == z.dfDeflate:
        return 0
    if fmt == z.dfZlib:
        return 2
    flg, p = data[3], 10
    if flg & 4:
        p += 2 + data[10] + 256 * data[11]
    for bit in (8, 16):
        if flg & bit:
            p = data.index(b"\0", p) + 1
    if flg & 2:
        p += 2
    return p


def model_points(data, fmt, span):
    """The index's points by their definition: (bit, out, crc, window) per segment point."""
    P = _payload_start(data, fmt)
    blocks = dt.parse(data[P:])
    starts, o = [], 0
    for b in blocks:
        starts.append((b.bit_start + 8 * P, o))
        o += b.size()
    total = o
    pts, i = [], 0
    for k in range(total // 32768 + 1):
        while i < len(starts) and starts[i][1] < k * 32768:
            i += 1
        if i == len(starts):
            break
        if not pts or pts[-1] != starts[i]:
            pts.append(starts[i])
    out = zlib.decompressobj(-15).decompress(data[P:])
    assert len(out) == total
    res, nxt = [], 0
    for j, (bit, o) in enumerate(pts):
        end = pts[j + 1][1] if j + 1 < len(pts) else total
        win = o >= nxt
        if win:
            nxt = (o // span + 1) * span
        res.append((bit, o, zlib.crc32(out[o:end]), int(win)))
    return res, out


def index_points(idx):
    p = idx.points
    return [(int(b), int(o), int(c), int(w)) for b, o, c, w in zip(p["bit"], p["out"], p["crc"], p["window"])]


def _text(n, seed=1):
    rng = random.Random(seed)
    words = [bytes(rng.choice(b"abcdefghijklmnopqrstuvwxyz") for _ in range(rng.randint(2, 9))) for _ in range(3000)]
    out = bytearray()
    while len(out) < n:
        out += rng.choice(words) + (b"\n" if rng.random() < 0.1 else b" ")
    return bytes(out[:n])


def _finish(co, data):
    return co.compress(data) + co.flush()


def _members():
    text = _text(1 << 20)
    rnd = np.random.default_rng(5).integers(0, 256, 600000, dtype=np.uint8).tobytes()
    mix = text[:300000] + rnd[:200000] + bytes(150000) + text[300000:700000]
    co = zlib.compressobj(6, zlib.DEFLATED, 15)
    flushed = b""
    for k in range(0, len(text), 100000):
        flushed += co.compress(text[k:k + 100000]) + co.flush(zlib.Z_SYNC_FLUSH if k % 200000 else zlib.Z_FULL_FLUSH)
    flushed += co.flush()
    fixed = zlib.compressobj(6, zlib.DEFLATED, -15, 9, zlib.Z_FIXED)

    return [
        ("lib1-gzip-text", z.compress(text, 1, z.dfGzip), z.dfGzip),
        ("lib6-gzip-mix", z.compress(mix, 6, z.dfGzip), z.dfGzip),
        ("lib3-raw-text", z.compress(text, 3, z.dfDeflate), z.dfDeflate),
        ("lib-default-zlib-text", z.compress(text, z.DefaultCompression, z.dfZlib), z.dfZlib),
        ("lib9-raw-mix", z.compress(mix, 9, z.dfDeflate), z.dfDeflate),
        ("lib0-zlib-random", z.compress(rnd, 0, z.dfZlib), z.dfZlib),
        ("lib1-raw-random", z.compress(rnd, 1, z.dfDeflate), z.dfDeflate),
        ("lib-2-gzip-zeros", z.compress(bytes(1 << 20), -2, z.dfGzip), z.dfGzip),
        ("py6-zlib", zlib.compress(text, 6), z.dfZlib),
        ("py9-zlib", zlib.compress(text, 9), z.dfZlib),
        ("py1-zlib-text", zlib.compress(text, 1), z.dfZlib),
        ("py1-zlib-mix", zlib.compress(mix, 1), z.dfZlib),
        ("py6-zlib-flushes", flushed, z.dfZlib),
        ("py-fixed-raw", _finish(fixed, text[:400000]), z.dfDeflate),
        ("py-memlevel1-zlib", _finish(zlib.compressobj(6, zlib.DEFLATED, 15, 1), text), z.dfZlib),
    ]


MEMBERS = None


def members():
    global MEMBERS
    if MEMBERS is None:
        MEMBERS = _members()
    return MEMBERS


@pytest.mark.parametrize("span", [32768, 65536, 1 << 20])
def test_points_match_the_model(span):
    for name, data, fmt in members():
        want, out = model_points(data, fmt, span)
        idx = z.Index.build(data, fmt, span)
        assert idx.size == len(out), name
        assert index_points(idx) == want, name
        idx.close()


def test_golden_fixtures_points():
    gold = os.path.join(os.path.dirname(__file__), "golden")
    names = sorted(f for f in os.listdir(gold) if f.endswith(".gz"))
    checked = 0
    for f in names:
        data = open(os.path.join(gold, f), "rb").read()
        try:
            want, out = model_points(data, z.dfGzip, 65536)
        except Exception:
            continue   # not a single plain member (the model reads one member only)
        checked += 1
        idx = z.Index.build(data, z.dfGzip, 65536)
        assert index_points(idx) == want, f
        assert idx.extract(data, 0, idx.size) == out, f
    assert checked >= 20, checked


def _hand_built():
    from tests import deflate_writer as dw
    rng = random.Random(21)

    def lits(n):
        return [rng.randrange(256) for _ in range(n)]
    empties = [dw.Fixed([]) for _ in range(40)]
    streams = [
        ("empty-blocks", [dw.Fixed(lits(1000))] + empties + [dw.Fixed(lits(40000))] + empties + [dw.Fixed(lits(30000))]),
        ("32767-32768-32769", [dw.Fixed(lits(32767)), dw.Fixed(lits(32768)), dw.Fixed(lits(32769)), dw.Fixed(lits(5))]),
        ("one-long-block", [dw.Fixed(lits(100)), dw.Dynamic(lits(3 * 32768 + 777)), dw.Fixed(lits(9))]),
        ("stored-mid-stream", [dw.Fixed(lits(20000)), dw.Stored(bytes(lits(65535))), dw.Stored(b""),
                               dw.Fixed([1, 2, 3, (258, 3)] * 100), dw.Stored(bytes(lits(40000)))]),
        ("matches-across-points", [dw.Fixed(lits(33000)), dw.Fixed([(258, 32768)] * 300), dw.Fixed([(3, 1)] * 20000)]),
        ("one-block", [dw.Dynamic(lits(200000))]),
        ("empty-member", [dw.Fixed([])]),
    ]
    out = []
    for name, blocks in streams:
        raw = dw.raw(blocks)
        data = dw.replay(blocks)
        out.append((name + "-raw", raw, z.dfDeflate))
        out.append((name + "-zlib", dw.zlib_wrap(raw, data), z.dfZlib))
        out.append((name + "-gzip", dw.gzip_wrap(raw, data), z.dfGzip))
    return out


@pytest.mark.parametrize("span", [32768, 65536])
def test_hand_built_streams(span):
    for name, data, fmt in _hand_built():
        want, out = model_points(data, fmt, span)
        idx = z.Index.build(data, fmt, span)
        assert index_points(idx) == want, name
        got, goff, st = idx.extract_batch(data, [0] + [int(o) for o in idx.points["out"]], [len(out)] + [
            min(70000, len(out) - int(o)) for o in idx.points["out"]])
        assert (st == 0).all(), name
        assert got[:len(out)].tobytes() == out, name


def parse_export(buf):
    """The documented serialisation, read back: header fields, points and the decompressed windows."""
    import struct
    assert buf[:8] == b"ZB200IDX"
    version, fmt = struct.unpack_from("<II", buf, 8)
    payload, length, size, span, _ = struct.unpack_from("<5Q", buf, 16)
    np_, nw = struct.unpack_from("<QQ", buf, 120)
    pts = [struct.unpack_from("<QQII", buf, 136 + 24 * i) for i in range(np_)]
    pos = 136 + 24 * np_
    clen = struct.unpack_from("<%dQ" % nw, buf, pos)
    pos += 8 * nw
    wins = []
    for c in clen:
        wins.append(zlib.decompress(buf[pos:pos + c], -15))
        pos += c
    assert pos + 4 == len(buf) and struct.unpack_from("<I", buf, pos)[0] == zlib.crc32(buf[:pos])
    return dict(version=version, fmt=fmt, payload=payload, len=length, size=size, span=span, points=pts, windows=wins)


def test_windows_are_the_output_in_front_of_their_points():
    for name, data, fmt in members()[:6] + _hand_built()[:6]:
        idx = z.Index.build(data, fmt, 65536)
        out = z.uncompress(data, fmt)
        e = parse_export(idx.to_bytes())
        assert e["size"] == len(out) and e["len"] == len(data) and e["span"] == 65536
        wins = [o for _, o, _, w in e["points"] if w and o > 0]
        assert [out[o - 32768:o] for o in wins] == e["windows"], name


def test_serialisation_round_trip_and_determinism():
    text = _text(3 << 20, seed=31)
    data = z.compress(text, z.DefaultCompression, z.dfGzip)
    c1, c2 = z.Context(), z.Context()
    idx = z.Index.build(data, span=65536, ctx=c1)
    ref = idx.to_bytes()
    for ctx in (c1, c2):
        for _ in range(3):
            assert z.Index.build(data, span=65536, ctx=ctx).to_bytes() == ref
    back = z.Index.from_bytes(ref, ctx=c2)
    assert index_points(back) == index_points(idx) and back.size == idx.size
    rng = random.Random(3)
    offs = [rng.randrange(len(text) - 9000) for _ in range(300)]
    a = idx.extract_batch(data, offs, [9000] * 300)
    b = back.extract_batch(data, offs, [9000] * 300)
    assert (a[2] == 0).all() and (b[2] == 0).all() and a[0].tobytes() == b[0].tobytes()
    assert back.to_bytes() == ref


def _expect_arg(buf, ctx):
    with pytest.raises(z.ZippyError) as e:
        z.Index.from_bytes(buf, ctx=ctx)
    assert e.value.code == ERR_ARG


def test_malformed_indexes_are_rejected():
    import struct
    text = _text(300000, seed=32)
    data = z.compress(text, 1, z.dfZlib)
    ctx = z.Context()
    buf = z.Index.build(data, z.dfZlib, 65536, ctx=ctx).to_bytes()
    for k in range(len(buf)):
        _expect_arg(buf[:k], ctx)
    rng = random.Random(33)
    for _ in range(200):
        b = bytearray(buf)
        b[rng.randrange(len(b))] ^= 1 + rng.randrange(255)
        _expect_arg(bytes(b), ctx)

    def resealed(b):
        b = bytearray(b[:-4])
        return bytes(b) + struct.pack("<I", zlib.crc32(b))
    np_ = struct.unpack_from("<Q", buf, 120)[0]
    assert np_ >= 4
    # two points swapped (not increasing), a window flag flipped, a wrong count, a window that is not 32 KiB
    b = bytearray(buf)
    b[136 + 24:136 + 48], b[136 + 48:136 + 72] = buf[136 + 48:136 + 72], buf[136 + 24:136 + 48]
    _expect_arg(resealed(b), ctx)
    for p in range(np_):
        b = bytearray(buf)
        b[136 + 24 * p + 20] ^= 1
        _expect_arg(resealed(b), ctx)
    b = bytearray(buf)
    struct.pack_into("<Q", b, 120, np_ + 1)
    _expect_arg(resealed(b), ctx)
    e = parse_export(buf)
    assert e["windows"]
    short = zlib.compressobj(1, zlib.DEFLATED, -15)
    w0 = short.compress(e["windows"][0][:-1]) + short.flush()
    pos = 136 + 24 * np_
    nw = len(e["windows"])
    c0 = struct.unpack_from("<Q", buf, pos)[0]
    b = bytearray(buf[:pos]) + struct.pack("<Q", len(w0)) + buf[pos + 8:pos + 8 * nw] + w0 + \
        buf[pos + 8 * nw + c0:len(buf) - 4] + b"\0\0\0\0"
    _expect_arg(resealed(bytes(b)), ctx)
    z.Index.from_bytes(buf, ctx=ctx).close()


def test_cpp_index_matches_python(tmp_path):
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "cpp_index_test")
    libdir = os.path.join(root, "zippy_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe,
                           os.path.join(root, "tests", "native", "cpp_index_test.cpp"),
                           "-L" + libdir, "-l:libzippy_b200.so", "-Wl,-rpath," + libdir])
    text = _text(2 << 20, seed=34)
    data = z.compress(text, z.DefaultCompression, z.dfZlib)
    m, ix, rg = tmp_path / "m.bin", tmp_path / "ix.bin", tmp_path / "r.bin"
    m.write_bytes(data)
    subprocess.check_call([exe, str(m), str(z.dfZlib), "65536", str(ix), "1000000", "70000", str(rg)])
    assert ix.read_bytes() == z.Index.build(data, z.dfZlib, 65536).to_bytes()
    assert rg.read_bytes() == text[1000000:1070000]


def test_empty_and_tiny_members():
    for data in (zlib.compress(b""), zlib.compress(b"x"), z.compress(b"", 1, z.dfZlib)):
        idx = z.Index.build(data, z.dfZlib, 32768)
        want, out = model_points(data, z.dfZlib, 32768)
        assert index_points(idx) == want
        assert idx.extract(data, 0, idx.size) == out
        assert idx.extract(data, idx.size, 0) == b""


def _check_ranges(idx, data, out, ranges):
    offs = [a for a, _ in ranges]
    lens = [n for _, n in ranges]
    got, goff, st = idx.extract_batch(data, offs, lens)
    assert (st == 0).all()
    for i, (a, n) in enumerate(ranges):
        assert got[int(goff[i]):int(goff[i + 1])].tobytes() == out[a:a + n], (a, n)


def _edge_ranges(idx, size, rng):
    pts = [int(o) for o in idx.points["out"]]
    r = [(0, 0), (0, size), (size - 1, 1), (size, 0)]
    for p in pts[1:8] + pts[-4:]:
        for d in (-1, 0, 1):
            a = min(max(p + d, 0), size)
            r.append((a, min(5000, size - a)))
            r.append((max(a - 3000, 0), a - max(a - 3000, 0)))
    for _ in range(40):
        a = rng.randrange(size)
        r.append((a, rng.randrange(min(size - a, 300000) + 1)))
    r.append((size // 3, size // 2))
    r.append((size // 3 + 7, size // 2))
    return r


@pytest.mark.parametrize("group_bytes", [None, 100000])
def test_ranges_equal_uncompress(group_bytes, monkeypatch):
    if group_bytes:
        monkeypatch.setenv("ZB200_INDEX_GROUP_BYTES", str(group_bytes))
    ctx = z.Context()
    rng = random.Random(7)
    for name, data, fmt in members():
        out = z.uncompress(data, fmt)
        idx = z.Index.build(data, fmt, 65536, ctx=ctx)
        ranges = _edge_ranges(idx, len(out), rng)
        _check_ranges(idx, data, out, ranges)
        for a, n in ranges[:12]:
            assert idx.extract(data, a, n) == out[a:a + n], name
        idx.close()
    ctx.close()


@pytest.mark.parametrize("group_bytes", [None, 1 << 20])
def test_many_small_reads_on_a_large_member(group_bytes, monkeypatch):
    if group_bytes:
        monkeypatch.setenv("ZB200_INDEX_GROUP_BYTES", str(group_bytes))
    text = _text(4 << 20, seed=3) * 16
    data = z.compress(text, 1, z.dfGzip)
    idx = z.Index.build(data, ctx=z.Context())
    rng = random.Random(11)
    ranges = [(a, 4096) for a in (rng.randrange(len(text) - 4096) for _ in range(10000))]
    _check_ranges(idx, data, text, ranges)


def test_launches_do_not_grow_with_the_number_of_ranges():
    text = _text(8 << 20, seed=4)
    data = z.compress(text, 1, z.dfZlib)
    ctx = z.Context()
    idx = z.Index.build(data, z.dfZlib, 1 << 20, ctx=ctx)
    base = 3 << 20
    idx.extract_batch(data, [base], [4096])
    one = ctx.timing()["kernel_launches"]
    rng = random.Random(2)
    offs = [base + rng.randrange(1 << 20) for _ in range(1000)]
    _, _, st = idx.extract_batch(data, offs, [4096] * 1000)
    assert (st == 0).all()
    many = ctx.timing()["kernel_launches"]
    assert one == many


def test_one_read_uploads_only_its_chain():
    text = _text(256 << 20, seed=6)
    data = z.compress(text, 1, z.dfGzip)
    ctx = z.Context()
    idx = z.Index.build(data, ctx=ctx)
    pts = idx.points
    a = 100 << 20
    out, _, st = idx.extract_batch(data, [a], [4096])
    assert st[0] == 0 and out.tobytes() == text[a:a + 4096]
    h2d = ctx.timing()["h2d_bytes"]
    o, b, w = pts["out"].astype(np.int64), pts["bit"].astype(np.int64), pts["window"]
    wp = max(i for i in range(len(o)) if w[i] and o[i] <= a)
    ep = next((i for i in range(len(o)) if o[i] >= a + 4096), None)
    end_byte = (int(b[ep]) + 7) // 8 if ep is not None else len(data)
    assert h2d <= end_byte - int(b[wp]) // 8 + 32768 + 65536


def test_serial_members_decode_as_many_segments(capfd, monkeypatch):
    monkeypatch.setenv("ZB200_INDEX_LOG", "1")
    monkeypatch.setenv("ZB200_INDEX_GROUP_BYTES", str(4 << 20))
    rnd = np.random.default_rng(9).integers(0, 256, 16 << 20, dtype=np.uint8).tobytes()
    text = _text(16 << 20, seed=8)
    ctx = z.Context()
    for data, out in ((z.compress(rnd, 1, z.dfGzip), rnd), (zlib.compress(text, 6), text)):
        idx = z.Index.build(data, ctx=ctx)
        capfd.readouterr()
        assert idx.extract(data, 0, idx.size) == out
        err = capfd.readouterr().err
        lines = [l for l in err.splitlines() if l.startswith("zb200 index:")]
        assert len(lines) > 1
        assert sum(int(l.split(" chains, ")[1].split(" segments")[0]) for l in lines) > 1


def test_build_verdicts_follow_uncompress():
    from oracle import oracle as o
    text = _text(1 << 20, seed=12)
    rng = random.Random(13)
    for data in (z.compress(text, 1, z.dfGzip), zlib.compress(text, 6)):
        cases = [data[:len(data) // 2], data[:-1], data[:3]]
        for _ in range(16):
            b = bytearray(data)
            k = rng.randrange(len(b))
            b[k] ^= 1 << rng.randrange(8)
            cases.append(bytes(b))
        for c in cases:
            try:
                z.uncompress(c)
                want = 0
            except z.ZippyError as e:
                want = e.code
            try:
                o.uncompress(c)
                oracle = 0
            except o.ZippyError as e:
                oracle = e.code
            assert oracle == want
            try:
                z.Index.build(c).close()
                got = 0
            except z.ZippyError as e:
                got = e.code
            assert got == want


def test_argument_checks():
    text = _text(300000, seed=14)
    data = z.compress(text, 1, z.dfZlib)
    for span in (0, 1000, 32767, 32769, 65536 + 1):
        with pytest.raises(z.ZippyError) as e:
            z.Index.build(data, z.dfZlib, span)
        assert e.value.code == ERR_ARG
    with pytest.raises(z.ZippyError) as e:
        z.Index.build(data, 7)
    assert e.value.code == ERR_INVALID_FORMAT
    idx = z.Index.build(data, z.dfZlib)
    with pytest.raises(z.ZippyError) as e:
        idx.extract(data[:-1], 0, 1)
    assert e.value.code == ERR_ARG
    with pytest.raises(z.ZippyError) as e:
        idx.extract(data, idx.size - 10, 11)
    assert e.value.code == ERR_ARG
    # another member of the same length: stored blocks of inputs of one length
    r1, r2 = (np.random.default_rng(s).integers(0, 256, 200000, dtype=np.uint8).tobytes() for s in (1, 2))
    m1, m2 = z.compress(r1, 0, z.dfZlib), z.compress(r2, 0, z.dfZlib)
    assert len(m1) == len(m2)
    stored = z.Index.build(m1, z.dfZlib)
    assert stored.extract(m1, 5, 10) == r1[5:15]
    with pytest.raises(z.ZippyError) as e:
        stored.extract(m2, 5, 10)
    assert e.value.code == ERR_ARG
    tail = bytearray(data)
    tail[-1] ^= 1   # only the trailer differs
    with pytest.raises(z.ZippyError) as e:
        idx.extract(bytes(tail), 0, 1)
    assert e.value.code == ERR_ARG
    fake = bytearray(data)
    fake[5] ^= 1
    with pytest.raises(z.ZippyError) as e:
        idx.extract(bytes(fake), 0, 1)
    assert e.value.code == ERR_ARG


def test_a_corrupt_interval_fails_only_its_ranges():
    text = _text(4 << 20, seed=16)
    data = z.compress(text, 1, z.dfZlib)
    idx = z.Index.build(data, z.dfZlib, 1 << 20)
    bad = bytearray(data)
    mid = len(bad) // 2
    bad[mid] ^= 0x10
    pts = idx.points
    bits = pts["bit"].astype(np.int64)
    outs = pts["out"].astype(np.int64)
    # the interval holding the flipped byte
    p = int(np.searchsorted(bits, mid * 8, side="right")) - 1
    lo = int(outs[p])
    hi = int(outs[p + 1]) if p + 1 < len(outs) else len(text)
    wins = [int(o) for o, w in zip(outs, pts["window"]) if w]
    # window interval [w, w_next) containing the flipped interval: its chain crosses it
    wlo = max(w for w in wins if w <= lo)
    ranges = [(0, 4096), (len(text) - 4096, 4096), (lo, hi - lo), (wlo, 10)]
    out, goff, st = idx.extract_batch(bytes(bad), [a for a, _ in ranges], [n for _, n in ranges])
    assert st[2] != 0
    for i, (a, n) in enumerate(ranges):
        if st[i] == 0:
            assert out[int(goff[i]):int(goff[i + 1])].tobytes() == text[a:a + n]
    far = [i for i, (a, n) in enumerate(ranges) if a + n <= wlo or a >= hi + (1 << 20)]
    for i in far:
        assert st[i] == 0


def test_two_threads_share_one_index():
    import threading
    text = _text(8 << 20, seed=17)
    data = z.compress(text, z.DefaultCompression, z.dfGzip)
    idx = z.Index.build(data, span=65536)
    errs = []

    def work(seed):
        try:
            ctx = z.Context()
            rng = random.Random(seed)
            offs = [rng.randrange(len(text) - 5000) for _ in range(200)]
            h = z.Index(idx._h, ctx)
            out, goff, st = h.extract_batch(data, offs, [5000] * 200)
            h._h = None   # borrowed handle
            assert (st == 0).all()
            for i, a in enumerate(offs):
                assert out[int(goff[i]):int(goff[i + 1])].tobytes() == text[a:a + 5000]
            ctx.close()
        except Exception as e:  # pragma: no cover - reported below
            errs.append(e)

    ts = [threading.Thread(target=work, args=(s,)) for s in (1, 2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


def test_member_of_more_than_4_gib():
    """A Default-level member of 4 GiB + 1 MiB: ranges that straddle output offset 2^32 and that reach the end."""
    tile = _text(1 << 20, seed=41)
    n = 4097
    data = z.compress(tile * n, z.DefaultCompression, z.dfGzip)
    ctx = z.Context()
    idx = z.Index.build(data, ctx=ctx)
    size = n << 20
    assert idx.size == size
    ranges = [(2 ** 32 - 5000, 10000), (2 ** 32 - 1, 2), (2 ** 32, 4096), (size - 70000, 70000), (size - 1, 1),
              (2 ** 32 - (3 << 20), 4 << 20)]
    out, goff, st = idx.extract_batch(data, [a for a, _ in ranges], [k for _, k in ranges])
    assert (st == 0).all()
    for i, (a, k) in enumerate(ranges):
        want = b"".join(tile[max(a, t << 20) - (t << 20):min(a + k, (t + 1) << 20) - (t << 20)]
                        for t in range(a >> 20, ((a + k - 1) >> 20) + 1))
        assert out[int(goff[i]):int(goff[i + 1])].tobytes() == want, (a, k)
