"""Per-member preset dictionaries (zb200_*_dicts, dictionaries= in Python): every member against its lone _dict /
plain call and against the stream-after-flush definition at windows 9..15, k_lz2's tokens against the windowed
schedule model, zlib's zdict in both directions, RFC 7692 context-takeover chains, whole-call errors, capacities,
scale through both host pipelines, the k = 1 case against the _dict calls, and C++ against Python."""
import os
import random
import subprocess
import zlib

import numpy as np
import pytest

from tests import deflate_tokens as dt
from tests import util
from tests.test_dictionaries_model import LEVELS as LZ_LEVELS, WINDOW_BITS, edge_case, wmodel  # noqa: F401
from tests.test_dictionary_rules import stored, window
from tests.test_gpu_lz2_model import encode

pytestmark = pytest.mark.gpu

LEVELS = [-2, 0, 1, -1, 2, 6, 9]
DLENS = [1, 100, 8191, 32768, 100000, 0]


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


@pytest.fixture(scope="module")
def text():
    return util.text_corpus(util.load_corpus())


def _abi(z, fn, *args):
    return getattr(z._native.lib(), fn)(*args)


def _zlib_head(n, d):
    cmf = (n - 8) << 4 | 8
    flg = 0x20 | (31 - ((cmf << 8) | 0x20) % 31) % 31
    return bytes([cmf, flg]) + zlib.adler32(d).to_bytes(4, "big")


def _after_flush(z, level, n, d, m):
    """The definition of a dictionary member's blocks: a raw compress stream of window n fed D, sync-flushed, then M."""
    cs = z.CompressStream(level, z.dfDeflate, window_bits=n)
    cs.write(d)
    cs.flush(z.SyncFlush)
    out = cs.write(m) + cs.finish()
    cs.close()
    return out


@pytest.fixture(scope="module")
def table(text):
    """Dictionaries of every length in DLENS, members, and per member a dictionary object (None, shared, own)."""
    rng = random.Random(7)
    dicts = [text[a:a + k] for a, k in ((rng.randrange(len(text) - 100001), k) for k in DLENS)]
    items, names = [], []
    for i, k in enumerate([0, 1, 100, 4095, 65535, 65537, 70000, 3000, 20000, 5000, 40000, 12345, 1, 999]):
        a = rng.randrange(len(text) - k - 1)
        items.append(text[a:a + k] if i % 5 else bytes(rng.randrange(4) for _ in range(k)))
    # members with none, members sharing entries (the same object), members with their own (an equal copy)
    names = [None, 0, 0, 1, 2, 2, 3, 4, 5, None, 3, 4, 1, 5]
    objs = [None if j is None else dicts[j] for j in names]
    objs[10] = bytes(bytearray(dicts[3]))    # own entry, equal bytes
    items[7] = dicts[4][-3000:][:1000] + items[7][1000:]    # matches straight into W
    return dicts, items, objs


def _member_want(z, level, fmt, n, d, m):
    if not d:
        return z.compress_batch([m], level, fmt, window_bits=n)[0]
    if n == 15:
        return z.compress_batch([m], level, fmt, dictionary=d)[0]
    blocks = _after_flush(z, level, n, d, m) if level not in (0, 1, -2) else \
        z.compress_batch([m], level, z.dfDeflate, window_bits=n)[0]
    if fmt == z.dfDeflate:
        return blocks
    return _zlib_head(n, d) + blocks + zlib.adler32(m).to_bytes(4, "big")


# ---------------------------------------------------------------------- 1. the definition, member by member
@pytest.mark.parametrize("n", WINDOW_BITS)
def test_members_follow_the_definition(z, table, n):
    dicts, items, objs = table
    rng = random.Random(n)
    for fmt in (z.dfZlib, z.dfDeflate):
        wb = n if fmt == z.dfZlib else -n
        for level in LEVELS:
            got = z.compress_batch(items, level, fmt, window_bits=n, dictionaries=objs)
            for i, (m, d) in enumerate(zip(items, objs)):
                d = d or b""
                assert got[i] == _member_want(z, level, fmt, n, d, m), (fmt, level, n, i)
                assert zlib.decompressobj(wb, zdict=d).decompress(got[i]) == m if d else \
                    zlib.decompressobj(wb).decompress(got[i]) == m
            assert z.uncompress_batch(got, fmt, dictionaries=objs) == items
            sizes, st = z.uncompressed_sizes(got, fmt, dictionaries=objs)
            assert (st == 0).all() and list(sizes) == [len(m) for m in items]
            # the batch does not change a member: shuffled, and with every shared entry split into copies
            perm = list(range(len(items)))
            rng.shuffle(perm)
            sh = z.compress_batch([items[p] for p in perm], level, fmt, window_bits=n,
                                  dictionaries=[objs[p] for p in perm])
            assert [sh[perm.index(i)] for i in range(len(items))] == got
            split = [None if d is None else bytes(bytearray(d)) for d in objs]
            assert z.compress_batch(items, level, fmt, window_bits=n, dictionaries=split) == got


# ---------------------------------------------------------------------- 2. tokens under a window
@pytest.mark.parametrize("n", WINDOW_BITS)
def test_kernel_tokens_equal_the_windowed_model(z, wmodel, n):  # noqa: F811
    d, m = edge_case(n)
    w = window(d)
    for level in LZ_LEVELS:
        c = z.compress_batch([m], level, z.dfDeflate, window_bits=n, dictionaries=[d])[0]
        got = dt.member_chunks(dt.parse(stored(w) + c)[1:])
        want, _ = wmodel.member(w, m, level, n)
        assert len(got) == len(want), (n, level)
        compared = 0
        for k, (g, wt) in enumerate(zip(got, want)):
            if g.btype == 0:
                continue
            compared += 1
            assert np.array_equal(encode(g.tokens), wt), (n, level, k)
        assert compared >= 1
        dists = [t[1] for g in got if g.btype != 0 for t in g.tokens if not isinstance(t, int)]
        assert max(dists) == 1 << n, (n, level)


# ---------------------------------------------------------------------- 3. zlib in both directions
def _zlib_member(level, wb, d, m, rng):
    co = zlib.compressobj(level, zlib.DEFLATED, wb, zdict=d) if d else zlib.compressobj(level, zlib.DEFLATED, wb)
    out, pos = [], 0
    while pos < len(m):
        k = rng.choice((100, 5000, 40000))
        out.append(co.compress(m[pos:pos + k]))
        out.append(co.flush(rng.choice((zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH, zlib.Z_NO_FLUSH))))
        pos += k
    out.append(co.flush())
    return b"".join(out)


@pytest.mark.parametrize("n", [9, 12, 15])
def test_decodes_zlib_zdict_members(z, table, n):
    dicts, items, objs = table
    rng = random.Random(100 + n)
    for fmt, wb in ((z.dfZlib, n), (z.dfDeflate, -n)):
        comp, names, want = [], [], []
        for i, (m, d) in enumerate(zip(items, objs)):
            comp.append(_zlib_member(rng.choice((1, 6, 9)), wb, d, m, rng))
            names.append(d)
            want.append(m)
        if fmt == z.dfZlib:
            x = items[3]
            comp += [zlib.compress(x, 6), _zlib_member(6, n, dicts[2], x, rng), _zlib_member(6, n, dicts[2], x, rng),
                     _zlib_member(6, 31, None, x, rng)]
            names += [dicts[1], None, dicts[3], dicts[2]]   # no FDICT; FDICT named -1; the wrong dictionary; gzip
            want += [x, 13, 23, x]
        fmt_call = z.dfDetect if fmt == z.dfZlib else fmt
        back = z.uncompress_batch(comp, fmt_call, dictionaries=names)
        assert [r if isinstance(r, bytes) else r.code for r in back] == want, (fmt, n)
        sizes, st = z.uncompressed_sizes(comp, fmt_call, dictionaries=names)
        for s, t, w_ in zip(sizes, st, want):
            assert (t == 0 and s == len(w_)) if isinstance(w_, bytes) else t == w_
        # corrupted members: each one's verdict is its lone _dict / plain call's
        bad = []
        for c in comp:
            b = bytearray(c)
            b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
            bad.append(bytes(b) if rng.random() < 0.7 else bytes(b[:rng.randrange(len(b))]))
        got = z.uncompress_batch(bad, fmt_call, dictionaries=names)
        for b, d, g in zip(bad, names, got):
            lone = z.uncompress_batch([b], fmt_call, dictionary=d)[0]
            assert (g if isinstance(g, bytes) else g.code) == (lone if isinstance(lone, bytes) else lone.code)


# ---------------------------------------------------------------------- 4. RFC 7692 context takeover
@pytest.mark.parametrize("n", [10, 15])
def test_context_takeover_chains(z, text, n):
    rng = random.Random(n)
    conns = [[text[o:o + k] for o, k in ((rng.randrange(200000), rng.choice((5, 200, 3000, 20000))) for _ in range(6))]
             for _ in range(8)]
    msgs, dicts = [], []
    for c in conns:
        seen = b""
        for m in c:
            msgs.append(m)
            dicts.append(seen[-(1 << n):] or None)
            seen += m
    for level in (1, 6, -1):
        comp = z.compress_batch(msgs, level, z.dfDeflate, window_bits=n, dictionaries=dicts)
        for m, d, c in zip(msgs, dicts, comp):
            do = zlib.decompressobj(-n, zdict=d) if d else zlib.decompressobj(-n)
            assert do.decompress(c) == m
        assert z.uncompress_batch(comp, z.dfDeflate, dictionaries=dicts) == msgs
    # a chain zlib wrote: one raw stream per connection, a sync flush per message (an empty final block appended)
    wire = []
    for c in conns:
        co = zlib.compressobj(6, zlib.DEFLATED, -n)
        for m in c:
            wire.append(co.compress(m) + co.flush(zlib.Z_SYNC_FLUSH) + b"\x03\x00")
    assert z.uncompress_batch(wire, z.dfDeflate, dictionaries=dicts) == msgs


# ---------------------------------------------------------------------- 5. arguments and capacity
def _call(z, items, fmt, dict_list, of, level=6, n=15, cap=None, offs_override=None):
    ctx = z.default_context()
    base, offs = z._pack(items)
    db, do = z._pack(dict_list)
    if offs_override is not None:
        do = np.array(offs_override, np.uint64)
    of = np.array(of, np.int32)
    L = z._native.lib()
    bound = sum(int(L.zb200_compress_bound(len(x), fmt)) + 4 for x in items)
    out = np.zeros(bound + 64, np.uint8)
    oo = np.zeros(len(items) + 1, np.uint64)
    st = np.full(len(items), 77, np.int32)
    rc = _abi(z, "zb200_compress_batch_dicts", ctx._h, base.ctypes.data, offs.ctypes.data, len(items), level, fmt, n,
              db.ctypes.data, do.ctypes.data, len(do) - 1, of.ctypes.data, out.ctypes.data,
              bound if cap is None else cap, oo.ctypes.data, st.ctypes.data)
    return rc, st, [bytes(out[int(oo[i]):int(oo[i + 1])]) for i in range(len(items))] if rc == 0 else None


def test_whole_call_errors_leave_statuses(z, text):
    items = [text[:1000], text[1000:3000]]
    ds = [text[5000:9000], b""]
    for of in ([0, 2], [-2, 0]):
        rc, st, _ = _call(z, items, z.dfZlib, ds, of)
        assert rc == 22 and (st == 77).all()
    rc, st, _ = _call(z, items, z.dfZlib, ds, [0, 1], offs_override=[0, 4000, 3000])
    assert rc == 22 and (st == 77).all()
    rc, st, _ = _call(z, items, z.dfGzip, ds, [-1, 0])
    assert rc == 2 and (st == 77).all()
    rc, st, _ = _call(z, items, z.dfGzip, ds, [1, -1])     # only an empty dictionary named: a plain gzip call
    assert rc == 0
    rc, st, _ = _call(z, items, z.dfZlib, ds, [0, 1], n=7)
    assert rc == 22 and (st == 77).all()
    # decode side
    comp = z.compress_batch(items, 6, z.dfZlib, dictionaries=[ds[0], None])
    cb, co = z._pack(comp)
    db, do = z._pack(ds)
    for of in ([0, 2], [-2, 0]):
        o = np.array(of, np.int32)
        sizes = np.zeros(2, np.uint64)
        st = np.full(2, 77, np.int32)
        assert _abi(z, "zb200_uncompress_sizes_dicts", z.default_context()._h, cb.ctypes.data, co.ctypes.data, 2,
                    z.dfZlib, db.ctypes.data, do.ctypes.data, 2, o.ctypes.data, sizes.ctypes.data, st.ctypes.data) == 22
        assert (st == 77).all()
    # an empty table (k = 0) names nothing: any entry >= 0 is out of range, on both sides
    nothing = np.zeros(1, np.uint64)
    for of in ([0, -1], [-1, 0]):
        o = np.array(of, np.int32)
        sizes = np.zeros(2, np.uint64)
        st = np.full(2, 77, np.int32)
        assert _abi(z, "zb200_uncompress_sizes_dicts", z.default_context()._h, cb.ctypes.data, co.ctypes.data, 2,
                    z.dfZlib, db.ctypes.data, nothing.ctypes.data, 0, o.ctypes.data, sizes.ctypes.data,
                    st.ctypes.data) == 22
        assert (st == 77).all()
        rc, st, _ = _call(z, items, z.dfZlib, [], of)
        assert rc == 22 and (st == 77).all()
    rc, st, got = _call(z, items, z.dfZlib, [], [-1, -1])
    assert rc == 0 and got == z.compress_batch(items, 6, z.dfZlib)
    # a null dict_of with members, and decreasing offsets with no members, fail on both sides
    out = np.zeros(16, np.uint8)
    lens = np.zeros(2, np.uint64)
    st = np.full(2, 77, np.int32)
    dofs = np.zeros(3, np.uint64)
    assert _abi(z, "zb200_uncompress_batch_dicts", z.default_context()._h, cb.ctypes.data, co.ctypes.data, 2,
                z.dfZlib, db.ctypes.data, nothing.ctypes.data, 0, None, out.ctypes.data, dofs.ctypes.data,
                lens.ctypes.data, st.ctypes.data) == 22
    assert (st == 77).all()
    bad = np.array([0, 4000, 3000], np.uint64)
    for fn, args in (("zb200_uncompress_batch_dicts", (None, out.ctypes.data, dofs.ctypes.data, lens.ctypes.data,
                                                       st.ctypes.data)),
                     ("zb200_uncompress_sizes_dicts", (None, lens.ctypes.data, st.ctypes.data))):
        assert _abi(z, fn, z.default_context()._h, cb.ctypes.data, co.ctypes.data, 0, z.dfZlib, db.ctypes.data,
                    bad.ctypes.data, 2, *args) == 22
    with pytest.raises(z.ZippyError):
        z.compress_batch(items, 6, z.dfZlib, dictionary=ds[0], dictionaries=[None, None])
    with pytest.raises(z.ZippyError):
        z.uncompress_batch(comp, z.dfZlib, dictionary=ds[0], dictionaries=[None, None])


def test_exact_bounds(z, text):
    L = z._native.lib()
    rng = random.Random(3)
    ds = [text[:32768], rng.randbytes(100)]
    for fmt in (z.dfZlib, z.dfDeflate):
        for x in (rng.randbytes(70000), text[40000:40000 + 5000], b""):
            for of in ([0], [1], [-1]):
                for level in (0, 6):
                    cap = int(L.zb200_compress_bound(len(x), fmt)) + (4 if fmt == z.dfZlib and of[0] >= 0 else 0)
                    rc, _, got = _call(z, [x], fmt, ds, of, level=level, cap=cap)
                    assert rc == 0 and len(got[0]) <= cap
                    exact = len(got[0])
                    assert _call(z, [x], fmt, ds, of, level=level, cap=exact)[0] == 0
                    assert _call(z, [x], fmt, ds, of, level=level, cap=exact - 1)[0] == 19


# ---------------------------------------------------------------------- 6. scale
@pytest.mark.parametrize("gated", ["0", "1"])
@pytest.mark.parametrize("group", ["1", "3"])
def test_distinct_dictionaries_at_scale(z, text, gated, group, monkeypatch):
    monkeypatch.setenv("ZB200_UNC_GATED", gated)
    monkeypatch.setenv("ZB200_GROUP_CHUNKS", group)
    ctx = z.Context()
    try:
        # uneven lengths: a member's first chunk may sit at any address modulo 16, and each of the k = n / 4
        # dictionaries is named by members in different launch groups, so several aligned copies of one window go up
        # in different groups
        n, k = 65536, 16384
        rng = np.random.default_rng(11)
        tarr = np.frombuffer(text, np.uint8)
        lens = rng.integers(700, 1400, n)
        starts = rng.integers(0, len(text) - 32768, k)
        dicts = [tarr[s:s + 32768].tobytes() for s in starts]
        names = [dicts[i % k] for i in range(n)]
        base = np.concatenate([tarr[starts[i % k] + 30000:starts[i % k] + 30000 + lens[i]] for i in range(n)])
        offs = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(lens, out=offs[1:])
        comp, co = ctx.compress_batch(base, offs, -1, z.dfZlib, window_bits=15, dictionaries=names)
        for i in list(range(0, n, 4099)) + list(range(1, 17)):
            m, c = bytes(base[int(offs[i]):int(offs[i + 1])]), bytes(comp[int(co[i]):int(co[i + 1])])
            assert zlib.decompressobj(15, zdict=names[i]).decompress(c) == m
            assert c == ctx.compress_batch(np.frombuffer(m, np.uint8), np.array([0, len(m)], np.uint64), -1, z.dfZlib,
                                           dictionary=names[i])[0].tobytes()
        # the group boundaries change nothing: the same bytes as a context with the default groups
        monkeypatch.delenv("ZB200_GROUP_CHUNKS")
        ref_ctx = z.Context()
        try:
            rcomp, rco = ref_ctx.compress_batch(base, offs, -1, z.dfZlib, dictionaries=names)
        finally:
            ref_ctx.close()
        assert np.array_equal(rco, co) and np.array_equal(rcomp, comp)
        sizes, st = ctx.uncompressed_sizes(comp, co, z.dfZlib, dictionaries=names)
        assert (st == 0).all() and np.array_equal(sizes, lens)
        out, do, got_lens, st = ctx.uncompress_batch(comp, co, z.dfZlib, dictionaries=names)
        assert (st == 0).all() and np.array_equal(got_lens, lens) and np.array_equal(out, base)
    finally:
        ctx.close()


# ---------------------------------------------------------------------- 7. one path
def test_dict_calls_are_the_k1_case(z, table):
    """The _dict calls and a k = 1 table give the same bytes and verdicts.  Both run the same table path, so this pins
    the entry points' argument mapping, not the definition: tests/test_gpu_dictionary.py anchors the k = 1 bytes."""
    dicts, items, _ = table
    for d in dicts:
        for fmt in (z.dfZlib, z.dfDeflate):
            for level in LEVELS:
                old = z.compress_batch(items, level, fmt, dictionary=d)
                new = z.compress_batch(items, level, fmt, dictionaries=[d] * len(items))
                assert old == new, (len(d), fmt, level)
            comp = old + [b"\x78\x20\0\0\0\0\x03\0\0\0\0\1", b"\x00\x01", b""]
            a = z.uncompress_batch(comp, fmt, dictionary=d)
            b = z.uncompress_batch(comp, fmt, dictionaries=[d] * len(comp))
            assert [r if isinstance(r, bytes) else r.code for r in a] == [r if isinstance(r, bytes) else r.code for r in b]


# ---------------------------------------------------------------------- 8. C++
def test_cpp_equals_python(z, table, tmp_path):
    dicts, items, objs = table
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "cpp_dicts_test")
    libdir = os.path.join(root, "zippy_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(root, "tests", "native", "cpp_dicts_test.cpp"),
                           "-L" + libdir, "-l:libzippy_b200.so", "-Wl,-rpath," + libdir])
    of = [-1 if d is None else dicts.index(d) for d in objs]   # (an own copy names the equal entry)

    def blob(parts):
        return b"".join(len(p).to_bytes(8, "little") + p for p in parts)

    for fmt, level, n in ((z.dfZlib, 6, 15), (z.dfDeflate, -1, 10), (z.dfZlib, 9, 12)):
        py = z.compress_batch(items, level, fmt, window_bits=n, dictionaries=objs)
        (tmp_path / "items").write_bytes(blob(items))
        (tmp_path / "dicts").write_bytes(blob(dicts))
        (tmp_path / "of").write_bytes(np.array(of, np.int32).tobytes())
        (tmp_path / "py").write_bytes(blob(py))
        subprocess.check_call([exe, str(tmp_path / "items"), str(tmp_path / "dicts"), str(tmp_path / "of"), str(level),
                               str(fmt), str(n), str(tmp_path / "py"), str(tmp_path / "cpp")])
        assert (tmp_path / "cpp").read_bytes() == blob(py)
