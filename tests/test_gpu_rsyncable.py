"""Rsyncable compression on the GPU (zb_rsync.cu; zb200_rsyncable_chunks and the _rsyncable compress calls).

The kernel's chunk starts equal tests/native/rsync_model.c's on edge lengths, the corpus, random, constant and
periodic data, planted candidates around every kernel boundary, every source offset mod 16 and a member over 4 GiB.
The members hold one block (or stored run) per model chunk, inflate everywhere, and do not depend on their batch, the
device call or their address.  An edit changes only the compressed bytes near it.
"""
import ctypes
import os
import random
import subprocess
import zlib

import numpy as np
import pytest

import zippy_b200 as z
from zippy_b200 import _native
from oracle import oracle as o
from tests import deflate_tokens as dt
from tests import util
from tests.test_rsyncable_model import CHUNK, MIN, build_model, cap_bound, plant, rule_cuts

pytestmark = pytest.mark.gpu

TILE = 16384          # k_rsync_cand's tile
RUN = 128             # positions per lane in a tile
WBITS = {z.dfGzip: 31, z.dfZlib: 15, z.dfDeflate: -15}
HEAD = {z.dfGzip: 10, z.dfZlib: 2, z.dfDeflate: 0}
TAIL = {z.dfGzip: 8, z.dfZlib: 4, z.dfDeflate: 0}
FL = 3                # gzip FNAME letters of every gzip member here


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return build_model(tmp_path_factory)


@pytest.fixture(scope="module")
def corpus():
    return util.load_corpus()


def _same(model, items):
    got = z.rsyncable_chunks(items)
    for i, (b, g) in enumerate(zip(items, got)):
        want = model.chunks(b)
        assert np.array_equal(g, want), (i, len(b), g[:8], want[:8])


def test_edge_lengths_corpus_and_random(model, corpus):
    rng = random.Random(1)
    lens = [0, 1, 63, 64, 65, MIN - 1, MIN, MIN + 1, 65535, 65536, 65537]
    items = [rng.randbytes(n) for n in lens] + list(corpus.values()) + [rng.randbytes(4 << 20),
                                                                        util.text_corpus(corpus)]
    _same(model, items)
    _same(model, items[::-1])           # mixed lengths in another order
    for x in items:                     # and alone
        _same(model, [x])


def test_constant_and_periodic(model):
    _same(model, [bytes([b]) * 150000 for b in range(256)])
    rng = random.Random(2)
    _same(model, [(rng.randbytes(p) * (300000 // p + 1))[:300000] for p in range(1, 101)])


def _planted(n, positions, seed):
    b = bytearray(random.Random(seed).randbytes(n))
    for p in positions:
        plant(b, p)
    return bytes(b)


def test_planted_candidates(model):
    items = []
    # at MIN exactly, at L - 1, and 1 byte closer than MIN to another
    items.append(_planted(100000, [MIN, 99999], 10))
    items.append(_planted(100000, [MIN + 100, 2 * MIN + 99], 11))
    items.append(_planted(100000, [MIN + 100, 2 * MIN + 100], 12))
    # around every tile boundary and lane run of the kernel, and pairs across a tile boundary MIN and MIN - 1 apart
    for k in range(1, 6):
        for d in (-3, -1, 0, 1, 2, 63, 64, 65):
            items.append(_planted(6 * TILE, [k * TILE + d], 100 * k + d + 50))
        for j in (1, 31, 32, 64, 127):
            items.append(_planted(6 * TILE, [k * TILE + j * RUN - 1, k * TILE + j * RUN], 1000 * k + j))
    for a in (TILE - 1, TILE + 5, 2 * TILE - 1):
        for gap in (MIN - 1, MIN, MIN + 1):
            items.append(_planted(8 * TILE, [a, a + gap], a + gap))
    # dense candidates, one every 40 bytes: no cut at all
    items.append(_planted(4 * TILE, range(3, 4 * TILE, 40), 77))
    for b in items:
        assert len(b) >= 3
    _same(model, items)


def test_source_offsets_mod_16(model, corpus):
    rng = random.Random(4)
    x = rng.randbytes(300000)
    want = model.chunks(x)
    ctx = z.default_context()
    for k in range(16):
        base = np.frombuffer(bytes(k) + x + bytes(5), dtype=np.uint8)
        got = ctx.rsyncable_chunks(base, [k, k + len(x)])
        assert np.array_equal(got[0], want), k


def test_member_over_4_gib(model):
    rng = np.random.default_rng(9)
    piece = rng.integers(0, 256, 64 << 20, dtype=np.uint8)
    n = (4 << 30) + (1 << 20)
    buf = np.empty(n + 5, dtype=np.uint8)
    for off in range(0, n, len(piece)):
        m = min(len(piece), n - off)
        buf[off:off + m] = piece[:m]
        piece[rng.integers(0, len(piece), 64)] ^= 0x5a     # each repeat differs a little
    buf[n:] = 7
    got = z.default_context().rsyncable_chunks(buf, [0, n])[0]
    out = np.zeros(cap_bound(n), dtype=np.uint64)
    cnt = model.L.rs_model_chunks(buf.ctypes.data_as(ctypes.c_char_p), n, out.ctypes.data, out.size)
    assert np.array_equal(got, out[:cnt])
    assert got[-1] > (1 << 32)
    del buf


# ---- layout -------------------------------------------------------------------------------------------------------
def split_chunks(blocks, lengths):
    """The member's blocks, split by the chunk lengths they should stand for: a coded chunk is one block of that
    size, followed unless it is the last by the empty stored joint; a stored chunk is stored blocks that add up to
    it (of at most 65535 bytes each).  -> per chunk, its block types."""
    out, i = [], 0
    for k, ln in enumerate(lengths):
        last = k == len(lengths) - 1
        b = blocks[i]
        if b.btype != 0:
            assert b.size() == ln, (k, b.size(), ln)
            assert b.final == last
            i += 1
            if not last:
                j = blocks[i]
                assert j.btype == 0 and not j.tokens and not j.final, k
                i += 1
            out.append(b.btype)
            continue
        got = 0
        while True:
            b = blocks[i]
            assert b.btype == 0 and len(b.tokens) <= 65535
            got += len(b.tokens)
            i += 1
            if got >= ln:
                break
        assert got == ln and blocks[i - 1].final == last, (k, got, ln)
        out.append(0)
    assert i == len(blocks)
    return out


def _layout_input(corpus):
    rng = random.Random(21)
    T = util.text_corpus(corpus)
    b = bytearray(T[:700000] + rng.randbytes(300000) + bytes(200000) + T[900000:1300000])
    for p in (MIN, 5 * MIN + 3, 700000 + 2 * MIN, 1000000 + MIN + 1, len(b) - 1):
        plant(b, p)
    return bytes(b)


@pytest.mark.parametrize("level", [0, -2, 1, 6, 9])
def test_layout_equals_the_model(model, corpus, level):
    x = _layout_input(corpus)
    st = model.chunks(x).astype(np.int64)
    lengths = np.diff(np.append(st, len(x))).tolist()
    assert len(lengths) > (len(x) + CHUNK - 1) // CHUNK   # the content moved the grid
    for fmt in (z.dfGzip, z.dfZlib, z.dfDeflate):
        m = z.compress_batch([x], level, fmt, fname_lens=[FL], rsyncable=True)[0]
        assert zlib.decompress(m, WBITS[fmt]) == x
        assert o.uncompress(m, fmt) == x
        assert z.uncompress(m, fmt) == x
        head = HEAD[fmt] + (FL + 1 if fmt == z.dfGzip else 0)
        kinds = split_chunks(dt.parse(m[head:len(m) - TAIL[fmt]]), lengths)
        if level == 0:
            assert set(kinds) == {0}


def test_every_level_and_empty_members():
    items = [b"", b"a", bytes(70000), random.Random(3).randbytes(200000)]
    for level in (0, -2, 1, -1, 2, 3, 4, 5, 6, 7, 8, 9):
        for fmt in (z.dfGzip, z.dfZlib, z.dfDeflate):
            for x, m in zip(items, z.compress_batch(items, level, fmt, rsyncable=True)):
                assert zlib.decompress(m, WBITS[fmt]) == x, (level, fmt, len(x))
        assert z.uncompress(z.compress(items[3], level, z.dfZlib, rsyncable=True)) == items[3]
        assert zlib.decompress(z.deflate(items[3], level, rsyncable=True), -15) == items[3]


# ---- independence -------------------------------------------------------------------------------------------------
def test_member_bytes_do_not_depend_on_batch_device_or_offset(corpus):
    import torch
    x = _layout_input(corpus)[:900000]
    others = [b"q" * 1000, random.Random(8).randbytes(150000), corpus["html"]]
    for level in (0, 1, 6):
        for fmt in (z.dfGzip, z.dfDeflate):
            alone = z.compress_batch([x], level, fmt, fname_lens=[FL], rsyncable=True)[0]
            batch = z.compress_batch(others + [x], level, fmt, fname_lens=[FL] * 4, rsyncable=True)[3]
            assert batch == alone
            ctx = z.default_context()
            for k in range(16):
                base = np.frombuffer(bytes(k) + x + bytes(3), dtype=np.uint8)
                out, oo = ctx.compress_batch(base, [k, k + len(x)], level, fmt, [FL], rsyncable=True)
                assert out[:int(oo[1])].tobytes() == alone, k
            cap = _native.lib().zb200_compress_bound_rsyncable(len(x), fmt) + 64
            for k in (0, 5, 13):
                src = torch.tensor(np.frombuffer(bytes(k) + x, dtype=np.uint8), device="cuda")
                dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
                oo = ctx.compress_batch_device(src.data_ptr(), [k, k + len(x)], level, fmt, dst.data_ptr(), cap,
                                               fname_lens=[FL], rsyncable=True)
                assert dst[:int(oo[1])].cpu().numpy().tobytes() == alone, k


# ---- locality -----------------------------------------------------------------------------------------------------
def _mix(corpus, n, seed):
    rng = random.Random(seed)
    T = util.text_corpus(corpus)
    parts, size = [], 0
    while size < n:
        if rng.random() < 0.7:
            a = rng.randrange(len(T) - 400000)
            p = T[a:a + rng.randrange(50000, 400000)]
        else:
            p = rng.randbytes(rng.randrange(20000, 200000))
        parts.append(p)
        size += len(p)
    return b"".join(parts)[:n]


def _out_before(comp, n):
    """How many bytes the first n bytes of a raw member decode to."""
    return len(zlib.decompressobj(-15).decompress(comp[:n]))


def _first_prefix_reaching(comp, want):
    """The shortest prefix of a raw member that decodes to at least `want` bytes."""
    lo, hi = 0, len(comp)
    while lo < hi:
        mid = (lo + hi) // 2
        if _out_before(comp, mid) >= want:
            hi = mid
        else:
            lo = mid + 1
    return lo


def _chunk_start(comp, s):
    """The byte offset in a raw member at which the chunk starting at input position s starts: just past the joint
    (00 00 ff ff) behind the chunk before it, or where the stored chunk before it ends."""
    x = _first_prefix_reaching(comp, s)   # the chunk before it has decoded; its end-of-block code and joint follow
    j = comp.find(b"\x00\x00\xff\xff", max(0, x - 8), x + 8)
    return j + 4 if j >= 0 else x


def _common_prefix(a, b):
    n = min(len(a), len(b))
    x = np.frombuffer(a[:n], dtype=np.uint8) != np.frombuffer(b[:n], dtype=np.uint8)
    return int(np.argmax(x)) if x.any() else n


def _common_suffix(a, b):
    return _common_prefix(a[::-1], b[::-1])


@pytest.fixture(scope="module")
def locality_input(corpus):
    return _mix(corpus, 24 << 20, 31)


def _edits(base):
    rng = random.Random(6)
    e = 9_000_000 + 777
    yield "insert", e, e, base[:e] + b"~inserted~" + base[e:]
    yield "delete", e, e + 4000, base[:e] + base[e + 4000:]
    yield "overwrite", e, e + 300, base[:e] + rng.randbytes(300) + base[e + 300:]
    yield "prepend", 0, 0, rng.randbytes(7) + base


@pytest.mark.parametrize("level", [0, 1, 6, 9])
def test_an_edit_changes_only_nearby_bytes(model, locality_input, level):
    base = locality_input
    lz = level not in (0, 1)
    old = z.compress_batch([base], level, z.dfDeflate, rsyncable=True)[0]
    old_st = model.chunks(base).astype(np.int64)
    for name, e, old_end, new in _edits(base):
        new_end = old_end + len(new) - len(base)
        delta = len(new) - len(base)
        comp = z.compress_batch([new], level, z.dfDeflate, rsyncable=True)[0]
        assert zlib.decompress(comp, -15) == new
        new_st = model.chunks(new).astype(np.int64)
        # chunks that end before the edit: their compressed bytes are the common prefix
        ends = np.append(old_st[1:], len(base))
        kept = int(ends[ends <= e].max()) if (ends <= e).any() else 0
        assert _out_before(old[:_common_prefix(old, comp)], len(old)) >= kept, name
        # the first cut at which the inputs agree again; at the LZ levels also past 32 KiB of history
        cuts = rule_cuts(model.candidates(new))
        c = int(cuts[cuts >= new_end + MIN + 64][0])
        s = int(new_st[(new_st >= c) & ((new_st - 32768 >= new_end) if lz else True)][0])
        assert s - delta in set(old_st.tolist()), name
        suffix = _common_suffix(old, comp)
        assert _chunk_start(comp, s) >= len(comp) - suffix, (name, s, suffix)
        assert s - new_end < (512 << 10), name
    # control: the plain grid shifts with an insertion and almost nothing after it stays the same
    ins = next(_edits(base))[3]
    a = z.compress_batch([base], level, z.dfDeflate)[0]
    b = z.compress_batch([ins], level, z.dfDeflate)[0]
    assert _common_suffix(a, b) < len(a) // 100


# ---- bound, decode path, refusals ---------------------------------------------------------------------------------
def test_bound():
    n = 4 << 20
    b = bytearray(random.Random(12).randbytes(n))
    for p in range(MIN, n, MIN):
        plant(b, p)
    L = _native.lib()
    for fmt in (z.dfGzip, z.dfZlib, z.dfDeflate):
        m = z.compress_batch([bytes(b)], 6, fmt, fname_lens=[25], rsyncable=True)[0]
        assert zlib.decompress(m, WBITS[fmt]) == b
        assert L.zb200_compress_bound(n, fmt) < len(m) <= L.zb200_compress_bound_rsyncable(n, fmt)


def test_decode_path_through_joint_segments(corpus, monkeypatch):
    """A large rsyncable member's segments are not 64 KiB apart: the optimistic pass fails and one count pass
    sizes them (the launch count of tests/test_gpu_joint_segments.py)."""
    from tests.test_gpu_joint_segments import BASE, PER_WINDOW, _ctx, _one
    raw = _mix(corpus, 6_000_000, 41)
    ctx = _ctx(z, monkeypatch)
    seen = {}
    for level in (z.DefaultCompression, 1):
        for fmt in (z.dfGzip, z.dfZlib, z.dfDeflate):
            blob = ctx.compress_batch(np.frombuffer(raw, dtype=np.uint8), [0, len(raw)], level, fmt, [FL],
                                      rsyncable=True)
            got, st, launches = _one(ctx, blob[0][:int(blob[1][1])].tobytes(), fmt)
            assert st == 0 and got == raw, (level, fmt, st)
            seen[(level, fmt)] = launches
        plain = ctx.compress_batch(np.frombuffer(raw, dtype=np.uint8), [0, len(raw)], level, z.dfGzip, [FL])
        got, st, launches = _one(ctx, plain[0][:int(plain[1][1])].tobytes(), z.dfGzip)
        assert st == 0 and got == raw
        seen[(level, "plain")] = launches
    print("decode launches", seen)
    for fmt in (z.dfGzip, z.dfZlib, z.dfDeflate):
        # past the optimistic pass, a count pass and the window's marker decode and resolve ran: the member decoded
        # as segments at its joints, not serially
        assert seen[(z.DefaultCompression, fmt)] >= BASE + 1 + PER_WINDOW, seen
    ctx.close()


def test_refusals():
    x = b"hello rsyncable" * 1000
    bad = [dict(dictionary=b"hello"), dict(dictionaries=[b"hello"]), dict(index_span=1 << 20),
           dict(strategy=z.StrategyFiltered), dict(window_bits=12), dict(optimal=True)]
    ctx = z.default_context()
    for kw in bad:
        with pytest.raises(z.ZippyError) as e:
            ctx.compress_batch(np.frombuffer(x, dtype=np.uint8), [0, len(x)], 6, z.dfZlib, rsyncable=True, **kw)
        assert e.value.code == 22, kw
    with pytest.raises(z.ZippyError) as e:
        z.compress(x, 6, z.dfZlib, dictionary=b"hello", rsyncable=True)
    assert e.value.code == 22
    with pytest.raises(z.ZippyError) as e:
        z.default_context().compress_batch_device(0, [0, 0], 6, z.dfZlib, 0, 0, window_bits=10, rsyncable=True)
    assert e.value.code == 22
    # the C calls check their arguments before they touch statuses
    L = _native.lib()
    st = np.full(1, 1234, dtype=np.int32)
    offs = np.array([0, len(x)], dtype=np.uint64)
    out = np.zeros(L.zb200_compress_bound_rsyncable(len(x), z.dfZlib), dtype=np.uint8)
    oo = np.zeros(2, dtype=np.uint64)
    src = np.frombuffer(x, dtype=np.uint8)
    h = z.default_context()._h
    for level, fmt in ((10, z.dfZlib), (6, 7)):
        rc = L.zb200_compress_batch_rsyncable(h, src.ctypes.data, offs.ctypes.data, 1, level, fmt, None,
                                              out.ctypes.data, out.size, oo.ctypes.data, st.ctypes.data)
        assert rc != 0 and st[0] == 1234


def test_flag_off_is_unchanged(corpus):
    x = corpus["alice29.txt"]
    for level in (0, 1, 6):
        assert z.compress_batch([x], level, z.dfZlib) == z.compress_batch([x], level, z.dfZlib, rsyncable=False)


def test_tarball_gzip_hook(corpus, tmp_path):
    import tarfile
    from zippy_b200.tarballs import create_tarball
    src = tmp_path / "src"
    src.mkdir()
    (src / "a.txt").write_bytes(corpus["alice29.txt"])
    (src / "r.bin").write_bytes(random.Random(13).randbytes(100000))
    create_tarball(str(src), str(tmp_path / "t.tar.gz"), gzip=lambda b: z.compress(b, rsyncable=True))
    with tarfile.open(tmp_path / "t.tar.gz") as t:
        assert sorted(m.name.split("/")[-1] for m in t.getmembers() if m.isfile()) == ["a.txt", "r.bin"]


def test_cpp_rsyncable(corpus, tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "cpp_rsyncable_test")
    libdir = os.path.join(root, "zippy_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe,
                           os.path.join(root, "tests", "native", "cpp_rsyncable_test.cpp"),
                           "-L" + libdir, "-l:libzippy_b200.so", "-Wl,-rpath," + libdir])
    data = corpus["lcet10.txt"]
    inp = tmp_path / "in.bin"
    inp.write_bytes(data)
    for level, fmt in ((1, z.dfZlib), (6, z.dfDeflate), (9, z.dfGzip), (0, z.dfGzip)):
        outs = [tmp_path / ("o%d.bin" % i) for i in range(3)]
        subprocess.check_call([exe, str(inp), str(level), str(fmt), str(FL)] + [str(p) for p in outs])
        want = z.compress_batch([data, data[:len(data) // 2]], level, fmt, fname_lens=[FL, FL], rsyncable=True)
        assert outs[0].read_bytes() == want[0]
        assert outs[1].read_bytes() == want[0]
        assert outs[2].read_bytes() == want[1]
