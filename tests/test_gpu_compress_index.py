"""An index written while compressing (zb200_compress_batch_index, zb200_compress_batch_device_index and compress
streams begun with an index): the members are the bytes the calls without an index write, and every index exports
to exactly the bytes Index.build gives for its member, whose points tests/test_gpu_index.py's model_points defines."""
import os
import random
import zlib

import numpy as np
import pytest

from tests import util
from tests.test_gpu_index import index_points, model_points

pytestmark = pytest.mark.gpu

z = pytest.importorskip("zippy_b200")

ERR_ARG, ERR_INVALID_LEVEL, ERR_INVALID_FORMAT = 22, 1, 2
LEVELS = list(range(-2, 10))
FORMATS = [("gzip", 2), ("zlib", 1), ("deflate", 3)]
SPANS = [32768, 65536, 98304, 1 << 20]


@pytest.fixture(scope="module")
def text():
    T = util.text_corpus(util.load_corpus())
    return (T * (3 * (1 << 20) // len(T) + 1))[:3 * (1 << 20) + 12345]


def _inputs(T):
    """The sizes and contents the issue lists: edges of 32 KiB / 64 KiB, stored chunks, zeros, mixed chunks."""
    rng = random.Random(7)
    rnd = bytes(rng.randrange(256) for _ in range(300000))
    mixed = b"".join((rnd[i * 65536:(i + 1) * 65536] if i % 2 else T[i * 65536:(i + 1) * 65536]) for i in range(5))
    out = [("empty", b""), ("one", b"x")]
    for n in (32767, 32768, 32769, 65535, 65536, 65537, 131072):
        out.append(("text-%d" % n, T[:n]))
    out += [("text-big", T), ("random", rnd), ("random-65536", rnd[:65536]), ("random-131073", rnd[:131073]),
            ("zeros", bytes(200000)), ("mixed", mixed)]
    return out


def _exp(data, fmt, span):
    idx = z.Index.build(data, fmt, span)
    b = idx.to_bytes()
    idx.close()
    return b


def _check_batch(items, level, fmt, span, ctx=None, fname_lens=None):
    ctx = ctx or z.default_context()
    base, offs = z._pack(items)
    out, oo = ctx.compress_batch(base, offs, level, fmt, fname_lens)
    out2, oo2, idx = ctx.compress_batch(base, offs, level, fmt, fname_lens, index_span=span)
    assert out.tobytes() == out2.tobytes() and (oo == oo2).all()
    for i in range(len(items)):
        member = out[int(oo[i]):int(oo[i + 1])].tobytes()
        assert idx[i].to_bytes() == _exp(member, fmt, span), (level, fmt, span, i, len(items[i]))
    return out, oo, idx


@pytest.mark.parametrize("fmt", [f for _, f in FORMATS])
@pytest.mark.parametrize("level", LEVELS)
def test_index_equals_build(text, level, fmt):
    items = [d for _, d in _inputs(text)]
    fl = [(i * 7) % 26 for i in range(len(items))] if fmt == z.dfGzip else None
    for span in SPANS:
        _, _, idx = _check_batch(items, level, fmt, span, fname_lens=fl)
        for x in idx:
            x.close()


@pytest.mark.parametrize("fmt", [f for _, f in FORMATS])
@pytest.mark.parametrize("level", [0, 1, -1, 9])
def test_points_equal_the_model(text, level, fmt):
    items = [d for n, d in _inputs(text) if n not in ("text-big",)]
    base, offs = z._pack(items)
    out, oo, idx = z.default_context().compress_batch(base, offs, level, fmt, index_span=65536)
    for i, d in enumerate(items):
        member = out[int(oo[i]):int(oo[i + 1])].tobytes()
        want, dec = model_points(member, fmt, 65536)
        assert dec == d
        assert index_points(idx[i]) == want, (level, fmt, i)


@pytest.mark.parametrize("group", ["1", "3"])
def test_launch_group_edges(text, group, monkeypatch):
    monkeypatch.setenv("ZB200_GROUP_CHUNKS", group)
    ctx = z.Context()
    try:
        items = [d for _, d in _inputs(text)]
        rng = random.Random(int(group))
        rng.shuffle(items)
        for level, fmt in ((1, z.dfGzip), (-1, z.dfZlib), (0, z.dfDeflate), (6, z.dfGzip)):
            _check_batch(items, level, fmt, 32768, ctx=ctx)
    finally:
        ctx.close()


def test_device_input_matches_host(text):
    torch = pytest.importorskip("torch")
    items = [d for _, d in _inputs(text)]
    base, offs = z._pack(items)
    ctx = z.default_context()
    d_src = torch.from_numpy(base.copy()).cuda()
    cap = int(sum(z._native.lib().zb200_compress_bound(len(x), 2) + 64 for x in items)) + 4096
    for level in (0, 1, -1):
        for _, fmt in FORMATS:
            d_a = torch.empty(cap, dtype=torch.uint8, device="cuda")
            d_b = torch.empty(cap, dtype=torch.uint8, device="cuda")
            oo = ctx.compress_batch_device(d_src.data_ptr(), offs, level, fmt, d_a.data_ptr(), cap)
            oo2, idx = ctx.compress_batch_device(d_src.data_ptr(), offs, level, fmt, d_b.data_ptr(), cap,
                                                 index_span=65536)
            torch.cuda.synchronize()
            a = d_a[:int(oo[-1])].cpu().numpy().tobytes()
            b = d_b[:int(oo2[-1])].cpu().numpy().tobytes()
            assert a == b and (oo == oo2).all()
            for i in range(len(items)):
                member = a[int(oo[i]):int(oo[i + 1])]
                assert idx[i].to_bytes() == _exp(member, fmt, 65536), (level, fmt, i)


def test_reads_from_the_compress_time_index(text):
    rng = random.Random(3)
    for level, fmt in ((1, z.dfGzip), (6, z.dfZlib), (0, z.dfDeflate)):
        member, idx = z.compress_with_index(text, level, fmt, span=98304)
        out = z.uncompress(member, fmt)
        assert out == text
        for ix in (idx, z.Index.from_bytes(idx.to_bytes())):
            pts = [int(o) for o in ix.points["out"]]
            ranges = [(0, len(out)), (len(out), 0)]
            for p in pts[1:6] + pts[-3:]:
                for d in (-1, 0, 1):
                    a = min(max(p + d, 0), len(out))
                    ranges.append((a, min(70000, len(out) - a)))
            for _ in range(20):
                a = rng.randrange(len(out))
                ranges.append((a, rng.randrange(min(len(out) - a, 200000) + 1)))
            got, goff, st = ix.extract_batch(member, [a for a, _ in ranges], [n for _, n in ranges])
            assert (st == 0).all()
            for i, (a, n) in enumerate(ranges):
                assert got[int(goff[i]):int(goff[i + 1])].tobytes() == out[a:a + n]


def test_batch_with_index_helper(text):
    items = [text[:100000], b"", text[5:70000]]
    res = z.compress_batch_with_index(items, 1, z.dfGzip, span=32768)
    for (member, idx), d in zip(res, items):
        assert zlib.decompress(member, 31) == d
        assert idx.to_bytes() == _exp(member, z.dfGzip, 32768)


# ---- streams ----
@pytest.fixture(scope="module")
def stream_contexts():
    mp = pytest.MonkeyPatch()
    ctxs = {}
    try:
        for name, v in (("one", "1"), ("three", str(3 * 65536 + 5))):
            mp.setenv("ZB200_STREAM_BATCH_BYTES", v)
            ctxs[name] = z.Context()
    finally:
        mp.undo()
    yield ctxs
    for c in ctxs.values():
        c.close()


def _run_stream(ctx, data, level, fmt, span, cuts, flushes, finish_after_flush=False):
    """cuts: write boundaries; flushes: {position: mode} flushed after the write that ends there."""
    s = z.CompressStream(level, fmt, fname_len=5 if fmt == z.dfGzip else None, ctx=ctx, index_span=span)
    out, prev = [], 0
    for c in sorted(set(cuts) | set(flushes) | {len(data)}):
        out.append(s.write(data[prev:c]))
        prev = c
        if c in flushes:
            out.append(s.flush(flushes[c]))
    if finish_after_flush:
        out.append(s.flush(z.SyncFlush))
    out.append(s.finish())
    idx = s.index()
    s.close()
    return b"".join(out), idx


@pytest.mark.parametrize("ctxname", ["one", "three"])
def test_stream_index_equals_build(text, stream_contexts, ctxname):
    ctx = stream_contexts[ctxname]
    rng = random.Random(11)
    rnd = bytes(rng.randrange(256) for _ in range(400000))
    data = (text[:300000] + rnd + text[300000:700000])
    edges = [1, 5000, 8191, 8192, 8193, 32767, 32768, 32769, 65535, 65537]
    for level, fmt in ((1, z.dfGzip), (-1, z.dfZlib), (0, z.dfDeflate), (-2, z.dfGzip), (6, z.dfDeflate)):
        for trial in range(2):
            cuts = sorted(rng.randrange(len(data)) for _ in range(12))
            fl = {e: (z.SyncFlush if (e + trial) % 2 else z.FullFlush) for e in edges}
            fl.update({rng.randrange(len(data)): z.SyncFlush for _ in range(4)})
            member, idx = _run_stream(ctx, data, level, fmt, SPANS[trial + 1], cuts, fl,
                                      finish_after_flush=bool(trial))
            assert z.uncompress(member, fmt) == data
            assert idx.to_bytes() == _exp(member, fmt, SPANS[trial + 1]), (level, fmt, trial)


def test_stream_flush_every_100_bytes(text, stream_contexts):
    data = text[:1 << 20]
    fl = {p: z.SyncFlush for p in range(100, len(data), 100)}
    for level, fmt in ((1, z.dfGzip), (0, z.dfZlib)):
        member, idx = _run_stream(stream_contexts["three"], data, level, fmt, 65536, [], fl)
        assert idx.to_bytes() == _exp(member, fmt, 65536)
        want, _ = model_points(member, fmt, 65536)
        assert index_points(idx) == want


def test_stream_empty_and_tiny(stream_contexts):
    for data in (b"", b"a", b"ab" * 20000):
        for level, fmt in ((1, z.dfGzip), (0, z.dfDeflate), (-1, z.dfZlib)):
            member, idx = _run_stream(stream_contexts["one"], data, level, fmt, 32768, [], {})
            assert idx.to_bytes() == _exp(member, fmt, 32768)
            member, idx = _run_stream(stream_contexts["one"], data, level, fmt, 32768, [], {}, finish_after_flush=True)
            assert idx.to_bytes() == _exp(member, fmt, 32768)


def test_stream_past_4_gib():
    """One Default-level 4 GiB + 1 MiB member written in 256 MiB pieces: offsets and bit positions past 2^32."""
    rng = random.Random(41)
    words = [bytes(rng.choice(b"abcdefghij") for _ in range(rng.randrange(2, 9))) for _ in range(3000)]
    tile = b" ".join(rng.choice(words) for _ in range(200000))[:1 << 20]
    block = tile * 256
    total = (4 << 30) + (1 << 20)
    s = z.CompressStream(z.DefaultCompression, z.dfGzip, fname_len=0, index_span=1 << 26)
    out, w = [], 0
    while w < total:
        n = min(len(block), total - w)
        out.append(s.write(block[:n]))
        w += n
    out.append(s.finish())
    idx = s.index()
    s.close()
    member = b"".join(out)
    assert idx.size == total
    assert idx.to_bytes() == _exp(member, z.dfGzip, 1 << 26)


# ---- errors ----
def test_errors(text):
    L, ctx = z._native.lib(), z.default_context()
    base, offs = z._pack([text[:1000]])
    for span in (0, 1, 32767, 32769, 65537):
        with pytest.raises(z.ZippyError) as e:
            ctx.compress_batch(base, offs, 1, z.dfGzip, index_span=span)
        assert e.value.code == ERR_ARG
        with pytest.raises(z.ZippyError) as e:
            z.CompressStream(1, z.dfGzip, index_span=span)
        assert e.value.code == ERR_ARG
    with pytest.raises(z.ZippyError) as e:
        ctx.compress_batch(base, offs, 10, z.dfGzip, index_span=32768)
    assert e.value.code == ERR_INVALID_LEVEL
    with pytest.raises(z.ZippyError) as e:
        ctx.compress_batch(base, offs, 1, z.dfDetect, index_span=7)
    assert e.value.code == ERR_INVALID_FORMAT
    s = z.CompressStream(1, z.dfGzip, index_span=32768)
    s.write(text[:100000])
    with pytest.raises(z.ZippyError) as e:
        s.index()
    assert e.value.code == ERR_ARG
    s.finish()
    assert s.index().size == 100000
    s.close()
    s = z.CompressStream(1, z.dfGzip)
    s.finish()
    with pytest.raises(z.ZippyError) as e:
        s.index()
    assert e.value.code == ERR_ARG
    s.close()
    # a call that fails leaves every entry NULL, with the status of the call without an index
    import ctypes
    out = np.empty(16, np.uint8)
    oo = np.zeros(2, np.uint64)
    st = np.zeros(1, np.int32)
    hs = (ctypes.c_void_p * 1)(123)
    rc_plain = L.zb200_compress_batch(ctx._h, base.ctypes.data, offs.ctypes.data, 1, 1, 2, None, out.ctypes.data,
                                      out.size, oo.ctypes.data, st.ctypes.data)
    rc = L.zb200_compress_batch_index(ctx._h, base.ctypes.data, offs.ctypes.data, 1, 1, 2, None, out.ctypes.data,
                                      out.size, oo.ctypes.data, st.ctypes.data, 32768, hs)
    assert rc == rc_plain != 0 and hs[0] is None


def test_cpp_equals_python(tmp_path, text):
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "cpp_compress_index_test")
    libdir = os.path.join(root, "zippy_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe,
                           os.path.join(root, "tests", "native", "cpp_compress_index_test.cpp"),
                           "-L" + libdir, "-l:libzippy_b200.so", "-Wl,-rpath," + libdir])
    data = text[:700001]
    inp = tmp_path / "in.bin"
    inp.write_bytes(data)
    for level, fmt, fl in ((1, z.dfGzip, 7), (-1, z.dfZlib, 0), (0, z.dfDeflate, 0)):
        outs = [tmp_path / ("o%d.bin" % i) for i in range(4)]
        subprocess.check_call([exe, str(inp), str(level), str(fmt), "65536", str(fl), "100000"] + [str(o) for o in outs])
        base, offs = z._pack([data])
        out, oo, idx = z.default_context().compress_batch(base, offs, level, fmt, [fl] if fmt == z.dfGzip else None,
                                                          index_span=65536)
        assert outs[0].read_bytes() == out.tobytes()
        assert outs[1].read_bytes() == idx[0].to_bytes()
        s = z.CompressStream(level, fmt, fname_len=fl, index_span=65536)
        m = b""
        for off in range(0, len(data), 100000):
            m += s.write(data[off:off + 100000])
            if off == 0:
                m += s.flush()
        m += s.finish()
        assert outs[2].read_bytes() == m
        assert outs[3].read_bytes() == s.index().to_bytes() == _exp(m, fmt, 65536)
        s.close()
