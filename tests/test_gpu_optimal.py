"""The optimal parse on the GPU (k_opt; zb200_compress_batch_optimal, its device and stream forms).

The kernel's tokens equal tests/native/opt_model.c's chunk by chunk, at windows 9, 12 and 15 and after 1..32767
bytes of history (stream segments after a sync flush); every member inflates with zlib, the oracle and uncompress;
a member's bytes do not depend on its batch, the level, the device-resident call or a stream's write splits; and
the refusals leave statuses alone.
"""
import ctypes
import random
import zlib

import numpy as np
import pytest

import zippy_b200 as z
from tests import deflate_tokens as dt
from tests import util
from tests.test_optimal_model import CHUNK, build_model, decode, encode, model_inputs

pytestmark = pytest.mark.gpu

WBITS = {z.dfGzip: 31, z.dfZlib: 15, z.dfDeflate: -15}


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return build_model(tmp_path_factory)


def _block_tokens(raw):
    """Token lists of the non-empty blocks of a raw stream, in order (a stored block as its bytes)."""
    return [(b.btype, list(b.tokens)) for b in dt.parse(raw) if b.tokens]


def _compare(name, raw, buf, wanted):
    """wanted: the model's chunks, in order.  Every coded block must hold exactly the next chunk's tokens."""
    got = _block_tokens(raw)
    assert len(got) >= len([w for w in wanted if len(w)]), name
    bad, gi, compared = [], 0, 0
    for k, w in enumerate(wanted):
        if len(w) == 0:
            continue
        bt, toks = got[gi]
        gi += 1
        if bt == 0:
            continue
        compared += 1
        if not np.array_equal(encode(toks), w):
            a = encode(toks)
            i = int(np.argmax(a[:min(len(a), len(w))] != w[:min(len(a), len(w))])) if len(a) and len(w) else 0
            bad.append((name, k, i, decode(a[max(0, i - 2):i + 3]), decode(w[max(0, i - 2):i + 3])))
    return bad, compared


@pytest.mark.parametrize("window_bits", [9, 12, 15])
def test_kernel_tokens_equal_the_model(model, corpus, window_bits):
    xs = model_inputs(corpus)
    one_shot = [(n, b) for n, b, h in xs if h == 0]
    comp = z.compress_batch([b for _, b in one_shot], 9, z.dfDeflate, window_bits=window_bits, optimal=True)
    bad, compared = [], 0
    for (name, x), c in zip(one_shot, comp):
        assert zlib.decompress(c, -window_bits) == x, name
        b, k = _compare(name, c, x, model.run(x, 0, window_bits))
        bad += b
        compared += k
    # history: a stream's segment after a sync flush at h sees min(32768, h) bytes of the member before it
    for name, buf, h in xs:
        if h == 0:
            continue
        s = z.CompressStream(6, z.dfDeflate, window_bits=window_bits, optimal=True)
        raw = s.write(buf[:h]) + s.flush(z.SyncFlush) + s.write(buf[h:]) + s.finish()
        s.close()
        assert zlib.decompress(raw, -window_bits) == buf, name
        want = model.run(buf[:h], 0, window_bits) + model.run(buf, h, window_bits)
        b, k = _compare(name, raw, buf, want)
        bad += b
        compared += k
    assert not bad, bad[:10]
    assert compared >= 30


def _edge_members():
    rng = random.Random(0x0D7)
    T = util.text_corpus(util.load_corpus())
    xs = [b"", b"q", bytes(100000), rng.randbytes(70000), T[:CHUNK - 1], T[5:CHUNK + 5], T[9:CHUNK + 10],
          T[100:100 + 3 * CHUNK + 7]]
    return xs


@pytest.mark.parametrize("fmt", [z.dfGzip, z.dfZlib, z.dfDeflate])
def test_members_inflate_everywhere(fmt):
    from oracle import oracle as o
    xs = _edge_members()
    comp = z.compress_batch(xs, z.DefaultCompression, fmt, optimal=True)
    for x, c in zip(xs, comp):
        assert zlib.decompress(c, WBITS[fmt]) == x
        assert z.uncompress(c, fmt) == x
        if fmt != z.dfDeflate:
            assert o.uncompress(c) == x
        assert len(c) <= z._native.lib().zb200_compress_bound(len(x), fmt)


def test_bytes_do_not_depend_on_batch_level_or_call(corpus):
    xs = _edge_members() + [corpus["urls.10K"][:200000], corpus["html"]]
    a = z.compress_batch(xs, 9, z.dfZlib, optimal=True)
    b = z.compress_batch(xs[::-1], 1, z.dfZlib, optimal=True)[::-1]
    c = [z.compress_batch([x], -1, z.dfZlib, optimal=True)[0] for x in xs]
    assert a == b == c
    assert z.compress(xs[-1], 5, z.dfZlib, optimal=True) == a[-1]
    assert z.deflate(xs[-1], optimal=True) == z.compress_batch([xs[-1]], 9, z.dfDeflate, optimal=True)[0]
    assert a[-1][:2] == bytes([0x78, 0x01])
    import torch
    base, offs = z._pack(xs)
    src = torch.from_numpy(np.frombuffer(bytes(base), dtype=np.uint8).copy()).cuda()
    cap = sum(z._native.lib().zb200_compress_bound(len(x), z.dfZlib) + 64 for x in xs) + 64
    dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    ctx = z.default_context()
    oo = ctx.compress_batch_device(src.data_ptr(), offs, 3, z.dfZlib, dst.data_ptr(), cap, optimal=True)
    out = dst.cpu().numpy()
    assert [out[int(oo[i]):int(oo[i + 1])].tobytes() for i in range(len(xs))] == a


def test_stream_writes_the_one_shot_member(corpus):
    rng = random.Random(0x57E)
    T = util.text_corpus(corpus)
    x = T[777:777 + 3 * CHUNK + 12345]
    want = z.compress_batch([x], 9, z.dfGzip, fname_lens=[3], optimal=True)[0]
    s = z.CompressStream(9, z.dfGzip, fname_len=3, optimal=True)
    out, i = b"", 0
    while i < len(x):
        k = rng.randrange(1, 70000)
        out += s.write(x[i:i + k])
        i += k
    out += s.finish()
    s.close()
    assert out == want
    # a full flush drops the history: a fresh raw inflater starts right after it
    s = z.CompressStream(9, z.dfDeflate, optimal=True)
    f = 50000
    head = s.write(x[:f]) + s.flush(z.FullFlush)
    tail = s.write(x[f:]) + s.finish()
    s.close()
    assert zlib.decompress(head + tail, -15) == x
    assert zlib.decompressobj(-15).decompress(tail) == x[f:]


def test_refusals_leave_statuses_alone():
    L = z._native.lib()
    ctx = z.default_context()._h
    src = np.frombuffer(b"hello hello hello", dtype=np.uint8).copy()
    offs = np.array([0, src.size], dtype=np.uint64)
    out = np.zeros(256, dtype=np.uint8)
    oo = np.zeros(2, dtype=np.uint64)
    st = np.full(1, 77, dtype=np.int32)
    for wb in (7, 8, 16, -15):
        fmt = z.dfGzip if wb == 8 else z.dfZlib
        rc = L.zb200_compress_batch_optimal(ctx, src.ctypes.data, offs.ctypes.data, 1, wb, fmt, None, out.ctypes.data,
                                            out.size, oo.ctypes.data, st.ctypes.data)
        assert rc == 22 and st[0] == 77, wb
        h = ctypes.c_void_p()
        assert L.zb200_compress_stream_begin_optimal(ctx, wb, fmt, 0, ctypes.byref(h)) == 22
    for kw in (dict(strategy=z.StrategyFiltered), dict(dictionary=b"hello"), dict(index_span=1 << 20)):
        with pytest.raises(z.ZippyError) as e:
            z.compress_batch([b"hello"], 9, z.dfZlib, optimal=True, **kw) if "index_span" not in kw else \
                z.default_context().compress_batch(src, offs, 9, z.dfZlib, optimal=True, **kw)
        assert e.value.code == 22
    for lvl in (0, -2):
        with pytest.raises(z.ZippyError) as e:
            z.compress(b"hello", lvl, z.dfZlib, optimal=True)
        assert e.value.code == 22
    with pytest.raises(z.ZippyError) as e:
        z.compress_batch([b"a"], 9, z.dfZlib, optimal=True, dictionaries=[b"x"])
    assert e.value.code == 22


def test_cpp_equals_python(tmp_path, corpus):
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "cpp_optimal_test")
    libdir = os.path.join(root, "zippy_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(root, "tests", "native", "cpp_optimal_test.cpp"),
                           "-L" + libdir, "-l:libzippy_b200.so", "-Wl,-rpath," + libdir])
    data = corpus["alice29.txt"]
    inp = tmp_path / "in.bin"
    inp.write_bytes(data)
    for n, fmt in ((9, z.dfZlib), (12, z.dfDeflate), (15, z.dfGzip)):
        o1, o2 = tmp_path / "m.bin", tmp_path / "s.bin"
        subprocess.check_call([exe, str(inp), str(n), str(fmt), "5", "30000", str(o1), str(o2)])
        if fmt != z.dfGzip:
            assert o1.read_bytes() == z.compress_batch([data], 9, fmt, window_bits=n, optimal=True)[0]
        s = z.CompressStream(9, fmt, fname_len=5, window_bits=n, optimal=True)
        m = b""
        for off in range(0, len(data), 30000):
            m += s.write(data[off:off + 30000])
            if off == 0:
                m += s.flush()
        m += s.finish()
        s.close()
        assert o2.read_bytes() == m
