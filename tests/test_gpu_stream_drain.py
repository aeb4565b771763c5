"""Draining decompress streams (zb200_decompress_stream_drain, DecompressStream.drain).

A receiver that writes what a sender emitted up to a flush and then drains has read everything the sender wrote
up to that flush -- whatever the batching threshold, although the flush's empty stored block (and up to three
bytes of the block before it) lie in the 8 (gzip) / 4 (zlib) bytes held back as the possible trailer.  Once the
header is decided, that is (19 member bytes, and for gzip the whole header and 9 bytes more); before that a drain
decodes nothing.  finish still gives uncompress's output and status."""
import os
import random
import subprocess
import zlib

import pytest

from tests import util
from tests.test_gpu_stream_flush import FULL, SYNC, flushed

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
WBITS = {"gzip": 31, "zlib": 15, "deflate": -15}


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


def _df(z, fmt):
    return {"gzip": z.dfGzip, "zlib": z.dfZlib, "deflate": z.dfDeflate, "detect": z.dfDetect}[fmt]


@pytest.fixture(scope="module")
def contexts(z):
    """'default': the 64 MiB threshold (only drain and finish launch); 'some': a launch once about 100 000
    compressed bytes are pending."""
    mp = pytest.MonkeyPatch()
    ctxs = {"default": z.Context()}
    try:
        mp.setenv("ZB200_DSTREAM_BATCH_BYTES", "100000")
        ctxs["some"] = z.Context()
    finally:
        mp.undo()
    yield ctxs
    for c in ctxs.values():
        c.close()


def _lib_sender(z, data, level, fmt, offs, mode):
    """-> (member, [(input offset, compressed length) after each flush]) from this library's CompressStream"""
    comp, ends = flushed(z, None, data, level, fmt, [(o, mode) for o in offs], fname_len=4)
    return comp, list(zip(offs, ends))


def _zlib_sender(data, fmt, offs, mode, level=6):
    """-> the same from Python's zlib with Z_SYNC_FLUSH / Z_FULL_FLUSH"""
    co = zlib.compressobj(level, zlib.DEFLATED, WBITS[fmt])
    out, points, lo = bytearray(), [], 0
    for o in offs:
        out += co.compress(data[lo:o])
        out += co.flush(zlib.Z_SYNC_FLUSH if mode == SYNC else zlib.Z_FULL_FLUSH)
        points.append((o, len(out)))
        lo = o
    out += co.compress(data[lo:]) + co.flush()
    return bytes(out), points


def decided_at(comp, fmt):
    """Member bytes from which the header is decided: 19 and, for gzip, the whole header and 9 bytes more (the
    wrapper's length rule, zb_parse_wrapper); at once for raw streams."""
    if fmt == "deflate":
        return 0
    if fmt == "zlib":
        return 19
    p = 10
    if comp[3] & 8:
        p = comp.index(0, 10) + 1
    return max(19, p + 9)


def receive(z, ctx, comp, points, df, data, raw):
    """Write the member up to each flush point, drain, and check what has been read -> (bytes read, status)."""
    got, lo = bytearray(), 0
    need = 0 if raw else decided_at(comp, "gzip" if comp[:2] == b"\x1f\x8b" else "zlib")
    try:
        with z.DecompressStream(df, ctx) as s:
            for off, end in points:
                got += s.write(comp[lo:end])
                got += s.drain()
                lo = end
                if end >= need:
                    assert bytes(got) == data[:off], (off, end, len(got))
                else:
                    assert data.startswith(bytes(got))
            got += s.write(comp[lo:])
            got += s.finish()
    except z.ZippyError as e:
        return bytes(got), e.code
    return bytes(got), 0


def _offsets(n, rng, k=6):
    return sorted({1, 5000, 8193, 40000, *(rng.randrange(1, n) for _ in range(k))} - {n})


@pytest.fixture(scope="module")
def texts(corpus):
    rng = random.Random(0xD7)
    T = util.text_corpus(corpus)
    o = rng.randrange(len(T) - 400000)
    return {"text": T[o:o + 200001], "mix": T[:50000] + rng.randbytes(30000) + bytes(40000) + T[50000:90000]}


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,df", [("gzip", "gzip"), ("zlib", "zlib"), ("deflate", "deflate"), ("gzip", "detect"),
                                    ("zlib", "detect")])
def test_drain_after_each_flush_of_this_library(z, contexts, texts, fmt, df):
    rng = random.Random(0xA1)
    for name, data in texts.items():
        for level in (-2, 0, 1, -1, 6):
            for mode in (SYNC, FULL):
                comp, points = _lib_sender(z, data, level, fmt, _offsets(len(data), rng), mode)
                for ctx in ("default", "some"):
                    got, st = receive(z, contexts[ctx], comp, points, _df(z, df), data, fmt == "deflate")
                    assert (got, st) == (data, 0), (name, level, mode, ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,df", [("gzip", "gzip"), ("zlib", "zlib"), ("deflate", "deflate"), ("gzip", "detect"),
                                    ("zlib", "detect")])
def test_drain_after_each_zlib_flush(z, contexts, texts, fmt, df):
    """Python zlib's own sync and full flushes, every few bytes as well as far apart."""
    data = texts["text"]
    for mode in (SYNC, FULL):
        for step in (7, 1000, 70001):
            # (until 32 KiB of output exist, every drain decodes again from the payload start: keep these short)
            n = 3000 if step == 7 else 100000 if step == 1000 else len(data)
            offs = list(range(step, n, step))
            comp, points = _zlib_sender(data[:n], fmt, offs, mode, level=1 if step == 7 else 6)
            got, st = receive(z, contexts["default"], comp, points, _df(z, df), data[:n], fmt == "deflate")
            assert (got, st) == (data[:n], 0), (mode, step)


def _one_shot(z, comp, df):
    try:
        return z.uncompress(comp, df), 0
    except z.ZippyError as e:
        return None, e.code


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["gzip", "zlib", "deflate"])
def test_finish_after_drains_is_uncompress(z, contexts, texts, fmt):
    """Corruptions and truncations after a drain point, and a member cut inside its trailer: what was drained is
    the input up to the drain point, and finish gives uncompress's output and status."""
    data = texts["text"]
    rng = random.Random(0xC0)
    comp, points = _lib_sender(z, data, -1, fmt, [3000, 30000, 90000, 150000], SYNC)
    zc, zpoints = _zlib_sender(data, fmt, [3000, 30000, 90000, 150000], SYNC)
    trailer = {"gzip": 8, "zlib": 4, "deflate": 0}[fmt]
    cases = []
    for c, pts in ((comp, points), (zc, zpoints)):
        for off, end in pts[1:3]:
            for _ in range(3):
                bad = bytearray(c)
                i = rng.randrange(end, len(c))
                bad[i] ^= 1 << rng.randrange(8)
                cases.append((bytes(bad), [p for p in pts if p[1] <= i]))
            cases.append((c[:end + rng.randrange(1, 2000)], [p for p in pts if p[1] <= end]))
            cases.append((c[:end], [p for p in pts if p[1] <= end]))
        for cut in range(1, trailer + 1):
            cases.append((c[:-cut], pts))
        cases.append((c[:-trailer - 2] if trailer else c[:-2], pts))
    for ci, (c, pts) in enumerate(cases):
        pts = [(o, e) for o, e in pts if e <= len(c)]
        want = _one_shot(z, c, _df(z, fmt))
        for ctx in ("default", "some"):
            got, st = receive(z, contexts[ctx], c, pts, _df(z, fmt), data, fmt == "deflate")
            assert st == want[1], (ci, ctx, st, want[1])
            if st == 0:
                assert got == want[0]


@pytest.mark.gpu
def test_drain_contract(z, contexts, texts):
    """drain on an empty stream, before 19 bytes have arrived, and after finish."""
    data = texts["text"][:5000]
    comp = z.compress(data, -1, z.dfGzip)
    for df in ("gzip", "detect", "zlib", "deflate"):
        with z.DecompressStream(_df(z, df), contexts["default"]) as s:
            assert s.drain() == b""
            assert s.drain() == b""
    with z.DecompressStream(z.dfGzip, contexts["default"]) as s:
        assert s.write(comp[:18]) == b"" and s.drain() == b""
        got = s.write(comp[18:]) + s.drain() + s.finish()
        assert got == data
        with pytest.raises(z.ZippyError) as e:
            s.drain()
        assert e.value.code == 22
    # a failure is the stream's error: every later call repeats it
    bad = bytearray(z.compress(data, 1, z.dfDeflate))
    bad[0] |= 6                      # block type 3
    with z.DecompressStream(z.dfDeflate, contexts["default"]) as s:
        s.write(bytes(bad))
        with pytest.raises(z.ZippyError) as e:
            s.drain()
            s.finish()
        code = e.value.code
        with pytest.raises(z.ZippyError) as e:
            s.drain()
        assert e.value.code == code


def _cpp_flush_exe(tmp_path):
    exe = str(tmp_path / "cpp_flush_test")
    libdir = os.path.join(ROOT, "zippy_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(HERE, "native", "cpp_flush_test.cpp"),
                           "-L" + libdir, "-l:libzippy_b200.so", "-Wl,-rpath," + libdir])
    return exe


def test_cpp_flush_compiles_and_links(tmp_path):
    """CompressStream::flush and DecompressStream::drain of include/zippy_b200.hpp build against the library."""
    import __graft_entry__ as g
    g.build()
    assert os.path.exists(_cpp_flush_exe(tmp_path))


@pytest.mark.gpu
@pytest.mark.parametrize("level,fmt,msg", [(-1, "gzip", 1024), (1, "zlib", 65536), (6, "deflate", 3000)])
def test_cpp_flush_matches_python(z, texts, tmp_path, level, fmt, msg):
    exe = _cpp_flush_exe(tmp_path)
    data = texts["text"][:300000]
    src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
    src.write_bytes(data)
    subprocess.check_call([exe, str(src), str(dst), str(level), str(_df(z, fmt)), str(msg)])
    offs = list(range(msg, len(data), msg)) + [len(data)]
    py, _ = flushed(z, None, data, level, fmt, [(o, SYNC) for o in offs], fname_len=0)
    assert dst.read_bytes() == py
    assert zlib.decompress(py, WBITS[fmt]) == data
