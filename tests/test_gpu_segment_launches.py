"""Exact kernel launch counts (zb200_timing.kernel_launches) of the segment decode paths that no other test pins: one
decompress stream launch on each of its paths, Index.build with and without joints, one extract_batch range, and the
speculative segments of a large foreign member.  Each count is derived from zb_api.cu in the comment beside it; the
paths share their launch mechanics, so a change to one of them shows up here."""
import re
import zlib

import numpy as np
import pytest

from tests import util

pytestmark = pytest.mark.gpu

z = pytest.importorskip("zippy_b200")


@pytest.fixture(scope="module")
def text(corpus):
    return util.text_corpus(corpus)


@pytest.fixture(scope="module")
def log_ctx():
    """A context whose decompress streams name their decode path on stderr and launch only at finish for these
    members (the batching threshold is far above their sizes)."""
    mp = pytest.MonkeyPatch()
    mp.setenv("ZB200_DSTREAM_LOG", "1")
    mp.setenv("ZB200_DSTREAM_BATCH_BYTES", str(16 << 20))
    ctx = z.Context()
    mp.undo()
    yield ctx
    ctx.close()


def _raw(data, level):
    co = zlib.compressobj(level, zlib.DEFLATED, -15)
    return co.compress(data) + co.flush()


def _false_joint():
    """Stored blocks whose data holds one 00 00 ff ff, 40 000 bytes in: a joint that k_find_sync finds but that is
    not a block boundary."""
    rng = np.random.default_rng(5)
    data = bytes(rng.integers(1, 255, 40000, dtype=np.uint8)) + b"\x00\x00\xff\xff" + \
        bytes(rng.integers(1, 255, 40000, dtype=np.uint8))
    comp = _raw(data, 0)
    assert comp.count(b"\x00\x00\xff\xff") == 1
    return comp, data


def _one_launch(ctx, capfd, comp, df, data):
    """Writes the whole member, then finishes: the only launch is finish's.  -> (path, kernel launches)"""
    capfd.readouterr()
    with z.DecompressStream(df, ctx) as s:
        out = s.write(comp)
        out += s.finish()
    launches = ctx.timing()["kernel_launches"]
    assert out == data
    paths = re.findall(r"zb200 dstream: path=(\w+)", capfd.readouterr().err)
    assert len(paths) == 1, paths
    return paths[0], launches


def test_decompress_stream_joints(log_ctx, capfd, text):
    data = text[:300000]
    path, n = _one_launch(log_ctx, capfd, z.compress(data, 1, z.dfGzip), z.dfGzip, data)
    assert path == "joints"
    # k_find_sync 1, count pass 1, prefill 1, marker pass 1, resolve_groups 4, CRC-32 of the output 2
    assert n == 10


def test_decompress_stream_blocks(log_ctx, capfd, text):
    data = text[:300000]
    path, n = _one_launch(log_ctx, capfd, _raw(data, 6), z.dfDeflate, data)
    assert path == "blocks"
    # k_find_sync 1, k_find_blocks 1, count pass 1, prefill 1, marker pass 1, resolve_groups 4 (raw: no checksum)
    assert n == 9


def test_decompress_stream_serial(log_ctx, capfd, text):
    data = text[:60000]
    comp = zlib.compress(data, 6)
    assert len(comp) < 32768   # a payload of at most two 16 KiB gaps: no boundary search
    path, n = _one_launch(log_ctx, capfd, comp, z.dfZlib, data)
    assert path == "serial"
    # count pass 1, prefill 1, marker pass 1, resolve_groups 4, Adler-32 of the output 2
    assert n == 9


def test_decompress_stream_fallback(log_ctx, capfd):
    comp, data = _false_joint()
    path, n = _one_launch(log_ctx, capfd, comp, z.dfDeflate, data)
    assert path == "fallback"
    # k_find_sync 1, count pass over 2 segments 1 (segment 0 fails), count pass over 1 segment 1, prefill 1,
    # marker pass 1, resolve_groups 4
    assert n == 9


def test_index_build_with_joints(text):
    ctx = z.Context()
    data = text[:300000]
    idx = z.Index.build(z.compress(data, 1, z.dfGzip), z.dfGzip, 32768, ctx=ctx)
    assert idx.size == len(data)
    # decode_begin: inflate + verify 3; k_find_sync 1; count pass 1; recorder pass 1; interval CRC-32s 2; window gather 1
    assert ctx.timing()["kernel_launches"] == 9
    ctx.close()


def test_index_build_without_joints(text):
    ctx = z.Context()
    data = text[:300000]
    idx = z.Index.build(zlib.compress(data, 6), z.dfZlib, 32768, ctx=ctx)
    assert idx.size == len(data)
    # decode_begin 3; k_find_sync 1; k_find_blocks 1; count pass 1; recorder pass 1; interval CRC-32s 2; window gather 1
    assert ctx.timing()["kernel_launches"] == 10
    ctx.close()


def test_extract_one_range(text):
    ctx = z.Context()
    data = text[:300000]
    comp = z.compress(data, 1, z.dfGzip)
    idx = z.Index.build(comp, z.dfGzip, 32768, ctx=ctx)
    out, _, st = idx.extract_batch(comp, [100000], [5000])
    assert st[0] == 0 and out.tobytes() == data[100000:105000]
    # prefill 1, window gather 1, marker pass 1, resolve_groups 4, interval CRC-32s 2, gather of the range 1
    assert ctx.timing()["kernel_launches"] == 10
    ctx.close()


def test_speculative_foreign_zlib(text):
    ctx = z.Context()
    data = (text + text[::-1])[:2300000]
    comp = zlib.compress(data, 6)
    assert len(comp) > 512 << 10   # a single member this long takes the segment paths
    out, do, lens, st = ctx.uncompress_batch(np.frombuffer(comp, dtype=np.uint8), np.array([0, len(comp)], dtype=np.uint64),
                                             z.dfZlib)
    assert st[0] == 0 and out[int(do[0]):int(do[0]) + int(lens[0])].tobytes() == data
    # k_find_sync finds nothing (not counted); k_find_blocks 1, count pass 1, prefill + marker pass 2, resolve 2;
    # then the whole-member launch with the member skipped: inflate + verify 3
    assert ctx.timing()["kernel_launches"] == 9
    ctx.close()
