"""The CRC-32 / Adler-32 kernels against zlib at every piece, warp, lane and fold boundary (tests/checksum_shapes.py),
through each of their callers:

A. the standalone calls (crc32 / adler32, checksum_batch, checksum_batch_device at every base shift), alone and in
   batches that put many pieces on every CTA, both combine kernels in one call, a reused Context, a buffer past 4 GiB;
B. the trailer verdict of batch decodes (host, caller sizes, device, both host pipelines), members made by Python's
   zlib, with flipped trailer bytes, wrong ISIZEs and members that fail to inflate, against the oracle's verdicts;
C. inflate_batch_crc32, the running check of a DecompressStream, the DICTIDs of per-member dictionaries;
D. the compress-side fold (k_member_check): trailers at every level and strategy, compress streams, a 4 GiB member.

Every checksum is compared with zlib.crc32 / zlib.adler32 of the same bytes."""
import os
import re
import zlib

import numpy as np
import pytest

from tests import checksum_shapes as cs
from tests import util

pytestmark = pytest.mark.gpu

KINDS = ("crc32", "adler32")
REF = {"crc32": zlib.crc32, "adler32": zlib.adler32}


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


@pytest.fixture(scope="module")
def o():
    from oracle import oracle
    return oracle


@pytest.fixture(scope="module")
def text(corpus):
    return util.text_corpus(corpus)


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return t


def _need_free(torch, nbytes):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip("needs %d GiB of free device memory" % (nbytes >> 30))


def _offsets(lengths):
    offs = np.zeros(len(lengths) + 1, dtype=np.uint64)
    np.cumsum(np.asarray(lengths, dtype=np.uint64), out=offs[1:])
    return offs


def _refs(blob, offs, kind):
    mv = memoryview(blob)
    return [REF[kind](mv[int(offs[i]):int(offs[i + 1])]) for i in range(len(offs) - 1)]


def _check(got, want, offs, what):
    got = [int(x) for x in got]
    bad = [(i, int(offs[i + 1] - offs[i]), got[i], want[i]) for i in range(len(want)) if got[i] != want[i]]
    assert not bad, "%s: (index, length, got, zlib) %s" % (what, bad[:8])


# ---------------------------------------------------------------------------------------------------------------
# A. the standalone calls

@pytest.mark.parametrize("fill", ["random", "ff", "zeros"])
def test_sweep_alone_and_in_one_batch(z, fill):
    """Every sweep size in one batch (many ring stages and descriptor refreshes per CTA), then each alone (grid =
    its piece count), both kinds."""
    offs = _offsets(cs.SWEEP)
    blob = cs.content(fill, int(offs[-1]), seed=7)
    ctx = z.Context()
    for kind in KINDS:
        want = _refs(blob, offs, kind)
        _check(ctx.checksum_batch(blob, offs, kind), want, offs, "batch %s %s" % (fill, kind))
        one = ctx.crc32 if kind == "crc32" else ctx.adler32
        got = [one(blob[int(offs[i]):int(offs[i + 1])]) for i in range(len(cs.SWEEP))]
        _check(got, want, offs, "alone %s %s" % (fill, kind))
    ctx.close()


def test_device_sweep_at_every_base_shift(z, torch):
    """checksum_batch_device from torch memory at base shifts 0..15, buffers placed so that full pieces start at
    every address mod 16 (the aligned and unaligned row loads of the CRC path, misaligned Adler)."""
    _, _, offs, _ = cs.device_layout()
    blob = cs.content("random", int(offs[-1]), seed=8)
    want = {k: _refs(blob, offs, k) for k in KINDS}
    ctx = z.Context()
    ctx.set_stream(ctx.LEGACY_DEFAULT_STREAM)
    host = torch.from_numpy(blob.copy())
    d_all = torch.zeros(blob.size + 64, dtype=torch.uint8, device="cuda")
    for shift in range(16):
        d_all.zero_()
        d_all[shift:shift + blob.size] = host.cuda()
        for kind in KINDS:
            _check(ctx.checksum_batch_device(d_all.data_ptr() + shift, offs, kind), want[kind], offs,
                   "device shift %d %s" % (shift, kind))
    ctx.close()


def test_many_tiny_buffers_with_empties(z):
    rng = np.random.default_rng(9)
    lengths = rng.integers(0, 41, 100000)
    lengths[::7] = 0
    offs = _offsets(lengths)
    blob = cs.content("random", int(offs[-1]), seed=10)
    ctx = z.Context()
    for kind in KINDS:
        _check(ctx.checksum_batch(blob, offs, kind), _refs(blob, offs, kind), offs, "tiny " + kind)
    ctx.close()


def test_exactly_big_pieces_beside_a_bigger_buffer(z):
    """A buffer of exactly ZB_CK_BIG_PIECES pieces stays with k_buffer_combine while a bigger one in the same call
    turns k_buffer_combine_big on; then the same buffer alone.  A fresh Context first, so no earlier result sits in
    the output buffer."""
    n0, n1 = cs.BIG_PIECES * cs.PIECE, cs.BIG_PIECES * cs.PIECE + 1
    blob = cs.content("random", n0 + n1, seed=11)
    for order in ((n0, n1), (n1, n0)):
        offs = _offsets(order)
        for kind in KINDS:
            ctx = z.Context()
            _check(ctx.checksum_batch(blob, offs, kind), _refs(blob, offs, kind), offs, "pair %s %s" % (order, kind))
            ctx.close()
    ctx = z.Context()
    alone = blob[:n0]
    assert ctx.crc32(alone) == zlib.crc32(alone) and ctx.adler32(alone) == zlib.adler32(alone)
    ctx.close()


def test_both_combine_kernels_in_one_call(z):
    rng = np.random.default_rng(12)
    lengths = list(rng.integers(0, 3000, 10000))
    lengths[4321] = (64 << 20) + 1
    offs = _offsets(lengths)
    blob = cs.content("random", int(offs[-1]), seed=13)
    ctx = z.Context()
    for kind in KINDS:
        _check(ctx.checksum_batch(blob, offs, kind), _refs(blob, offs, kind), offs, "mixed " + kind)
    ctx.close()


def test_context_reuse_large_small_large(z):
    """The scratch (pieces, partials, outputs) is sized by the largest call: a smaller call after it must not see
    the larger call's stale entries, nor the larger call repeated see the smaller one's."""
    big = [5, (96 << 20) + 1, 2048 * 19, 32768 * 40 + 3]
    small = [3, 65536, 0, 2048 * 21]
    ob, osm = _offsets(big), _offsets(small)
    bb = cs.content("random", int(ob[-1]), seed=14)
    sb = cs.content("ff", int(osm[-1]))
    ctx = z.Context()
    for kind in KINDS:
        for blob, offs in ((bb, ob), (sb, osm), (bb, ob)):
            _check(ctx.checksum_batch(blob, offs, kind), _refs(blob, offs, kind), offs, "reuse " + kind)
        for blob, offs in ((bb, ob), (sb, osm)):
            one = ctx.crc32 if kind == "crc32" else ctx.adler32
            x = blob[int(offs[1]):int(offs[2])]
            assert one(x) == REF[kind](x)
    ctx.close()


def test_a_buffer_past_4_GiB(z, torch):
    _need_free(torch, 12 << 30)
    n = cs.HUGE[0]
    blob = np.resize(cs.content("random", (1 << 20) + 7, seed=15), n)   # period prime to the piece size
    blob[n - 5000:] = cs.content("random", 5000, seed=16)
    ctx = z.Context()
    assert ctx.crc32(blob) == zlib.crc32(blob)
    assert ctx.adler32(blob) == zlib.adler32(blob)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# B. decode verification

def _with_oracle(o, items):
    """[(name, member, output or None, output length)] -> (base, offs, names, outputs, oracle categories, output
    lengths); every corrupted member must be one the oracle refuses"""
    names = [x[0] for x in items]
    outs = [x[2] for x in items]
    offs = _offsets([len(x[1]) for x in items])
    base = np.frombuffer(b"".join(x[1] for x in items), dtype=np.uint8)
    _, _, ost = o.uncompress_batch(base, offs, o.dfDetect, threads=os.cpu_count() or 1)
    cats = [_category(int(s)) for s in ost]
    for name, out, c in zip(names, outs, cats):
        assert (c == 0) == (out is not None), (name, c)
    return base, offs, names, outs, cats, np.array([x[3] for x in items], dtype=np.uint64)


@pytest.fixture(scope="module")
def verify_batch(o, text):
    """gzip and zlib members of the sweep sizes up to ZB_CK_BIG_PIECES pieces + 1 byte interleaved, each followed by
    its corruptions (_with_oracle).  Up to 300 KB of output: each trailer check byte flipped, gzip ISIZE +- 1 and a
    member that fails to inflate.  Above, to bound the run time: one check byte flipped, and ISIZE +- 1 on every
    third gzip member.  Its members of more than BIG_MEMBER_BYTES send host decodes group by group."""
    items = []
    fills = ("random", "text", "zeros", "ff")
    for i, n in enumerate(cs.SWEEP):
        if n > cs.BIG_PIECES * cs.PIECE + 1:
            continue   # the big fold with many more pieces: part A
        fmts = ("gzip", "zlib") if n < cs.LARGE else (("gzip", "zlib")[i % 2],)
        for fmt in fmts:
            data = cs.content(fills[i % 4], n, seed=100 + i, text=text).tobytes()
            level = (0, 1, 6, 9)[i % 4] if n <= (1 << 20) + 1 else i % 2
            m = cs.member(data, fmt, level)
            items.append(("%s %d good" % (fmt, n), m, data, n))
            small = n <= 300000
            bad = cs.corruptions(m, fmt, n, flips=range(4) if small else (i % 4,), isize=small or i % 3 == 0,
                                 bad=small)
            items += [("%s %d %s" % (fmt, n, name), b, None, n) for name, b in bad]
    assert max(len(x[1]) for x in items) >= cs.BIG_MEMBER_BYTES
    return _with_oracle(o, items)


@pytest.fixture(scope="module")
def pipe_batch(o, text):
    """cs.pipeline_members: every member below BIG_MEMBER_BYTES, so host decodes take the host pipeline"""
    items = cs.pipeline_members(text)
    assert max(len(x[1]) for x in items) < cs.BIG_MEMBER_BYTES
    return _with_oracle(o, items)


def _category(s):
    return s if s in (0, 14, 18) else "other"


def _verify(names, outs, cats, get, lens, st, what):
    bad = []
    for i, (name, out, c) in enumerate(zip(names, outs, cats)):
        if _category(int(st[i])) != c:
            bad.append((name, int(st[i]), c))
        elif out is not None and (int(lens[i]) != len(out) or get(i) != out):
            bad.append((name, "bytes differ"))
    assert not bad, "%s: %d of %d wrong, e.g. %s" % (what, len(bad), len(names), bad[:8])


@pytest.mark.parametrize("mode", ["isize", "caller_sizes"])
def test_decode_verdicts_host(z, verify_batch, mode):
    """The group-by-group host path (the batch holds large members).  Sizes from the members (ISIZE, the sizing
    pass), or 2x the output from the caller: every buffer's capacity then ends in empty pieces."""
    base, offs, names, outs, cats, ns = verify_batch
    sizes = 2 * ns + np.uint64(7) if mode == "caller_sizes" else None
    ctx = z.Context()
    out, do, lens, st = ctx.uncompress_batch(base, offs, z.dfDetect, sizes=sizes)
    _verify(names, outs, cats, lambda i: out[int(do[i]):int(do[i]) + int(lens[i])].tobytes(), lens, st, mode)
    ctx.close()


def test_decode_verdicts_device(z, torch, verify_batch):
    base, offs, names, outs, cats, ns = verify_batch
    ctx = z.Context()
    ctx.set_stream(ctx.LEGACY_DEFAULT_STREAM)
    do = _offsets(2 * ns + np.uint64(7))
    d_src = torch.from_numpy(base.copy()).cuda()
    d_dst = torch.zeros(int(do[-1]) + 64, dtype=torch.uint8, device="cuda")
    lens, st = ctx.uncompress_batch_device(d_src.data_ptr(), offs, z.dfDetect, d_dst.data_ptr(), do)
    host = d_dst.cpu().numpy()
    _verify(names, outs, cats, lambda i: host[int(do[i]):int(do[i]) + int(lens[i])].tobytes(), lens, st, "device")
    ctx.close()


@pytest.mark.parametrize("sizes", ["isize", "caller_sizes"])
@pytest.mark.parametrize("gated", ["0", "1"])
def test_decode_verdicts_host_pipelines(z, pipe_batch, monkeypatch, gated, sizes):
    """The host pipeline, gated (one inflate launch behind the copy-in) and one launch per group, each group's
    checksum launch offsetting pieces, first pieces and partials: groups of about three pieces of output, so members
    of many pieces fill groups alone.  Caller sizes of 2x the output put empty pieces in every group."""
    base, offs, names, outs, cats, ns = pipe_batch
    monkeypatch.setenv("ZB200_UNC_GATED", gated)
    monkeypatch.setenv("ZB200_UNC_GROUP_BYTES", str(3 * cs.PIECE + 5))
    ctx = z.Context()
    monkeypatch.delenv("ZB200_UNC_GATED")
    monkeypatch.delenv("ZB200_UNC_GROUP_BYTES")
    out, do, lens, st = ctx.uncompress_batch(base, offs, z.dfDetect,
                                             sizes=2 * ns + np.uint64(7) if sizes == "caller_sizes" else None)
    _verify(names, outs, cats, lambda i: out[int(do[i]):int(do[i]) + int(lens[i])].tobytes(), lens, st,
            "gated=%s %s" % (gated, sizes))
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# C. the other callers

def test_inflate_batch_crc32_sweep(z, text):
    """Raw members of the sweep sizes into slots above and below their output (status 19 -> the one-by-one redo)"""
    sizes = cs.SMALL_SWEEP + [cs.BIG_PIECES * cs.PIECE + 1]
    datas = [cs.content(("random", "text", "ff")[i % 3], n, seed=200 + i, text=text).tobytes()
             for i, n in enumerate(sizes)]
    members = []
    for i, d in enumerate(datas):
        c = zlib.compressobj((1, 6, 0)[i % 3], zlib.DEFLATED, -15)
        members.append(c.compress(d) + c.flush())
    offs = _offsets([len(m) for m in members])
    base = np.frombuffer(b"".join(members), dtype=np.uint8)
    slots = [len(d) + (1 + i % 5) * 1000 if i % 2 or not d else len(d) - 1 for i, d in enumerate(datas)]
    ctx = z.Context()
    out, do, lens, crcs, st = ctx.inflate_batch_crc32(base, offs, slots)
    bad = [(len(d), int(st[i]), int(crcs[i]), zlib.crc32(d)) for i, d in enumerate(datas)
           if int(st[i]) != 0 or int(crcs[i]) != zlib.crc32(d) or int(lens[i]) != len(d)
           or out[int(do[i]):int(do[i]) + len(d)].tobytes() != d]
    assert not bad, bad[:8]
    ctx.close()


def _stored_member(fmt, data, cuts):
    """A member of stored blocks ending at every cut (blocks of at most 65535 bytes) -> (member, write ends): the
    compressed offsets at which each cut's blocks are complete."""
    head = b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff" if fmt == "gzip" else b"\x78\x01"
    parts, ends, pos = [head], [], len(head)
    lo = 0
    for k, hi in enumerate(cuts):
        while True:
            n = min(65535, hi - lo)
            final = k == len(cuts) - 1 and lo + n == hi
            blk = bytes([1 if final else 0]) + n.to_bytes(2, "little") + (n ^ 0xFFFF).to_bytes(2, "little")
            parts.append(blk + data[lo:lo + n])
            pos += len(blk) + n
            lo += n
            if lo == hi:
                break
        ends.append(pos)
    if fmt == "gzip":
        parts.append(zlib.crc32(data).to_bytes(4, "little") + (len(data) & 0xFFFFFFFF).to_bytes(4, "little"))
    else:
        parts.append(zlib.adler32(data).to_bytes(4, "big"))
    return b"".join(parts), ends


@pytest.mark.parametrize("fmt", ["gzip", "zlib"])
def test_decompress_stream_running_check(z, monkeypatch, capfd, fmt):
    """A launch at every write, writes ending where the stored blocks of each segment end: every launch checksums
    one segment of a share multiple, 65 536, the Adler modulus and around it, many pieces, and the host combine
    folds them (the launch log shows that every segment ends a launch); then the same member with its trailer check
    corrupted."""
    segs = [2048 * 17, 65536, 65521, 65522, 131072, 1, 65520, 32768 * 33 + 3, 2048 * 5, 17 * 65521 - 1, 3]
    data = cs.content("random", sum(segs), seed=300).tobytes()
    cuts = [int(c) for c in np.cumsum(segs)]
    member, ends = _stored_member(fmt, data, cuts)
    monkeypatch.setenv("ZB200_DSTREAM_BATCH_BYTES", "1")
    monkeypatch.setenv("ZB200_DSTREAM_LOG", "1")
    ctx = z.Context()
    monkeypatch.delenv("ZB200_DSTREAM_BATCH_BYTES")
    monkeypatch.delenv("ZB200_DSTREAM_LOG")
    assert zlib.decompress(member, 31 if fmt == "gzip" else 15) == data
    for corrupt in (False, True):
        m = bytearray(member)
        if corrupt:
            m[-8 if fmt == "gzip" else -1] ^= 0x5A
        got, code = [], 0
        capfd.readouterr()
        try:
            with z.DecompressStream(z.dfGzip if fmt == "gzip" else z.dfZlib, ctx) as s:
                lo = 0
                for hi in ends + [len(m)]:
                    got.append(s.write(bytes(m[lo:hi])))
                    lo = hi
                got.append(s.finish())
        except z.ZippyError as e:
            code = e.code
        if corrupt:
            assert code == 14, code
        else:
            assert code == 0 and b"".join(got) == data
            launch_ends = set(np.cumsum([int(x) for x in re.findall(r"zb200 dstream: .* out=(\d+)",
                                                                     capfd.readouterr().err)]).tolist())
            # a gzip stream holds its last 8 input bytes back as the possible trailer: where the write after a cut
            # is shorter than that (the 1-byte segment), the blocks before the cut are decoded in the launch of
            # that write, so the cut ends no launch of its own
            writes = np.diff([0] + ends + [len(m)])
            short = {c for c, w in zip(cuts, writes[1:]) if fmt == "gzip" and w < 8}
            assert short == ({cuts[4]} if fmt == "gzip" else set())
            assert set(cuts) - short <= launch_ends, sorted(set(cuts) - short - launch_ends)
    ctx.close()


def test_dictids_through_the_device_adler(z, text):
    """More than 256 KiB of named dictionary entries: their DICTIDs are Adler-32s from the checksum kernels, over
    runs of named entries broken by unnamed ones, and one entry larger than 256 MiB alone."""
    L = z._native.lib()
    named_sizes = [1, 3, 4095, 32768, 2048 * 17, 65521, 65536, 131072, 32768 * 33 + 3, (1 << 20) + 1,
                   (256 << 20) + 5, 2048 * 23]
    entries, of_entry = [], []
    for i, n in enumerate(named_sizes):
        if i % 3 == 1:
            entries.append(cs.content("random", 777 * i + 5, seed=400 + i).tobytes())   # named by no member
        of_entry.append(len(entries))
        entries.append(cs.content(("random", "ff", "text")[i % 3], n, seed=500 + i, text=text).tobytes())
    inputs = [text[1000 * i:1000 * i + 3000] for i in range(len(named_sizes) + 2)]
    dict_of = np.array(of_entry + [-1, of_entry[3]], dtype=np.int32)
    offs = _offsets([len(x) for x in inputs])
    base = np.frombuffer(b"".join(inputs), dtype=np.uint8)
    doffs = _offsets([len(e) for e in entries])
    dbase = np.frombuffer(b"".join(entries), dtype=np.uint8)
    out = np.empty(sum(len(x) for x in inputs) * 2 + 4096, dtype=np.uint8)
    oo = np.zeros(len(inputs) + 1, dtype=np.uint64)
    st = np.zeros(len(inputs), dtype=np.int32)
    ctx = z.Context()
    rc = L.zb200_compress_batch_dicts(ctx._h, base.ctypes.data, offs.ctypes.data, len(inputs), 1, z.dfZlib, 15,
                                      dbase.ctypes.data, doffs.ctypes.data, len(entries), dict_of.ctypes.data,
                                      out.ctypes.data, out.size, oo.ctypes.data, st.ctypes.data)
    assert rc == 0 and not st.any()
    for i, x in enumerate(inputs):
        m = out[int(oo[i]):int(oo[i + 1])].tobytes()
        j = int(dict_of[i])
        if j < 0:
            assert not m[1] & 0x20 and zlib.decompress(m) == x
            continue
        d = entries[j]
        assert m[1] & 0x20, i
        assert int.from_bytes(m[2:6], "big") == zlib.adler32(d), (i, len(d))
        dec = zlib.decompressobj(zdict=d)
        assert dec.decompress(m) + dec.flush() == x
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# D. the compress-side fold

def _trailer_ok(fmt, m, x):
    if fmt == "gzip":
        return int.from_bytes(m[-8:-4], "little") == zlib.crc32(x) and int.from_bytes(m[-4:], "little") == len(x) % (1 << 32)
    return int.from_bytes(m[-4:], "big") == zlib.adler32(x)


@pytest.fixture(scope="module")
def member_inputs(text):
    return [cs.content(("text", "random")[i % 2], n, seed=600 + i, text=text).tobytes()
            for i, n in enumerate(cs.MEMBER_SWEEP)]


@pytest.mark.parametrize("level,strategy", [(0, 0), (1, 0), (-2, 0), (-1, 0), (6, 0), (9, 0), (-1, 3), (-1, 4)],
                         ids=["L0", "L1", "Huffman", "Ldefault", "L6", "L9", "RLE", "FIXED"])
@pytest.mark.parametrize("fmt", ["gzip", "zlib"])
def test_member_trailers(z, member_inputs, fmt, level, strategy):
    """every member_classes length in one batch: 1, 2..32, 33..63, multiples of 32 and over 1024 chunks, exactly one
    and two chunks"""
    base = np.frombuffer(b"".join(member_inputs), dtype=np.uint8)
    offs = _offsets([len(x) for x in member_inputs])
    ctx = z.Context()
    out, oo = ctx.compress_batch(base, offs, level, z.dfGzip if fmt == "gzip" else z.dfZlib, strategy=strategy)
    bad = [len(x) for i, x in enumerate(member_inputs)
           if not _trailer_ok(fmt, out[int(oo[i]):int(oo[i + 1])].tobytes(), x)]
    assert not bad, bad
    for i in (0, 1, 3, 5):   # the short ones decode too
        m = out[int(oo[i]):int(oo[i + 1])].tobytes()
        assert zlib.decompress(m, 31 if fmt == "gzip" else 15) == member_inputs[i]
    ctx.close()


@pytest.mark.parametrize("level", [1, -1])
@pytest.mark.parametrize("fmt", ["gzip", "zlib"])
def test_compress_stream_carry_in(z, text, monkeypatch, fmt, level):
    """a launch at every write, writes cut so the carry-in is one chunk, two, a ragged tail, the Adler modulus, ..."""
    monkeypatch.setenv("ZB200_STREAM_BATCH_BYTES", "1")
    ctx = z.Context()
    monkeypatch.delenv("ZB200_STREAM_BATCH_BYTES")
    data = cs.content("text", sum(cs.STREAM_CUTS), text=text).tobytes()
    parts = []
    with z.CompressStream(level, z.dfGzip if fmt == "gzip" else z.dfZlib, fname_len=0, ctx=ctx) as s:
        lo = 0
        for w in cs.STREAM_CUTS:
            parts.append(s.write(data[lo:lo + w]))
            lo += w
        parts.append(s.finish())
    m = b"".join(parts)
    assert _trailer_ok(fmt, m, data)
    assert zlib.decompress(m, 31 if fmt == "gzip" else 15) == data
    ctx.close()


def test_member_past_4_GiB_device(z, torch, text):
    _need_free(torch, 12 << 30)
    n = cs.HUGE_MEMBER
    host = np.resize(np.frombuffer(text, dtype=np.uint8), n)
    host[::4097] = 0xA5          # not a pure period of the corpus
    L = z._native.lib()
    cap = int(L.zb200_compress_bound(n, z.dfGzip)) + 4096
    ctx = z.Context()
    ctx.set_stream(ctx.LEGACY_DEFAULT_STREAM)
    d_src = torch.from_numpy(host).cuda()
    d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    oo = ctx.compress_batch_device(d_src.data_ptr(), np.array([0, n], dtype=np.uint64), 1, z.dfGzip,
                                   d_dst.data_ptr(), cap)
    del d_src
    end = int(oo[1])
    tail = d_dst[end - 8:end].cpu().numpy().tobytes()
    assert int.from_bytes(tail[:4], "little") == zlib.crc32(host)
    assert int.from_bytes(tail[4:], "little") == n % (1 << 32)
    ctx.close()
