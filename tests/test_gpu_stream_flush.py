"""Sync and full flushes of compress streams (zb200_compress_stream_flush, CompressStream.flush).

The flush offsets cut a member into flush segments, each cut into 64 KiB chunks from its own start; levels -1 and
2..9 see min(32 KiB, bytes since the member start or the last full flush) of history, so a chunk after a flush may
have any history length, and k_lz2's segment grid is anchored on the chunk start (DESIGN.md section 8 h).

The CPU part checks the schedule model (tests/native/lz2_schedule_model.c: lz2_model_schedule, the rules of
tests/native/lz2_model.c with the segment grid anchored on the chunk start) on its own: with one chunk per 64 KiB
and no resets it is lz2_model; with any cuts and resets its tokens rebuild the member, no match
crosses a reset, and the odd history lengths are reached and matched into.  The GPU part checks the stream: no
change without a flush, the prefix property after every flush, full-flush independence, the finished member,
determinism, the tokens against the model, and the error contract."""
import ctypes
import os
import random
import struct
import subprocess
import zlib

import numpy as np
import pytest

from tests import deflate_tokens as dt
from tests import deflate_writer as dw
from tests import util
from tests.test_gpu_lz2_model import COUNTERS, Model, decode, encode

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "native", "lz2_schedule_model.c")   # includes lz2_model.c: exports both entry points
CHUNK, SUB = 65536, 8192
LZ_LEVELS = [-1, 2, 3, 4, 5, 6, 7, 8, 9]
ALL_LEVELS = [-2, 0, 1, -1] + list(range(2, 10))
FORMATS = ("gzip", "zlib", "deflate")
WBITS = {"gzip": 31, "zlib": 15, "deflate": -15}
SYNC, FULL = 2, 3
HIST_LENGTHS = (1, 4095, 8191, 8193, 20000, 32767)


# ---------------------------------------------------------------------- the schedule and the model
def schedule(n, flushes):
    """Chunks of a member of n bytes flushed at `flushes` ([(offset, mode)], ascending; a flush with nothing new
    is a no-op) -> (bounds, hist_from, sizes of the flush segments' chunks): what the stream compresses."""
    bounds, hist_from, lo, reset = [0], [], 0, 0
    for off, mode in flushes:
        if off > lo:
            for c in range(lo, off, CHUNK):
                bounds.append(min(off, c + CHUNK))
                hist_from.append(reset)
            lo = off
            if mode == FULL:
                reset = off
    for c in range(lo, n, CHUNK):     # finish: the rest ...
        bounds.append(min(n, c + CHUNK))
        hist_from.append(reset)
    if n == lo:                       # ... or an empty last chunk (no input, or finish right after a flush)
        bounds.append(n)
        hist_from.append(reset)
    return bounds, hist_from


class ScheduleModel(Model):
    def __init__(self, so):
        super().__init__(so)
        self.L.lz2_model_schedule.restype = ctypes.c_int64
        self.L.lz2_model_schedule.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p,
                                              ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint64,
                                              ctypes.c_void_p, ctypes.c_void_p]

    def run_schedule(self, member, level, bounds, hist_from, counters=None):
        """-> one array of encoded tokens per chunk of the schedule."""
        n, nch = len(member), len(hist_from)
        b = np.array(bounds, dtype=np.uint64)
        h = np.array(hist_from, dtype=np.uint64)
        tok = np.zeros(n + 16, dtype=np.uint32)
        per = np.zeros(nch, dtype=np.uint32)
        cnt = np.zeros(len(COUNTERS), dtype=np.uint64)
        got = self.L.lz2_model_schedule(bytes(member), n, level, b.ctypes.data, h.ctypes.data, nch, tok.ctypes.data,
                                        tok.size, per.ctypes.data, cnt.ctypes.data)
        assert got >= 0, got
        if counters is not None:
            for k, v in zip(COUNTERS, cnt.tolist()):
                counters[k] = counters.get(k, 0) + v
        edges = np.concatenate([[0], np.cumsum(per.astype(np.int64))])
        assert edges[-1] == got
        return [tok[edges[i]:edges[i + 1]] for i in range(nch)]


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lz2_schedule") / "liblz2_model.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, SRC])
    return ScheduleModel(so)


def _seven_bit(rng, n):
    """High-entropy bytes (7 random bits each): a Huffman block beats a stored one, so the tokens are written."""
    return bytearray((np.frombuffer(rng.randbytes(n), dtype=np.uint8) | 0x80).tobytes())


def history_member(h, seed=0):
    """A member flushed at h: h bytes of history, then a chunk that copies the member's first 300 bytes (the
    oldest history byte, in the partial segment 0 of the chunk's grid) at distance <= 32768, and more history
    slices further on."""
    rng = random.Random(0x4157 + h + seed)
    x = _seven_bit(rng, h + 40000)
    p0 = max(1, min(1000, 32768 - h))
    x[h + p0:h + p0 + 300] = x[0:300]
    for src in (h // 2, max(0, h - 100)):
        dst = h + 3000 + src % 5000
        x[dst:dst + 200] = x[src:src + 200]
    return bytes(x), p0


def _match_sources(chunks, bounds):
    """-> [(member position of the match, distance, length)] of every match of every chunk"""
    out = []
    for k, arr in enumerate(chunks):
        pos = bounds[k]
        for t in decode(arr):
            if isinstance(t, int):
                pos += 1
            else:
                out.append((pos, t[1], t[0], k))
                pos += t[0]
    return out


def _check_schedule_tokens(member, chunks, bounds, hist_from):
    for k, arr in enumerate(chunks):
        toks = decode(arr)
        assert sum(1 if isinstance(t, int) else t[0] for t in toks) == bounds[k + 1] - bounds[k], k
    for pos, d, ln, k in _match_sources(chunks, bounds):
        assert 4 <= ln <= 258 and 1 <= d <= 32768, (pos, d, ln)
        assert pos - d >= hist_from[k], ("a match reaches across a reset or before the member", pos, d, k)
        p = pos - bounds[k]
        assert p // SUB == (p + ln - 1) // SUB, ("match across a sub-chunk end", pos, ln)
    assert dt.rebuild([dt.Block(2, False, 0, 0, decode(a)) for a in chunks]) == member


def _fixed_stream(chunks):
    blocks = []
    for k, arr in enumerate(chunks):
        last = k == len(chunks) - 1
        blocks.append(dw.Fixed(decode(arr), final=last))
        if not last:
            blocks.append(dw.Stored(b"", final=False))
    return dw.raw(blocks)


def _cpu_inputs(corpus):
    rng = random.Random(0xF1)
    T = util.text_corpus(corpus)
    o = rng.randrange(len(T) - 300000)
    return {"text": T[o:o + 250001], "html": corpus["html"][:150000],
            "mix": T[:60000] + bytes(_seven_bit(rng, 30000)) + bytes(20000) + T[60000:110000]}


def test_schedule_helper():
    assert schedule(10, []) == ([0, 10], [0])
    assert schedule(0, []) == ([0, 0], [0])
    assert schedule(200000, [(1, SYNC), (70000, FULL)]) == ([0, 1, 65537, 70000, 135536, 200000], [0, 0, 0, 70000, 70000])
    assert schedule(5, [(5, SYNC)]) == ([0, 5, 5], [0, 0])
    assert schedule(5, [(0, SYNC), (2, FULL), (2, SYNC)]) == ([0, 2, 5], [0, 2])


@pytest.mark.parametrize("level", LZ_LEVELS)
def test_model_schedule_without_flushes_is_lz2_model(model, corpus, level):
    """One segment per 64 KiB and no resets: lz2_model's tokens exactly."""
    for name, x in _cpu_inputs(corpus).items():
        n = len(x)
        bounds = list(range(0, n, CHUNK)) + [n]
        got = model.run_schedule(x, level, bounds, [0] * (len(bounds) - 1))
        want = model.run(x, level)
        assert len(got) == len(want) and all(np.array_equal(g, w) for g, w in zip(got, want)), name


@pytest.mark.parametrize("level", LZ_LEVELS)
def test_model_schedule_cuts_and_resets(model, corpus, level):
    """Arbitrary cuts and resets: the tokens rebuild the member, no match crosses a reset or reaches before the
    member, and packed with fixed codes and sync blocks they inflate with zlib."""
    rng = random.Random(0x5C + level)
    for name, x in _cpu_inputs(corpus).items():
        n = len(x)
        for trial in range(3):
            offs = sorted({rng.randrange(1, n) for _ in range(6)} | {8191, 20000, 32769})
            flushes = [(f, rng.choice((SYNC, FULL))) for f in offs]
            bounds, hist_from = schedule(n, flushes)
            chunks = model.run_schedule(x, level, bounds, hist_from)
            _check_schedule_tokens(x, chunks, bounds, hist_from)
            assert zlib.decompress(_fixed_stream(chunks), -15) == x, (name, flushes)


@pytest.mark.parametrize("level", LZ_LEVELS)
def test_model_reaches_odd_history_lengths(model, level):
    """Chunks with 1, 4095, 8191, 8193, 20000 and 32767 bytes of history match into that history, down to its
    oldest byte (the partial first segment of the chunk's grid)."""
    for h in HIST_LENGTHS:
        x, p0 = history_member(h)
        bounds, hist_from = schedule(len(x), [(h, SYNC)])
        assert bounds[1] == h and min(32768, bounds[1] - hist_from[1]) == h
        chunks = model.run_schedule(x, level, bounds, hist_from)
        _check_schedule_tokens(x, chunks, bounds, hist_from)
        into = [(pos, d) for pos, d, ln, k in _match_sources(chunks, bounds) if k == 1 and pos - d < h]
        assert into, (h, "no match into the history")
        # the copy of the member's first 300 bytes is matched into the partial first segment of the grid (a
        # direct-mapped static entry may hold a later position of the same hash, so not necessarily at byte 0)
        part = min(300, h % SUB or SUB)
        assert [1 for pos, d in into if h + p0 <= pos < h + p0 + 300 and pos - d < part], (h, into[:5])
        # after a full flush at h, the same chunk sees no history
        bounds, hist_from = schedule(len(x), [(h, FULL)])
        chunks = model.run_schedule(x, level, bounds, hist_from)
        _check_schedule_tokens(x, chunks, bounds, hist_from)
        assert not [1 for pos, d, ln, k in _match_sources(chunks, bounds) if k == 1 and pos - d < h]


# ---------------------------------------------------------------------- GPU: the stream
@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


def _df(z, fmt):
    return {"gzip": z.dfGzip, "zlib": z.dfZlib, "deflate": z.dfDeflate}[fmt]


@pytest.fixture(scope="module")
def contexts(z):
    """'default': the 64 MiB threshold; 'every': a launch whenever more than one chunk is pending; 'three':
    launches of about three chunks."""
    mp = pytest.MonkeyPatch()
    ctxs = {"default": z.Context()}
    try:
        for name, v in (("every", "1"), ("three", str(3 * CHUNK + 5))):
            mp.setenv("ZB200_STREAM_BATCH_BYTES", v)
            ctxs[name] = z.Context()
    finally:
        mp.undo()
    yield ctxs
    for c in ctxs.values():
        c.close()


def flushed(z, ctx, data, level, fmt, flushes, fname_len=3, splits=1, seed=0, on_flush=None):
    """Compress data with flushes at [(offset, mode)] -> (member, [output length after each flush]).  Between
    two flushes the input goes in `splits` writes at seeded offsets; on_flush(offset, output of the flush and
    the writes before it) is called after every flush."""
    rng = random.Random(seed)
    out, ends, lo = bytearray(), [], 0
    with z.CompressStream(level, _df(z, fmt), fname_len, ctx) as s:
        for off, mode in list(flushes) + [(len(data), None)]:
            cuts = sorted({lo, off, *(rng.randrange(lo, off + 1) for _ in range(splits - 1))})
            last = len(out) if not ends else ends[-1]
            for a, b in zip(cuts[:-1], cuts[1:]):
                out += s.write(data[a:b])
            lo = off
            if mode is None:
                break
            out += s.flush(mode)
            ends.append(len(out))
            if on_flush:
                on_flush(off, bytes(out[last:]))
        out += s.finish()
    return bytes(out), ends


def one_shot(ctx, z, data, level, fmt, fname_len=3):
    base, offs = z._pack([data])
    out, oo = ctx.compress_batch(base, offs, level, _df(z, fmt), [fname_len])
    return out[:int(oo[1])].tobytes()


def check_member(z, fmt, comp, data):
    """zlib, the oracle and uncompress decode the member; the trailer holds the CRC-32 / Adler-32 and ISIZE."""
    from oracle import oracle as o
    assert zlib.decompress(comp, WBITS[fmt]) == data
    assert o.uncompress(comp, {"gzip": o.dfGzip, "zlib": o.dfZlib, "deflate": o.dfDeflate}[fmt]) == data
    assert z.uncompress(comp, _df(z, fmt)) == data
    if fmt == "gzip":
        assert struct.unpack("<II", comp[-8:]) == (zlib.crc32(data), len(data) & 0xffffffff)
    elif fmt == "zlib":
        assert struct.unpack(">I", comp[-4:])[0] == zlib.adler32(data)


@pytest.fixture(scope="module")
def inputs(corpus):
    rng = random.Random(0xF5)
    T = util.text_corpus(corpus)
    o = rng.randrange(len(T) - 400000)
    text = T[o:o + 300001]
    return {"text": text, "random": rng.randbytes(150003), "zeros": bytes(140000),
            "mix": text[:70000] + rng.randbytes(40000) + bytes(50000) + text[70000:120000]}


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("level", ALL_LEVELS)
def test_flush_at_chunk_boundaries_changes_nothing(z, contexts, inputs, level, fmt):
    """Sync flushes at multiples of 65536 (full flushes too at the levels without history) give compress_batch's
    bytes; so does a stream whose every flush has nothing new."""
    data = inputs["text"][:3 * CHUNK + 1234]
    want = one_shot(contexts["default"], z, data, level, fmt)
    modes = (SYNC, FULL) if level in (0, 1, -2) else (SYNC,)
    for mode in modes:
        for ctx in ("default", "every"):
            got, _ = flushed(z, contexts[ctx], data, level, fmt, [(c, mode) for c in (CHUNK, 2 * CHUNK, 3 * CHUNK)])
            assert got == want, (mode, ctx)
    got, ends = flushed(z, contexts["default"], data, level, fmt, [(0, SYNC), (0, FULL)])
    assert got == want and ends == [0, 0]


SCHEDULES = {
    "1_5000": [1, 5000],
    "8k": [8191, 8192, 8193],
    "32k": [32767, 32768, 32769],
    "64k": [65535, 65537],
}


def _prefix_checker(fmt, data, seen):
    """on_flush callback: the output so far, through one zlib.decompressobj, is the input so far."""
    d = zlib.decompressobj(WBITS[fmt])
    state = {"off": 0}

    def on_flush(off, new):
        got = d.decompress(new)
        assert got == data[state["off"]:off], (off, state["off"], len(got))
        state["off"] = off
        seen.append(off)
    return on_flush


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("level", [-2, 0, 1, -1, 2, 6, 9])
def test_prefix_property(z, contexts, inputs, level, fmt):
    """After every flush, what the stream has emitted decodes to everything written so far; the member decodes."""
    rng = random.Random(0xB0 + level)
    for name, data in inputs.items():
        n = len(data)
        scheds = dict(SCHEDULES)
        scheds["random"] = sorted({rng.randrange(1, n) for _ in range(8)})
        for sname, offs in scheds.items():
            for mode in (SYNC, FULL):
                seen = []
                flushes = [(o, mode) for o in offs if o < n]
                comp, _ = flushed(z, contexts["every" if sname == "random" else "default"], data, level, fmt,
                                  flushes, splits=2, seed=sum(offs), on_flush=_prefix_checker(fmt, data, seen))
                assert seen == [o for o, _ in flushes]
                check_member(z, fmt, comp, data)


@pytest.mark.gpu
@pytest.mark.parametrize("level,mode", [(-1, SYNC), (1, FULL), (9, FULL)])
def test_prefix_property_every_100_bytes(z, contexts, corpus, level, mode):
    T = util.text_corpus(corpus)
    data = T[:1 << 20]
    seen = []
    flushes = [(o, mode) for o in range(100, len(data), 100)]
    comp, _ = flushed(z, contexts["default"], data, level, "gzip", flushes, on_flush=_prefix_checker("gzip", data, seen))
    assert len(seen) == len(flushes)
    check_member(z, "gzip", comp, data)


@pytest.mark.gpu
def test_flush_edges(z, contexts, inputs):
    """A flush before any input emits nothing; two flushes in a row, the second emits b""; a flush right after a
    threshold launch; finish right after a flush writes the empty final block and the trailer."""
    data = inputs["text"][:5 * CHUNK + 77]
    for fmt in FORMATS:
        for level in (-1, 1, 0):
            with z.CompressStream(level, _df(z, fmt), 0, contexts["three"]) as s:
                out = bytearray(s.flush())
                assert out == b""
                out += s.write(data[:4 * CHUNK + 10])          # a threshold launch: 4 chunks out, 10 bytes held
                assert len(out) > 0
                f = s.flush()
                assert f and s.flush() == b"" and s.flush(FULL) == b""
                out += f
                assert zlib.decompressobj(WBITS[fmt]).decompress(bytes(out)) == data[:4 * CHUNK + 10]
                out += s.write(data[4 * CHUNK + 10:])
                out += s.flush(FULL)
                tail = s.finish()
                out += tail
            if fmt != "deflate":
                body = tail[:-8] if fmt == "gzip" else tail[:-4]
            else:
                body = tail
            assert body == (b"\x01\x00\x00\xff\xff" if level == 0 else b"\x03\x00"), (fmt, level, tail)
            check_member(z, fmt, bytes(out), data)


@pytest.mark.gpu
@pytest.mark.parametrize("level", [-2, 0, 1, -1, 4, 9])
def test_full_flush_independence(z, contexts, inputs, level):
    """The bytes after each full flush inflate, with a fresh raw inflater, to the input after that flush."""
    rng = random.Random(0xFF + level)
    for name, data in inputs.items():
        for fmt in FORMATS:
            n = len(data)
            offs = sorted({8193, 40000, rng.randrange(1, n), rng.randrange(1, n)})
            flushes = [(o, FULL) for o in offs]
            comp, ends = flushed(z, contexts["default"], data, level, fmt, flushes)
            trailer = {"gzip": 8, "zlib": 4, "deflate": 0}[fmt]
            for (off, _), e in zip(flushes, ends):
                d = zlib.decompressobj(-15)
                assert d.decompress(comp[e:]) == data[off:], (name, fmt, off)
                assert d.eof and len(d.unused_data) == trailer
            check_member(z, fmt, comp, data)


@pytest.mark.gpu
@pytest.mark.parametrize("level", [-2, 1, -1, 6])
def test_determinism(z, contexts, inputs, level):
    """The same flush schedule under different write splits and thresholds gives identical bytes."""
    data = inputs["mix"]
    rng = random.Random(0xDE)
    flushes = [(o, rng.choice((SYNC, FULL))) for o in sorted({rng.randrange(1, len(data)) for _ in range(7)} | {70000})]
    ref = None
    for ctx in ("default", "every", "three"):
        for splits, seed in ((1, 0), (4, 1), (9, 2)):
            got, _ = flushed(z, contexts[ctx], data, level, "gzip", flushes, splits=splits, seed=seed)
            ref = ref or got
            assert got == ref, (ctx, splits)
    check_member(z, "gzip", ref, data)


def split_chunks(blocks, sizes):
    """The blocks of a flushed member -> its chunks, given each chunk's size: a fixed / dynamic block (followed,
    unless it is the last, by the empty stored block) or stored blocks that together hold the chunk."""
    out, i = [], 0
    for s in sizes:
        b = blocks[i]
        if b.btype == 0:
            toks = []
            while True:
                toks += blocks[i].tokens
                i += 1
                if len(toks) >= s or blocks[i - 1].final:
                    break
            assert len(toks) == s
            out.append(dt.Chunk(0, toks))
            continue
        assert b.size() == s, (b.size(), s)
        out.append(dt.Chunk(b.btype, b.tokens))
        i += 1
        if not b.final:
            j = blocks[i]
            assert j.btype == 0 and not j.tokens and not j.final
            i += 1
    assert i == len(blocks) and blocks[-1].final
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("level", LZ_LEVELS)
def test_kernel_tokens_equal_the_model(z, contexts, model, corpus, level):
    """Every chunk of flushed members, with histories of 1, 4095, 8191, 8193, 20000 and 32767 bytes (after a sync
    flush) and none (after a full flush), holds the model's tokens."""
    T = util.text_corpus(corpus)
    cases = []
    for h in HIST_LENGTHS:
        x, _ = history_member(h)
        cases += [(x, [(h, SYNC)]), (x, [(h, FULL)])]
        y = T[h * 3:h * 3 + h] + T[:80000]                 # text: the history is matched into everywhere
        cases.append((y, [(h, SYNC), (h + 30000, SYNC), (h + 30001, FULL)]))
    rng = random.Random(0x70 + level)
    x = T[100000:400000]
    cases.append((x, [(o, rng.choice((SYNC, FULL))) for o in sorted({rng.randrange(1, len(x)) for _ in range(10)})]))
    compared = stored = 0
    into = set()
    bad = []
    for ci, (x, flushes) in enumerate(cases):
        comp, _ = flushed(z, contexts["every"], x, level, "deflate", flushes)
        bounds, hist_from = schedule(len(x), flushes)
        want = model.run_schedule(x, level, bounds, hist_from)
        got = split_chunks(dt.parse(comp), [bounds[k + 1] - bounds[k] for k in range(len(hist_from))])
        assert len(got) == len(want)
        for k, (g, w) in enumerate(zip(got, want)):
            if g.btype == 0:
                assert bytes(g.tokens) == x[bounds[k]:bounds[k + 1]]
                stored += 1
                continue
            compared += 1
            ga = encode(g.tokens)
            if not np.array_equal(ga, w):
                bad.append((ci, k, bounds[k], hist_from[k]))
        for pos, d, ln, k in _match_sources(want, bounds):
            hb = min(32768, bounds[k] - hist_from[k])
            if pos - d < bounds[k] and hb in HIST_LENGTHS:
                into.add(hb)
    print("level %d: %d chunks compared, %d stored" % (level, compared, stored))
    assert not bad, bad[:10]
    assert compared >= 50 and compared >= 3 * stored
    assert into == set(HIST_LENGTHS), into


@pytest.mark.gpu
def test_error_contract(z, contexts, inputs):
    """An unknown mode and a flush after finish: ZB200_ERR_ARG; a too-small dst consumes nothing, and the retry
    gives the bytes an undisturbed stream gives."""
    from zippy_b200 import _native
    L = _native.lib()
    data = inputs["text"][:100000]
    with z.CompressStream(-1, z.dfGzip, 2, contexts["default"]) as s:
        s.write(data[:1000])
        for mode in (0, 1, 4, 5, -1):
            with pytest.raises(z.ZippyError) as e:
                s.flush(mode)
            assert e.value.code == 22
        s.finish()
        with pytest.raises(z.ZippyError) as e:
            s.flush()
        assert e.value.code == 22
    want, _ = flushed(z, contexts["default"], data, -1, "gzip", [(40000, SYNC), (70000, FULL)], fname_len=2)
    out = bytearray()
    with z.CompressStream(-1, z.dfGzip, 2, contexts["default"]) as s:
        for lo, hi, mode in ((0, 40000, SYNC), (40000, 70000, FULL)):
            out += s.write(data[lo:hi])
            buf = np.zeros(64, dtype=np.uint8)
            m = ctypes.c_size_t(7)
            assert L.zb200_compress_stream_flush(s._h, mode, buf.ctypes.data, buf.size, ctypes.byref(m)) == 19
            assert m.value == 0
            assert L.zb200_compress_stream_flush(s._h, mode, None, 0, ctypes.byref(m)) == 19
            cap = L.zb200_compress_stream_bound(s._h, 0)
            buf = np.zeros(cap, dtype=np.uint8)
            assert L.zb200_compress_stream_flush(s._h, mode, buf.ctypes.data, buf.size, ctypes.byref(m)) == 0
            assert 0 < m.value <= cap
            out += buf[:m.value].tobytes()
        out += s.write(data[70000:])
        out += s.finish()
    assert bytes(out) == want
    check_member(z, "gzip", want, data)
