"""The geometry of the checksum kernels (k_piece_checksum, k_piece_fold, k_buffer_combine, k_buffer_combine_big in
zb_inflate.cu, k_member_check in zb_deflate.cu) and the buffer shapes that reach each of their paths.

The constants are parsed from the sources, so a change to one of them moves the sweep with it or fails
tests/test_checksum_shapes.py instead of quietly leaving a path untested.  shape_classes / member_classes name the
structural paths a buffer / compressed member of a given length takes; SWEEP is a size list that hits every one.
"""
import os
import re
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "zippy_b200", "csrc")


def _define(fname, name):
    with open(os.path.join(CSRC, fname)) as f:
        m = re.search(r"^#define\s+%s\s+(\d+)u?\b" % re.escape(name), f.read(), re.M)
    if m is None:
        raise AssertionError("#define %s not found in %s" % (name, fname))
    return int(m.group(1))


PIECE = _define("zb_kernels.h", "ZB_CK_PIECE_BYTES")          # bytes per piece
BIG_PIECES = _define("zb_kernels.h", "ZB_CK_BIG_PIECES")      # above this many pieces: k_buffer_combine_big
CK_THREADS = _define("zb_inflate.cu", "CK_THREADS")            # k_piece_checksum<false>
CK_THREADS_ADLER = _define("zb_inflate.cu", "CK_THREADS_ADLER")  # k_piece_checksum<true> (adler32 calls)
CKB_THREADS = _define("zb_inflate.cu", "CKB_THREADS")          # k_buffer_combine_big
CHUNK = _define("zb_common.h", "ZB_CHUNK_BYTES")               # compress chunk (k_member_check)
ADLER_MOD = _define("zb_crc.h", "ZB_ADLER_MOD")


def _big_member_bytes():
    with open(os.path.join(CSRC, "zb_api.cu")) as f:
        m = re.search(r"uint64_t big_member_bytes = (\d+)ull << (\d+);", f.read())
    if m is None:
        raise AssertionError("big_member_bytes not found in zb_api.cu")
    return int(m.group(1)) << int(m.group(2))


# a host batch decode with a member of at least this many compressed bytes goes group by group; below it, every
# member of the batch goes through the host pipeline (gated or one launch per group)
BIG_MEMBER_BYTES = _big_member_bytes()

COMBINE_LANES = 32                     # k_buffer_combine: one warp per buffer, lane j folds pieces j, j + 32, ...
MEMBER_LANES = 32                      # k_member_check: one warp per member, 32 contiguous runs of chunks


def share_bytes(adler_only):
    """bytes per warp and piece on the Adler / ragged paths: 2 KiB (16 warps), 4 KiB in the Adler-only kernel"""
    return PIECE // ((CK_THREADS_ADLER if adler_only else CK_THREADS) // 32)


def n_pieces(length):
    return (length + PIECE - 1) // PIECE


def shape_classes(length, kind, adler_only=False):
    """The structural classes a buffer of `length` bytes hits in the standalone / verify checksum.
    kind: "crc32" or "adler32"; adler_only: the Adler-only instantiation (the adler32 calls)."""
    assert kind in ("crc32", "adler32") and not (adler_only and kind == "crc32")
    c = set()
    np_ = n_pieces(length)
    last = length - (np_ - 1) * PIECE if np_ else 0
    wb = share_bytes(adler_only)
    if length == 0:
        c.add("empty")
    elif length < 4:
        c.add("short")
    if 0 < last < PIECE:
        c.add("ragged")
        if last % wb == 0:
            c.add("ragged_share_multiple")     # the after-shift of every warp is a whole number of shares
        if last % 4:
            c.add("ragged_len_mod4")
        if last > wb:
            c.add("ragged_several_warps")
    if last == PIECE:
        c.add("full_last")
    if length >= PIECE:
        c.add("full_piece")
    if length == CHUNK:
        c.add("exactly_chunk")                 # ck_finish's shortcut
    if length == 2 * CHUNK:
        c.add("exactly_two_chunks")
    if np_ <= BIG_PIECES:
        if np_ > COMBINE_LANES:
            c.add("lane_ge32_ragged" if last < PIECE else "lane_ge32_full")
        if np_ > 2 * COMBINE_LANES:
            c.add("lane_horner_ge3")           # some lane folds three pieces or more
        if np_ == BIG_PIECES:
            c.add("exactly_big_pieces")
    else:
        c.add("big_fold")
        if last < PIECE and np_ - 1 >= CKB_THREADS:
            c.add("big_fold_ragged_ge_threads")
        if last == PIECE:
            c.add("big_fold_full_last")
        if np_ - 1 >= 2 * CKB_THREADS:
            c.add("big_fold_horner_ge3")
    if length >= 1 << 32:
        c.add("ge_4GiB")
    if kind == "adler32" and length >= ADLER_MOD:
        c.add("mod_p_%s" % {0: "0", 1: "1", ADLER_MOD - 1: "m1"}.get(length % ADLER_MOD, "other"))
    return c


# the classes every kind must reach with the sweep (and the huge sizes)
def required_shape_classes(kind, adler_only=False):
    req = {"empty", "short", "ragged", "ragged_share_multiple", "ragged_len_mod4", "ragged_several_warps", "full_last",
           "full_piece", "exactly_chunk", "exactly_two_chunks", "lane_ge32_ragged", "lane_ge32_full", "lane_horner_ge3",
           "exactly_big_pieces", "big_fold", "big_fold_ragged_ge_threads", "big_fold_full_last", "ge_4GiB"}
    if kind == "adler32":
        req |= {"mod_p_0", "mod_p_1", "mod_p_m1"}
    return req


def member_classes(length):
    """The classes a compressed member of `length` input bytes hits in k_member_check: its chunk count against the
    32-lane split and the shuffle tree, and the trailer's shift."""
    c = set()
    chunks = max(1, (length + CHUNK - 1) // CHUNK)
    if chunks == 1:
        c.add("chunks_1")
    elif chunks <= MEMBER_LANES:
        c.add("chunks_2_32")               # one chunk per lane, empty lanes in the tree
    elif chunks < 2 * MEMBER_LANES:
        c.add("chunks_33_63")              # two chunks on the first lanes, one on the last busy one, empty lanes
    if chunks > MEMBER_LANES and chunks % MEMBER_LANES == 0:
        c.add("chunks_multiple_of_32")     # every lane equally busy
    if chunks > 1024:
        c.add("chunks_gt_1024")
    if length and length % CHUNK == 0:
        c.add("whole_chunks")
    if length == CHUNK:
        c.add("exactly_chunk")             # the trailer's sub_mul[0] shortcut
    if length == 2 * CHUNK:
        c.add("exactly_two_chunks")        # the trailer's generic shift
    if length % CHUNK and chunks > 1:
        c.add("ragged_last_chunk")
    if length >= 1 << 32:
        c.add("ge_4GiB")
    return c


REQUIRED_MEMBER_CLASSES = {"chunks_1", "chunks_2_32", "chunks_33_63", "chunks_multiple_of_32", "chunks_gt_1024",
                           "whole_chunks", "exactly_chunk", "exactly_two_chunks", "ragged_last_chunk"}


def _sweep():
    s = set(range(0, 9))
    for c in (128, 2048, 4096, PIECE, CHUNK):
        s |= {c - 1, c, c + 1}
    s.add(2 * CHUNK)
    s |= {2048 * j for j in range(17, 32)}            # ragged last pieces of every share count (2 KiB multiples)
    for k in (2, 15, 16, 31, 32, 33, 63, 64, 65):
        s |= {PIECE * k + d for d in (0, 1, 3, 2048, 6144)}
    s |= {(1 << 20) - 1, (1 << 20) + 1}
    s |= {ADLER_MOD - 1, ADLER_MOD, ADLER_MOD + 1, 17 * ADLER_MOD, 17 * ADLER_MOD + 1, 17 * ADLER_MOD - 1}
    s |= {BIG_PIECES * PIECE + d for d in (-1, 0, 1)}
    s |= {3 * CKB_THREADS * PIECE + d for d in (-1, 0, 1)}
    return sorted(s)


SWEEP = _sweep()
LARGE = BIG_PIECES * PIECE - 1        # SWEEP sizes at or above this are the multi-MiB buffers of the big fold
SMALL_SWEEP = [n for n in SWEEP if n < LARGE]
HUGE = [(1 << 32) + 4097]             # a standalone checksum past 4 GiB (skipped without the memory)
MEMBER_SWEEP = [0, 1, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK, 2 * CHUNK + 7, 31 * CHUNK + 5, 32 * CHUNK, 33 * CHUNK,
                33 * CHUNK + 1, 40 * CHUNK + 77, 63 * CHUNK, 64 * CHUNK, 1025 * CHUNK + 3]
HUGE_MEMBER = (1 << 32) + (1 << 20) + 3
# compress-stream write cuts: the carry-in (the member's bytes before a launch) at a chunk, two chunks, a ragged
# tail, the Adler modulus and a span of many chunks
STREAM_CUTS = [CHUNK, 1, CHUNK - 1, 2 * CHUNK, ADLER_MOD, 3, 40 * CHUNK + 5, CHUNK, 2 * CHUNK + 1]


def content(kind, n, seed=0, text=b""):
    """n bytes: "random" (seeded), "zeros", "ff" (the largest Adler sums), "text" (`text` repeated) or "sparse"
    (zeros with a seeded random byte every 4093 bytes: compresses about 600:1, and unlike zeros its raw CRC-32 is
    not 0, so a wrong shift of it shows)"""
    if kind == "sparse":
        a = np.zeros(n, np.uint8)
        a[::4093] = np.random.default_rng(seed).integers(0, 256, a[::4093].size, dtype=np.uint8)
        return a
    if kind == "random":
        return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)
    if kind == "zeros":
        return np.zeros(n, np.uint8)
    if kind == "ff":
        return np.full(n, 0xFF, np.uint8)
    if kind == "text":
        t = np.frombuffer(text, np.uint8)
        return np.resize(t, n) if n else np.zeros(0, np.uint8)
    raise ValueError(kind)


def device_layout():
    """The buffers of the checksum_batch_device sweep: every sweep size below the big buffers and one buffer one
    byte past ZB_CK_BIG_PIECES pieces, buffer i starting at i (mod 16) -> (lengths, misalignments, place()'s
    offsets and indices)"""
    lengths = SMALL_SWEEP + [BIG_PIECES * PIECE + 1]
    mis = [i % 16 for i in range(len(lengths))]
    offs, which = place(lengths, mis)
    return lengths, mis, offs, which


def place(lengths, mis, base_shift=0):
    """Pack buffers of `lengths` so that buffer i starts at an address = base_shift + offset = mis[i] (mod 16), with
    filler buffers of 0..15 bytes between them.  -> (offsets uint64[m + 1], index of buffer i among the m buffers).
    The offsets describe one contiguous layout starting at the (16-byte aligned) base + base_shift."""
    offs, which, pos = [0], [], 0
    for n, want in zip(lengths, mis):
        pad = (want - base_shift - pos) % 16
        if pad:
            pos += pad
            offs.append(pos)
        which.append(len(offs) - 1)
        pos += n
        offs.append(pos)
    return np.array(offs, dtype=np.uint64), which


def full_piece_misalignments(lengths, mis, base_shift=0):
    """The set of (address mod 16) of the full pieces in place()'s layout"""
    offs, which = place(lengths, mis, base_shift)
    seen = set()
    for n, j in zip(lengths, which):
        for k in range(n // PIECE):
            seen.add((base_shift + int(offs[j]) + k * PIECE) % 16)
    return seen


# ---- members for the decode verdicts ----------------------------------------------------------------------------

def member(data, fmt, level):
    """a gzip / zlib member made by Python's zlib"""
    c = zlib.compressobj(level, zlib.DEFLATED, 31 if fmt == "gzip" else 15)
    return c.compress(data) + c.flush()


def bad_block(m, fmt):
    """the member with its first block's BTYPE set to 3 (reserved): it fails to inflate"""
    b = bytearray(m)
    b[10 if fmt == "gzip" else 2] |= 0x06
    return bytes(b)


def corruptions(m, fmt, n, flips=range(4), isize=True, bad=True):
    """-> [(name, member)]: each trailer check byte in `flips` flipped, gzip ISIZE +- 1, a member that fails to
    inflate"""
    out = []
    tail = len(m) - (8 if fmt == "gzip" else 4)
    for j in flips:
        b = bytearray(m)
        b[tail + j] ^= 0xFF
        out.append(("check byte %d" % j, bytes(b)))
    if fmt == "gzip" and isize:
        for d in (1, -1):
            b = bytearray(m)
            b[-4:] = ((n + d) & 0xFFFFFFFF).to_bytes(4, "little")
            out.append(("isize %+d" % d, bytes(b)))
    if bad:
        out.append(("bad block", bad_block(m, fmt)))
    return out


# the host-pipeline batch, every member compressed below BIG_MEMBER_BYTES: short and one-piece sizes, share-multiple
# ragged last pieces (2 KiB multiples of the CRC path), 65 536, 131 072, the Adler modulus, and pieces at lanes >= 32
# of the combine
PIPE_SWEEP = [0, 1, 3, 4, 5, 127, 2047, 2049, 4096, PIECE - 1, PIECE, PIECE + 1, 2048 * 18, 2048 * 23, 2048 * 31,
              ADLER_MOD - 1, ADLER_MOD, ADLER_MOD + 1, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK, 2 * PIECE + 2048,
              15 * PIECE + 6144, 16 * PIECE + 3, 32 * PIECE + 1, 33 * PIECE + 3, 33 * PIECE + 6144]


def pipeline_members(text):
    """-> [(name, member, output or None, output length)]: gzip and zlib members of PIPE_SWEEP, each followed by
    all of its corruptions.  Incompressible content only where it stays below BIG_MEMBER_BYTES; level 6 / 9 text
    and sparse content above."""
    items = []
    for i, n in enumerate(PIPE_SWEEP):
        fill = ("random", "text", "ff", "sparse")[i % 4] if n < BIG_MEMBER_BYTES - 4096 else ("text", "sparse")[i % 2]
        data = content(fill, n, seed=700 + i, text=text).tobytes()
        for fmt in ("gzip", "zlib"):
            m = member(data, fmt, (6, 9)[i % 2])
            items.append(("%s %d good" % (fmt, n), m, data, n))
            items += [("%s %d %s" % (fmt, n, name), b, None, n) for name, b in corruptions(m, fmt, n)]
    return items
