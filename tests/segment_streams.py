"""Members cut at sync joints, for the tests of the parallel joint decode (zb_api.cu: inflate_big_members and
inflate_member_joints; zb_inflate.cu: the parallel window resolve).

A joint is an empty non-final stored block, `00 00 ff ff` on a byte boundary: zlib's Z_SYNC_FLUSH writes one,
and so does this library after every 64 KiB chunk at levels -1 and 2..9.  Two kinds of builders:

- `sync_flushed`: Python's zlib as a foreign encoder, with a sync flush at chosen input offsets.
- `joint_member`: hand-built streams (tests/deflate_writer.py), one token list per segment, with an empty
  stored block after every segment and optional empty fixed blocks as padding (they add compressed bytes and
  no output, which keeps the joints below the decoder's density cap).

`analyse` finds the joints the way the host code does and decodes every segment on its own with zlib, with the
true 32 KiB in front of it as a preset dictionary and again with that window inverted: where the two outputs
first differ is the first output byte that comes from before the segment.  `plan` turns the segment list into
the launch count the host code must report for a single-member `uncompress_batch` call.
"""
import zlib
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from tests import deflate_writer as dw

CHUNK = 65536          # this library's chunk: the 64 KiB-per-segment guess
WIN = 32768            # the DEFLATE window; also the join rule's limit
MARK = b"\x00\x00\xff\xff"
ZLIB, GZIP, RAW = 1, 2, 3
WBITS = {RAW: -15, ZLIB: 15, GZIP: 31}


@dataclass
class Seg:
    n: int                  # output bytes
    back: Optional[int]     # offset of its first output byte that comes from before the segment; None: none does


@dataclass
class Member:
    blob: bytes
    fmt: int
    raw: bytes                      # the bytes the member stands for
    pos: int                        # payload start in blob
    end: int                        # payload end
    joints: List[int]               # blob offsets just behind every 00 00 ff ff in the payload
    bounds: List[int] = field(default_factory=list)   # segment boundaries as the host code sets them
    segs: List[Seg] = field(default_factory=list)     # the segments between true joints
    false: int = 0                  # joints that are not block boundaries (planted in stored data)

    @property
    def dense(self):
        """More than one joint per 32 compressed bytes: the host code does not take the joints (its cap)."""
        return len(self.joints) > (self.end - self.pos) // 32 + 64


def payload(blob, fmt):
    """Start and end of the DEFLATE data inside the wrapper (a gzip header without optional fields)."""
    if fmt == RAW:
        return 0, len(blob)
    if fmt == ZLIB:
        return 2, len(blob) - 4
    assert blob[3] == 0, "gzip header fields are not supported here"
    return 10, len(blob) - 8


def find_joints(blob, pos, end):
    out, p = [], blob.find(MARK, pos, end)
    while p != -1:
        out.append(p + 4)
        p = blob.find(MARK, p + 1, end)
    return out


def refers_back(piece):
    """True when a segment decoded alone (no window) fails because it refers to bytes before it."""
    try:
        d = zlib.decompressobj(-15)
        d.decompress(piece)
        return False
    except zlib.error as e:
        assert "invalid distance too far back" in str(e), e
        return True


def analyse(blob, fmt, raw, false_joints=()):
    """-> Member.  false_joints: blob offsets (behind the pattern) of planted joints inside stored data."""
    pos, end = payload(blob, fmt)
    j = find_joints(blob, pos, end)
    m = Member(blob, fmt, raw, pos, end, j, false=len(false_joints))
    m.bounds = [pos] + j if j and j[-1] >= end else [pos] + j + [end]
    true_b = [b for b in m.bounds if b not in set(false_joints)]
    out = bytearray()
    for i in range(len(true_b) - 1):
        piece = blob[true_b[i]:true_b[i + 1]]
        start = len(out)
        win = bytes(out[max(0, start - WIN):start])
        got = (zlib.decompressobj(-15, zdict=win) if win else zlib.decompressobj(-15)).decompress(piece)
        back = None
        if win:
            alt = (np.frombuffer(win, dtype=np.uint8) ^ 0xff).tobytes()
            g2 = zlib.decompressobj(-15, zdict=alt).decompress(piece)
            if g2 != got:
                a, b = np.frombuffer(got, dtype=np.uint8), np.frombuffer(g2, dtype=np.uint8)
                back = int(np.flatnonzero(a != b)[0])
        m.segs.append(Seg(len(got), back))
        out += got
    assert bytes(out) == raw, "the segments do not decode to the member's bytes"
    return m


# ---------------------------------------------------------------------------------------------- builders
def wrap(stream, raw, fmt):
    return stream if fmt == RAW else dw.zlib_wrap(stream, raw) if fmt == ZLIB else dw.gzip_wrap(stream, raw)


def sync_flushed(data, cuts, fmt=RAW, level=6, mem_level=8):
    """zlib's stream of `data` with a Z_SYNC_FLUSH at every input offset in `cuts` (increasing, inside data)."""
    c = zlib.compressobj(level, zlib.DEFLATED, WBITS[fmt], mem_level)
    out, prev = [], 0
    for x in cuts:
        assert prev < x < len(data)
        out += [c.compress(data[prev:x]), c.flush(zlib.Z_SYNC_FLUSH)]
        prev = x
    out += [c.compress(data[prev:]), c.flush()]
    return b"".join(out)


def every(n, k):
    """Cuts every k bytes of an n-byte input."""
    return list(range(k, n, k))


def random_cuts(n, seed, lo=1, hi=150000):
    rng = np.random.default_rng(seed)
    cuts, x = [], 0
    while True:
        x += int(rng.integers(lo, hi + 1))
        if x >= n:
            return cuts
        cuts.append(x)


def data(corpus_text, kind, n, seed=1):
    """text, runs (byte runs), zeros, or mix (text, runs and random stretches that zlib stores)."""
    rng = np.random.default_rng(seed)
    if kind == "text":
        return (corpus_text * (1 + n // len(corpus_text)))[:n]
    if kind == "runs":
        runs = rng.integers(1, 300, n // 50 + 1)
        return np.repeat(rng.integers(0, 256, len(runs), dtype=np.uint8), runs)[:n].tobytes()
    if kind == "zeros":
        return bytes(n)
    parts, k = [], 0
    while sum(map(len, parts)) < n:
        m = int(rng.integers(5000, 120000))
        sub = ("text", "runs", "random")[k % 3]
        if sub == "random":
            parts.append(rng.integers(0, 256, m, dtype=np.uint8).tobytes())
        else:
            off = int(rng.integers(0, len(corpus_text) - m)) if len(corpus_text) > m else 0
            parts.append(data(corpus_text[off:], sub, m, seed + k))
        k += 1
    return b"".join(parts)[:n]


PAD = 28   # empty fixed blocks (10 bits each): 35 compressed bytes per segment, above the density cap's 32


def joint_blocks(segments, pad=PAD, tail=None):
    """Blocks of a member whose segment i holds the blocks segments[i] (a token list is one fixed block),
    each followed by an empty non-final stored block -- the joint -- except the last (None: no blocks at all).  tail: None (the last
    segment's last block is final), "fixed" (a final empty fixed block after one more joint) or "stored" (a
    final empty stored block after the last segment: the payload ends with 00 00 ff ff)."""
    blocks = []
    for i, seg in enumerate(segments):
        if seg is None:            # nothing: this joint follows the previous one back to back
            seg = []
        else:
            blocks += [dw.Fixed([], final=False) for _ in range(pad)]
            seg = seg if seg and not isinstance(seg[0], (int, tuple)) else [dw.Fixed(list(seg))]
        for b in seg:
            b.final = False
            blocks.append(b)
        if i + 1 < len(segments) or tail == "fixed":
            blocks.append(dw.Stored(b"", final=False))
    if tail == "fixed":
        blocks.append(dw.Fixed([], final=True))
    elif tail == "stored":
        blocks.append(dw.Stored(b"", final=True))
    else:
        blocks[-1].final = True
    return blocks


def joint_member(segments, fmt=RAW, pad=PAD, tail=None, false_joints=()):
    """-> Member of the hand-built stream (see joint_blocks); its bytes come from deflate_writer.replay."""
    blocks = joint_blocks(segments, pad, tail)
    raw = dw.replay(blocks)
    stream = dw.raw(blocks)
    blob = wrap(stream, raw, fmt)
    shift = payload(blob, fmt)[0]
    return analyse(blob, fmt, raw, [shift + f for f in false_joints])


def history(n, seed):
    """Segment 0 of many hand-built members: n random bytes in stored blocks (no joint can hide in them:
    checked by the builders' tests)."""
    rng = np.random.default_rng(seed)
    b = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    return [dw.Stored(b[i:i + 65535], final=False) for i in range(0, n, 65535)]


def edge_tokens(k):
    """One segment's tokens: a copy from exactly 32768 back (the first byte of the incoming window when the
    segment starts a group), a copy that starts at the byte just before the segment (the window's last byte), a
    copy that straddles the segment start, then two literals that make the segment's bytes its own."""
    return [(258, 32768), (3, 259), (258, 258 + 130), 0x41 + k % 26, 0x61 + (k * 7) % 26]


# ---------------------------------------------------------------------------------------------- launches
BASE = 3                 # the ordinary inflate launch and the two kernels of its checksum pass
OPTIMISTIC = 2           # the joint search and the optimistic pass (every segment at 64 KiB)
COUNT = 2                # the joint search and the count pass without windows (when the optimistic pass is skipped)
WINDOW_GUESS = 2         # marker prefill + marker decode of one window
RESOLVE = 4              # k_resolve_groups, k_resolve_compose, k_resolve_tails_par, k_resolve_rest
SPECULATIVE = (1, 2, 4, 6)   # the speculative segments: block search [+ count [+ prefill + decode [+ resolve]]]


@dataclass
class Plan:
    path: str                       # "joint", "independent", "too_small" or "fallback"
    launches: Optional[int] = None  # None: the speculative segments or the serial decode take the member
    counts: int = 0                 # count_all rounds
    guess_failed: Optional[int] = None   # index of the window at which the 64 KiB guess failed
    windows: List[int] = field(default_factory=list)   # segments per resolved window


def join(sizes):
    """count_all's join rule: every segment that starts before output byte 32768 joins segment 0."""
    out, p = [sizes[0]], sizes[0]
    for n in sizes[1:]:
        if p >= WIN:
            out.append(n)
        else:
            out[0] += n
        p += n
    return out


def split_windows(sizes, w, counted):
    """[a, b) of every window: at most w segments and at most w * (32768 + 65536) scratch elements, where a
    segment costs 32768 + its size (65536 under the guess); a segment larger than that is a window alone."""
    out, a = [], 0
    while a < len(sizes):
        b, el = a, 0
        while b < len(sizes) and b - a < w:
            e = WIN + (sizes[b] if counted else CHUNK)
            if b > a and el + e > w * (WIN + CHUNK):
                break
            el += e
            b += 1
        out.append((a, b))
        a = b
    return out


def plan(m, mcap=None, window=8192, joints=True):
    """The path and kernel-launch count of a valid member `m` alone in uncompress_batch, mirroring
    inflate_big_members / inflate_member_joints.  mcap: the output slot (default: the exact size)."""
    sizes = [s.n for s in m.segs]
    total = sum(sizes)
    mcap = total if mcap is None else mcap
    S = len(m.bounds) - 1           # segments as the joint search sees them (false joints included)
    if m.end <= m.pos + 4 or not m.joints or m.dense or S < 2:
        return Plan("fallback")
    L = BASE
    guess = back_refs = False
    if (S - 1) * CHUNK < mcap:
        assert not m.false, "false joints are modelled only where the optimistic pass is skipped"
        L += OPTIMISTIC
        st = []
        for j, s in enumerate(m.segs):
            cap = CHUNK if j + 1 < S else mcap - (S - 1) * CHUNK
            # the first offending token decides: a reference before the segment (3) or one past the slot (19)
            st.append(3 if s.back is not None and s.back <= cap else 19 if s.n > cap else 0)
        if all(x == 0 for x in st) and all(n == CHUNK for n in sizes[:-1]):
            return Plan("independent", L)
        guess = not any((st[j] == 0 and sizes[j] != CHUNK) or st[j] == 19 for j in range(S - 1))
        back_refs = any(x == 3 for x in st[1:])
    if not (back_refs and joints):
        L += COUNT
        if m.false or any(s.back is not None for s in m.segs):
            if not joints:
                return Plan("fallback")
            guess = False
        else:
            return Plan("independent", L + 1) if total <= mcap else Plan("fallback")
    p = Plan("joint")
    counted = False

    def count_all():
        nonlocal sizes, L
        if m.false:                 # round 0 fails on both sides of every false joint: they are dropped
            L += 1
            p.counts += 1
        for rnd in range(3 - (1 if m.false else 0)):
            L += 1
            p.counts += 1
            new = join(sizes)
            if len(new) == len(sizes):
                return True
            sizes = new
        return False

    if not guess:
        if not count_all():
            return Plan("fallback")
        counted = True
        if total > mcap:
            return Plan("too_small")
    a = 0
    while a < len(sizes):
        a_, b = split_windows(sizes[a:], window, counted)[0]
        b += a
        L += WINDOW_GUESS
        if not counted and not all(sizes[i] == CHUNK if i + 1 < len(sizes) else sizes[i] <= CHUNK for i in range(a, b)):
            p.guess_failed = len(p.windows)
            if not count_all():
                return Plan("fallback")
            counted = True
            continue
        L += RESOLVE
        p.windows.append(b - a)
        a = b
    p.launches = L
    return p


def group_shape(nw):
    """Groups of one window: ceil(sqrt(nw)) segments each, the last one partial."""
    g = int(np.ceil(np.sqrt(nw)))
    return g, (nw + g - 1) // g


# ---------------------------------------------------------------------------------------------- the cases
INTERVALS = [100, 1000, 32767, 32768, 32769, 65535, 65536, 65537, 200000]
FMTS = (RAW, ZLIB, GZIP)
LEVELS = (1, 6, 9)
KINDS = ("text", "runs", "zeros", "mix")


def foreign_case(T, i, f):
    """-> (name, Member, intended cuts): zlib's stream sync-flushed every INTERVALS[i] bytes in format FMTS[f];
    levels and data kinds rotate through the intervals and formats."""
    k, fmt = INTERVALS[i], FMTS[f]
    level, kind = LEVELS[(i + f) % 3], KINDS[(i + 2 * f) % 4]
    if k <= 1000 and kind in ("runs", "zeros"):
        kind = "text"          # their joints would be denser than the cap: see dense_cases
    n = 3 * k + 12345 if k >= 32767 else 400000
    n = max(n, 600000) if k >= 65535 else n
    d = data(T, kind, n, seed=i * 3 + f)
    cuts = every(n, k)
    name = "every%d_%s_l%d_%s" % (k, kind, level, ("raw", "zlib", "gzip")[f])
    return name, analyse(sync_flushed(d, cuts, fmt, level), fmt, d), cuts


def random_case(T, seed):
    """Seeded intervals of 1..150 000 bytes over 1.5 MB."""
    d = data(T, ("text", "mix", "runs")[seed], 1_500_000, seed=40 + seed)
    cuts = random_cuts(len(d), seed)
    fmt = FMTS[seed]
    return "random_cuts_%d" % seed, analyse(sync_flushed(d, cuts, fmt, LEVELS[seed]), fmt, d), cuts


def foreign_cases(T):
    return [foreign_case(T, i, f) for i in range(len(INTERVALS)) for f in range(3)] + [random_case(T, s) for s in range(3)]


def many_segments_case(T):
    """100-byte flushes over 2 MB of text: about 20 000 segments, more than one 8192-segment window."""
    d = data(T, "text", 2_000_000, seed=7)
    cuts = every(len(d), 100)
    return analyse(sync_flushed(d, cuts, GZIP, 6), GZIP, d), cuts


def dense_cases(T):
    """Joints denser than one per 32 compressed bytes: the host code must not take them."""
    out = []
    for seed, (kind, lo, hi) in enumerate((("zeros", 1000, 1000), ("text", 1, 12), ("runs", 1, 200))):
        d = data(T, kind, 300000, seed=60 + seed)
        cuts = random_cuts(len(d), seed + 60, lo, hi)
        out.append(("dense_%s" % kind, analyse(sync_flushed(d, cuts, RAW, 6), RAW, d), cuts))
    return out


def seg_len(seg):
    """Output bytes of one hand-built segment (a token list, a block list or None)."""
    if seg is None:
        return 0
    if seg and not isinstance(seg[0], (int, tuple)):
        return sum(len(b.data) if isinstance(b, dw.Stored) else seg_len(b.tokens) for b in seg)
    return sum(1 if isinstance(t, int) else t[0] for t in seg)


def chain_segments(n, dist, seed):
    """Segment 0: 40 000 random bytes (dist 32768) or a single literal; then n segments of one (258, dist)
    match each, or of a seeded distance in 1..32768 (dist None)."""
    rng = np.random.default_rng(seed)
    segs = [history(40000, seed)] if dist != 1 else [[0x5a]]
    for _ in range(n):
        segs.append([(258, dist if dist else int(rng.integers(1, WIN + 1)))])
    return segs


def edge_segments(n, seed, big=()):
    """Segment 0: 40 000 random bytes; then n segments of edge_tokens; segment indices in `big` instead hold
    about 200 000 bytes of seeded copies (larger than the window's element budget at 2 segments)."""
    rng = np.random.default_rng(seed)
    segs = [history(40000, seed)]
    for k in range(1, n + 1):
        if k in big:
            segs.append([(258, int(rng.integers(1, WIN + 1))) for _ in range(776)] + [0x30 + k % 10])
        else:
            segs.append(edge_tokens(k))
    return segs


def start_rule_segments(start, dist, tiny):
    """Output bytes 0..start-1 (one stored segment, or `tiny` segments of a few bytes after a 2000-byte one),
    a joint, then a segment that opens with a match of distance `dist` (start: reaches byte 0; start + 1:
    byte -1), then three more segments."""
    rng = np.random.default_rng(start + dist + tiny)
    if not tiny:
        segs = [history(start, 3)]
    else:
        segs, left = [history(2000, 3)], start - 2000
        for k in range(tiny):
            m = left // (tiny - k)
            segs.append([dw.Stored(rng.integers(0, 256, m, dtype=np.uint8).tobytes(), final=False)])
            left -= m
    segs.append([(min(258, dist), dist), 0x41, 0x42])
    segs += [edge_tokens(k) for k in range(3)]
    return segs


def late_failure_member(T, odd, fmt=GZIP):
    """zlib, sync-flushed every 65536 input bytes except one segment of `odd` bytes, the first of the third
    window at 3 segments per window."""
    cuts, x = [], 0
    for k in range(14):
        x += odd if k == 6 else CHUNK
        cuts.append(x)
    d = data(T, "text", x + 30000, seed=odd)
    return analyse(sync_flushed(d, cuts, fmt, 6), fmt, d), cuts
