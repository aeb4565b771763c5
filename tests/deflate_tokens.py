"""A DEFLATE token reader for tests (RFC 1951).

`parse(raw)` walks a raw DEFLATE stream and returns its blocks with the tokens they hold, instead of the
bytes they stand for: a compressor's parse can then be compared decision by decision.  A token is a
literal byte (int 0..255) or a match (length, distance) -- the same form `deflate_writer` takes.  A stored
block's bytes are listed as literals.

Anything malformed raises `Malformed`: reserved block types, stored LEN/NLEN that disagree, HLIT > 286 or
HDIST > 30, over-subscribed codes, repeat codes with nothing to repeat or that run past HLIT + HDIST, a bit
pattern no code of the block matches, symbols 286/287, distance codes 30/31, a distance reaching before the
start of the stream, and a stream that ends before its final block does.  Incomplete codes are accepted, as
RFC 1951 does not forbid them; a pattern outside such a code is still an error.
"""
from dataclasses import dataclass, field

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
            227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
MAX_BITS = 15


class Malformed(ValueError):
    """The stream is not valid DEFLATE."""


@dataclass
class Block:
    btype: int                 # 0 stored, 1 fixed, 2 dynamic
    final: bool
    bit_start: int             # offset of the block's first header bit in the stream
    bit_end: int               # offset just past its end-of-block code (stored: past its last byte)
    tokens: list = field(default_factory=list)

    def size(self):
        """Bytes the block stands for."""
        return sum(1 if isinstance(t, int) else t[0] for t in self.tokens)


def _table(lengths):
    """Code lengths -> lookup table indexed by the next MAX_BITS stream bits: entry = symbol << 4 | length,
    0 where no code matches."""
    count = [0] * (MAX_BITS + 1)
    for n in lengths:
        count[n] += 1
    count[0] = 0
    left = 1
    for n in range(1, MAX_BITS + 1):
        left = 2 * left - count[n]
        if left < 0:
            raise Malformed("over-subscribed code")
    code, nxt = 0, [0] * (MAX_BITS + 2)
    for n in range(1, MAX_BITS + 1):
        code = (code + count[n - 1]) << 1
        nxt[n] = code
    tab = [0] * (1 << MAX_BITS)
    for sym, n in enumerate(lengths):
        if not n:
            continue
        c = nxt[n]
        nxt[n] += 1
        rev = int(format(c, "0%db" % n)[::-1], 2)   # codes are sent MSB first
        for k in range(rev, 1 << MAX_BITS, 1 << n):
            tab[k] = sym << 4 | n
    return tab


_FIXED = None


def _fixed_tables():
    global _FIXED
    if _FIXED is None:
        _FIXED = (_table([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8), _table([5] * 32))
    return _FIXED


class _Bits:
    def __init__(self, raw):
        self.raw = bytes(raw)
        self.n = len(self.raw)
        self.data = self.raw + bytes(8)
        self.ip = 0          # next byte to load
        self.buf = 0
        self.cnt = 0         # bits in buf

    def pos(self):
        return 8 * self.ip - self.cnt

    def fill(self, need):
        while self.cnt < need:
            if self.ip >= self.n + 8:
                raise Malformed("the stream ends early")
            self.buf |= self.data[self.ip] << self.cnt
            self.ip += 1
            self.cnt += 8

    def get(self, n):
        self.fill(n)
        v = self.buf & ((1 << n) - 1)
        self.buf >>= n
        self.cnt -= n
        return v

    def sym(self, tab):
        self.fill(MAX_BITS)
        e = tab[self.buf & 0x7fff]
        if not e:
            raise Malformed("no code matches")
        self.buf >>= e & 15
        self.cnt -= e & 15
        return e >> 4

    def check(self):
        if self.pos() > 8 * self.n:
            raise Malformed("the stream ends early")


def _dynamic_tables(br):
    hlit = br.get(5) + 257
    hdist = br.get(5) + 1
    hclen = br.get(4) + 4
    if hlit > 286 or hdist > 30:
        raise Malformed("HLIT %d / HDIST %d" % (hlit, hdist))
    cl = [0] * 19
    for i in range(hclen):
        cl[CL_ORDER[i]] = br.get(3)
    cltab = _table(cl)
    lens = []
    while len(lens) < hlit + hdist:
        s = br.sym(cltab)
        if s < 16:
            lens.append(s)
            continue
        if s == 16:
            if not lens:
                raise Malformed("repeat with nothing to repeat")
            v, r = lens[-1], 3 + br.get(2)
        elif s == 17:
            v, r = 0, 3 + br.get(3)
        else:
            v, r = 0, 11 + br.get(7)
        if len(lens) + r > hlit + hdist:
            raise Malformed("repeat past HLIT + HDIST")
        lens += [v] * r
    if lens[256] == 0:
        raise Malformed("no end-of-block code")
    return _table(lens[:hlit]), _table(lens[hlit:])


def _tokens(br, lt, dt, produced, out):
    """Decode one block's symbols up to its end-of-block code; -> bytes produced so far."""
    data = br.data
    while True:
        # refill once per token: a match is at most 15 + 5 + 15 + 13 bits
        while br.cnt < 48:
            if br.ip >= br.n + 8:
                raise Malformed("the stream ends early")
            br.buf |= data[br.ip] << br.cnt
            br.ip += 1
            br.cnt += 8
        buf = br.buf
        e = lt[buf & 0x7fff]
        if not e:
            raise Malformed("no code matches")
        n = e & 15
        s = e >> 4
        buf >>= n
        used = n
        if s < 256:
            out.append(s)
            produced += 1
        elif s == 256:
            br.buf = buf
            br.cnt -= used
            return produced
        else:
            if s > 285:
                raise Malformed("length symbol %d" % s)
            x = LEN_EXTRA[s - 257]
            length = LEN_BASE[s - 257] + (buf & ((1 << x) - 1))
            buf >>= x
            used += x
            e = dt[buf & 0x7fff]
            if not e:
                raise Malformed("no distance code matches")
            n = e & 15
            s = e >> 4
            buf >>= n
            used += n
            if s > 29:
                raise Malformed("distance symbol %d" % s)
            x = DIST_EXTRA[s]
            dist = DIST_BASE[s] + (buf & ((1 << x) - 1))
            buf >>= x
            used += x
            if dist > produced:
                raise Malformed("distance %d with %d bytes produced" % (dist, produced))
            out.append((length, dist))
            produced += length
        br.buf = buf
        br.cnt -= used


def parse(raw):
    """-> [Block] of the raw DEFLATE stream `raw`, up to and including its final block."""
    br = _Bits(raw)
    blocks, produced = [], 0
    while True:
        start = br.pos()
        final = bool(br.get(1))
        btype = br.get(2)
        if btype == 0:
            br.get(br.cnt & 7)                  # to the byte boundary; whole bytes stay buffered
            br.ip -= br.cnt >> 3                # give them back and read the rest byte-wise
            br.buf = br.cnt = 0
            lo = br.ip + 4
            if lo > br.n:
                raise Malformed("stored header past the end")
            ln = br.raw[lo - 4] | br.raw[lo - 3] << 8
            nl = br.raw[lo - 2] | br.raw[lo - 1] << 8
            if ln != (~nl & 0xffff):
                raise Malformed("stored LEN / NLEN")
            if lo + ln > br.n:
                raise Malformed("stored block past the end")
            toks = list(br.raw[lo:lo + ln])
            br.ip = lo + ln
            produced += ln
        elif btype == 3:
            raise Malformed("block type 3")
        else:
            lt, dt = _fixed_tables() if btype == 1 else _dynamic_tables(br)
            toks = []
            produced = _tokens(br, lt, dt, produced, toks)
        br.check()
        blocks.append(Block(btype, final, start, br.pos(), toks))
        if final:
            return blocks


def rebuild(blocks):
    """The bytes a block list stands for."""
    out = bytearray()
    for b in blocks:
        for t in b.tokens:
            if isinstance(t, int):
                out.append(t)
                continue
            length, dist = t
            if dist > len(out):
                raise Malformed("distance %d with %d bytes produced" % (dist, len(out)))
            src = out[len(out) - dist:len(out) - dist + length]
            if dist < length:   # the copy overlaps its own output: the source repeats with period dist
                src = (src * (length // dist + 1))[:length]
            out += src
    return bytes(out)


@dataclass
class Chunk:
    btype: int
    tokens: list


def member_chunks(blocks, chunk_bytes=65536):
    """Split the blocks of a member this library wrote into its chunks, checking the layout: a chunk is one
    fixed or dynamic block -- followed, unless it is the member's last, by the empty non-final stored block
    that byte-aligns the joint (00 00 ff ff) -- or stored blocks of 65535 bytes at most that together hold the
    chunk's bytes.  Every chunk but the last stands for exactly `chunk_bytes` bytes."""
    chunks, i, pending = [], 0, None
    if not blocks or not blocks[-1].final or any(b.final for b in blocks[:-1]):
        raise Malformed("one final block, at the end")
    while i < len(blocks):
        b = blocks[i]
        if b.btype == 0:
            pending = (pending or []) + b.tokens
            if len(pending) > chunk_bytes:
                raise Malformed("stored chunk longer than a chunk")
            if len(pending) == chunk_bytes or b.final:
                chunks.append(Chunk(0, pending))
                pending = None
            i += 1
            continue
        if pending is not None:
            raise Malformed("stored chunk cut short")
        if b.size() != chunk_bytes and not b.final:
            raise Malformed("chunk of %d bytes" % b.size())
        chunks.append(Chunk(b.btype, b.tokens))
        if b.final:
            i += 1
            continue
        if i + 1 >= len(blocks):
            raise Malformed("no joint after a chunk")
        j = blocks[i + 1]
        if j.btype != 0 or j.tokens or j.final:
            raise Malformed("a chunk is not followed by an empty stored block")
        i += 2
    if pending is not None:
        raise Malformed("stored chunk cut short")
    return chunks
