"""An independent DEFLATE writer for tests (RFC 1951, with RFC 1950 / 1952 wrappers).

Written from the RFCs alone: it does not use zlib, the oracle or any decoder.  Unlike an
encoder it writes exactly what it is told -- code lengths, header counts, code-length RLE
operations and raw symbols are all explicit -- so it can produce streams that no encoder
would: over-subscribed, incomplete, single-code and empty code sets, repeat codes that run
past HLIT + HDIST, symbols 286/287 and distances 30/31, wrong stored LEN/NLEN, wrong trailers.

Tokens of a compressed block:
    int 0..255            a literal
    (length, distance)    a match (3..258, 1..32768), coded with the RFC 1951 3.2.5 tables
    Sym(ll, lx, d, dx)    raw symbols: literal/length symbol `ll` (any 0..287), its extra bits
                          `lx` when 257 <= ll <= 284, then, if `d` is given, distance symbol `d`
                          (any 0..31) and its extra bits `dx` when d <= 29
    Bits(value, n)        n raw bits (a bit pattern no code of the block matches); also allowed
                          among the code-length RLE operations of a dynamic header

`replay(blocks)` computes the expected output from the block list alone, so a decoder under
test is compared with the stream's definition rather than with another decoder.
"""
import random
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
            227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0] + [i // 2 - 1 for i in range(2, 30)]
CLC_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LL = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_D = [5] * 32


class InvalidToken(ValueError):
    """replay() met a token that has no meaning (an invalid symbol or a distance too far back)."""


# ---------------------------------------------------------------------- bits
class BitWriter:
    """Values LSB first; Huffman codes MSB first (RFC 1951 3.1.1)."""

    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.nacc = 0
        self.nbits = 0

    def put(self, value, n):
        assert 0 <= value < (1 << n) or n == 0, (value, n)
        self.acc |= value << self.nacc
        self.nacc += n
        self.nbits += n
        while self.nacc >= 8:
            self.out.append(self.acc & 0xff)
            self.acc >>= 8
            self.nacc -= 8

    def put_code(self, code, length):
        self.put(int(format(code, "0%db" % length)[::-1], 2) if length else 0, length)

    def align(self):
        if self.nacc:
            self.put(0, 8 - self.nacc)

    def getvalue(self):
        return bytes(self.out) + (bytes([self.acc]) if self.nacc else b"")


def canonical_codes(lengths):
    """RFC 1951 3.2.2 from an explicit length list.  Over-subscribed sets get codes too (they
    overflow their length and are only useful to write a header a decoder must reject)."""
    bl_count = [0] * 16
    for ln in lengths:
        if ln:
            bl_count[ln] += 1
    code, next_code = 0, [0] * 16
    for bits in range(1, 16):
        code = (code + bl_count[bits - 1]) << 1
        next_code[bits] = code
    codes = [None] * len(lengths)
    for s, ln in enumerate(lengths):
        if ln:
            codes[s] = next_code[ln] & ((1 << ln) - 1)
            next_code[ln] += 1
    return codes


def kraft(lengths):
    """Sum of 2^-len as a fraction of 2^15: 32768 = complete, less = incomplete, more = over-subscribed."""
    return sum(1 << (15 - ln) for ln in lengths if ln)


def huffman_lengths(freqs, limit):
    """Code lengths <= limit for the nonzero frequencies (Huffman, then lengths over the limit are
    clamped and the Kraft sum repaired by lengthening the rarest short codes).  Never over-subscribed."""
    import heapq
    syms = [s for s, f in enumerate(freqs) if f > 0]
    lens = [0] * len(freqs)
    if len(syms) == 1:
        lens[syms[0]] = 1
        return lens
    heap = [(freqs[s], s, (s,)) for s in syms]
    heapq.heapify(heap)
    tie = len(freqs)
    while len(heap) > 1:
        fa, _, a = heapq.heappop(heap)
        fb, _, b = heapq.heappop(heap)
        for s in a + b:
            lens[s] += 1
        heapq.heappush(heap, (fa + fb, tie, a + b))
        tie += 1
    for s in syms:
        lens[s] = min(lens[s], limit)
    order = sorted(syms, key=lambda s: (freqs[s], -s))   # rarest first
    while sum(1 << (limit - lens[s]) for s in syms) > (1 << limit):
        s = max((s for s in order if lens[s] < limit), key=lambda s: (lens[s], -freqs[s]))
        lens[s] += 1
    while True:   # the repair can leave room: shorten codes until the set is complete again
        room = (1 << limit) - sum(1 << (limit - lens[s]) for s in syms)
        fits = [s for s in syms if lens[s] > 1 and (1 << (limit - lens[s])) <= room]
        if not room or not fits:
            return lens
        lens[max(fits, key=lambda s: (lens[s], freqs[s]))] -= 1


def chain_lengths(order, n):
    """A complete code over the symbols in `order`: lengths 1, 2, 3, ..., with the last two equal
    (with 16 symbols: 1..15 and 15).  The deepest possible code for the symbols at the end."""
    lens = [0] * n
    k = len(order)
    for i, s in enumerate(order):
        lens[s] = min(i + 1, k - 1) if k > 1 else 1
    return lens


# ---------------------------------------------------------------------- tokens and blocks
@dataclass
class Sym:
    ll: int
    lx: int = 0
    d: Optional[int] = None
    dx: int = 0


@dataclass
class Bits:
    value: int
    n: int


def length_symbol(length):
    assert 3 <= length <= 258
    if length == 258:
        return 285, 0
    i = max(k for k in range(28) if LEN_BASE[k] <= length)
    return 257 + i, length - LEN_BASE[i]


def distance_symbol(dist):
    assert 1 <= dist <= 32768
    i = max(k for k in range(30) if DIST_BASE[k] <= dist)
    return i, dist - DIST_BASE[i]


def token_symbols(tok):
    """-> Sym for any token (a match becomes its length and distance symbols)."""
    if isinstance(tok, Sym):
        return tok
    if isinstance(tok, int):
        return Sym(tok)
    ls, lx = length_symbol(tok[0])
    ds, dx = distance_symbol(tok[1])
    return Sym(ls, lx, ds, dx)


@dataclass
class Stored:
    data: bytes = b""
    final: Optional[bool] = None
    len_: Optional[int] = None    # LEN / NLEN as written (default: len(data) and its complement)
    nlen: Optional[int] = None


@dataclass
class Fixed:
    tokens: list = field(default_factory=list)
    final: Optional[bool] = None
    eob: bool = True


@dataclass
class Dynamic:
    tokens: list = field(default_factory=list)
    ll_lens: Optional[List[int]] = None   # default: Huffman lengths of the tokens (limit 15)
    d_lens: Optional[List[int]] = None
    final: Optional[bool] = None
    eob: bool = True
    hlit: Optional[int] = None            # as written (257..288); default len(ll_lens)
    hdist: Optional[int] = None           # 1..32; default len(d_lens)
    hclen: Optional[int] = None           # 4..19; default: trailing zero lengths trimmed
    cl_lens: Optional[List[int]] = None   # 19 code-length code lengths by symbol; default from the RLE
    rle: Optional[list] = None            # [(symbol 0..18, extra value)]; default rle_encode(ll_lens + d_lens)


def rle_encode(lengths):
    """Code lengths -> [(symbol, extra)] with 16 / 17 / 18 runs (RFC 1951 3.2.7)."""
    ops, i, n = [], 0, len(lengths)
    while i < n:
        v = lengths[i]
        run = 1
        while i + run < n and lengths[i + run] == v:
            run += 1
        if v == 0 and run >= 3:
            r = min(run, 138)
            ops.append((18, r - 11) if r >= 11 else (17, r - 3))
            i += r
            continue
        ops.append((v, 0))
        i += 1
        run -= 1
        while run >= 3:
            r = min(run, 6)
            ops.append((16, r - 3))
            i += r
            run -= r
    return ops


RLE_EXTRA = {16: 2, 17: 3, 18: 7}


def _frequencies(tokens, eob):
    ll, d = [0] * 286, [0] * 30
    for t in tokens:
        if isinstance(t, Bits):
            continue
        s = token_symbols(t)
        if s.ll < 286:
            ll[s.ll] += 1
        if s.d is not None and s.d < 30:
            d[s.d] += 1
    if eob:
        ll[256] += 1
    return ll, d


def _trim(lens, minimum):
    n = len(lens)
    while n > minimum and lens[n - 1] == 0:
        n -= 1
    return list(lens[:n])


def _write_tokens(bw, tokens, ll_codes, ll_lens, d_codes, d_lens, eob):
    for t in tokens:
        if isinstance(t, Bits):
            bw.put(t.value, t.n)
            continue
        s = token_symbols(t)
        bw.put_code(ll_codes[s.ll], ll_lens[s.ll])
        if 257 <= s.ll <= 284:
            bw.put(s.lx, LEN_EXTRA[s.ll - 257])
        if s.d is not None:
            bw.put_code(d_codes[s.d], d_lens[s.d])
            if s.d <= 29:
                bw.put(s.dx, DIST_EXTRA[s.d])
    if eob:
        bw.put_code(ll_codes[256], ll_lens[256])


def dynamic_header(blk):
    """-> (ll_lens, d_lens) the block's symbols are coded with (after defaults are filled in)."""
    ll_lens, d_lens = blk.ll_lens, blk.d_lens
    if ll_lens is None or d_lens is None:
        fl, fd = _frequencies(blk.tokens, blk.eob)
        if ll_lens is None:
            ll_lens = _trim(huffman_lengths(fl, 15), 257)
        if d_lens is None:
            d_lens = _trim(huffman_lengths(fd, 15), 1) if any(fd) else [0]
    return ll_lens, d_lens


def write_block(bw, blk, final):
    if isinstance(blk, Stored):
        bw.put(int(final), 1)
        bw.put(0, 2)
        bw.align()
        ln = len(blk.data) if blk.len_ is None else blk.len_
        nl = (~ln & 0xffff) if blk.nlen is None else blk.nlen
        bw.put(ln, 16)
        bw.put(nl, 16)
        bw.out += blk.data   # byte-aligned here
        bw.nbits += 8 * len(blk.data)
        return
    if isinstance(blk, Fixed):
        bw.put(int(final), 1)
        bw.put(1, 2)
        _write_tokens(bw, blk.tokens, canonical_codes(FIXED_LL), FIXED_LL, canonical_codes(FIXED_D), FIXED_D, blk.eob)
        return
    ll_lens, d_lens = dynamic_header(blk)
    rle = blk.rle if blk.rle is not None else rle_encode(list(ll_lens) + list(d_lens))
    cl_lens = blk.cl_lens
    if cl_lens is None:
        f = [0] * 19
        for op in rle:
            if not isinstance(op, Bits):
                f[op[0]] += 1
        if sum(1 for x in f if x) < 2:   # a single code would be incomplete: give it a partner
            f[18 if f[18] == 0 else 0] += 1
        cl_lens = huffman_lengths(f, 7)
    hclen = blk.hclen
    if hclen is None:
        hclen = 19
        while hclen > 4 and cl_lens[CLC_ORDER[hclen - 1]] == 0:
            hclen -= 1
    hlit = len(ll_lens) if blk.hlit is None else blk.hlit
    hdist = len(d_lens) if blk.hdist is None else blk.hdist
    bw.put(int(final), 1)
    bw.put(2, 2)
    bw.put(hlit - 257, 5)
    bw.put(hdist - 1, 5)
    bw.put(hclen - 4, 4)
    for i in range(hclen):
        bw.put(cl_lens[CLC_ORDER[i]], 3)
    cl_codes = canonical_codes(cl_lens)
    for op in rle:
        if isinstance(op, Bits):
            bw.put(op.value, op.n)
            continue
        s, x = op
        bw.put_code(cl_codes[s], cl_lens[s])
        if s in RLE_EXTRA:
            bw.put(x, RLE_EXTRA[s])
    ll_full = list(ll_lens) + [0] * (288 - len(ll_lens))
    d_full = list(d_lens) + [0] * (32 - len(d_lens))
    _write_tokens(bw, blk.tokens, canonical_codes(ll_full), ll_full, canonical_codes(d_full), d_full, blk.eob)


def raw(blocks, prefix=b""):
    """The raw DEFLATE stream of `blocks` (BFINAL on the last one unless a block says otherwise),
    after `prefix` bytes (for inflate(pos=k))."""
    bw = BitWriter()
    for b in prefix:
        bw.put(b, 8)
    for i, blk in enumerate(blocks):
        final = blk.final if blk.final is not None else i == len(blocks) - 1
        write_block(bw, blk, final)
    return bw.getvalue()


def block_bits(blocks):
    """Bit offset at which every block starts, and the stream's end bit."""
    bw, pos = BitWriter(), []
    for i, blk in enumerate(blocks):
        pos.append(bw.nbits)
        write_block(bw, blk, blk.final if blk.final is not None else i == len(blocks) - 1)
    return pos, bw.nbits


def replay(blocks):
    """The bytes `blocks` stand for, from the token definitions alone.  Raises InvalidToken."""
    out = bytearray()
    for blk in blocks:
        if isinstance(blk, Stored):
            out += blk.data
            continue
        for t in blk.tokens:
            if isinstance(t, Bits):
                raise InvalidToken("raw bits")
            s = token_symbols(t)
            if s.ll < 256:
                out.append(s.ll)
                continue
            if s.ll == 256 or s.ll > 285 or s.d is None or s.d > 29:
                raise InvalidToken("symbol %d / distance symbol %s" % (s.ll, s.d))
            length = LEN_BASE[s.ll - 257] + s.lx
            dist = DIST_BASE[s.d] + s.dx
            if dist > len(out):
                raise InvalidToken("distance %d with %d bytes produced" % (dist, len(out)))
            _copy(out, length, dist)
    return bytes(out)


def _copy(out, length, dist):
    """Append a match: byte k of it equals the byte `dist` before it (RFC 1951 3.2.3)."""
    if dist >= length:
        out += out[len(out) - dist:len(out) - dist + length]
    else:
        chunk = bytes(out[len(out) - dist:])
        out += (chunk * (length // dist + 1))[:length]


# ---------------------------------------------------------------------- wrappers
_CRC_TABLE = []
for _n in range(256):
    _c = _n
    for _ in range(8):
        _c = (_c >> 1) ^ 0xEDB88320 if _c & 1 else _c >> 1
    _CRC_TABLE.append(_c)


def crc32(data):
    c = 0xffffffff
    t = _CRC_TABLE
    for b in data:
        c = t[(c ^ b) & 0xff] ^ (c >> 8)
    return c ^ 0xffffffff


def adler32(data):
    a = np.frombuffer(bytes(data), dtype=np.uint8).astype(np.int64)
    n, s1, s2 = len(a), 1, 0
    for i in range(0, n, 1 << 20):   # weights stay far below 2^63 per piece
        p = a[i:i + (1 << 20)]
        m = len(p)
        s2 = (s2 + m * s1 + int(np.dot(np.arange(m, 0, -1, dtype=np.int64), p))) % 65521
        s1 = (s1 + int(p.sum())) % 65521
    return (s2 << 16) | s1


def zlib_wrap(stream, data, adler=None, header=b"\x78\x9c"):
    a = adler32(data) if adler is None else adler
    return header + stream + a.to_bytes(4, "big")


def gzip_wrap(stream, data, crc=None, isize=None, fname=b""):
    flg = 8 if fname else 0
    head = bytes([31, 139, 8, flg, 0, 0, 0, 0, 0, 255]) + (fname + b"\0" if fname else b"")
    c = crc32(data) if crc is None else crc
    n = len(data) & 0xffffffff if isize is None else isize
    return head + stream + c.to_bytes(4, "little") + n.to_bytes(4, "little")


# ---------------------------------------------------------------------- seeded valid streams
def phase_block(phase):
    """A fixed block of literals after which the next block starts at bit `phase` mod 32
    (when this block starts at a multiple of 32): 3 header bits + a 9-bit and b 8-bit literals + 7."""
    a = (phase - 10) % 8
    b = ((phase - 10 - 9 * a) % 32) // 8
    return Fixed([0x90 + i for i in range(a)] + [0x41 + i for i in range(b)], final=False)


def random_stream(seed, skew="flat", dist="short", kinds=("dynamic", "fixed", "stored"), nblocks=4, block_tokens=(1, 400),
                  phase=None, history=0):
    """A valid multi-block stream -> list of blocks (replay() gives its bytes).
    skew:    "flat" (Huffman lengths of the tokens) or "deep" (lengths forced up to 15 bits on both trees)
    dist:    "one" (distance 1), "short" (1..64), "far" (up to 32768, many at exactly 32768), or "dependent"
             (a far match, then matches that read bytes the previous match just wrote)
    kinds:   block types to draw from; block_tokens: token count range per compressed block
    phase:   0..31: a leading fixed block that puts the next block at this bit phase
    history: bytes of stored data first (far distances need 32768)"""
    rng = random.Random(seed)
    blocks, out = [], bytearray()
    if phase is not None:
        blocks.append(phase_block(phase))
        out += replay(blocks)
    while history > 0:
        n = min(history, 65535)
        data = rng.randbytes(n)
        blocks.append(Stored(data, final=False))
        out += data
        history -= n
    alphabet = bytes(rng.sample(range(256), rng.choice((4, 16, 60, 256))))
    for _ in range(nblocks):
        kind = rng.choice(kinds)
        if kind == "stored":
            data = rng.randbytes(rng.choice((0, 1, 7, 300, 4000)))
            blocks.append(Stored(data, final=False))
            out += data
            continue
        tokens = []
        for _ in range(rng.randint(*block_tokens)):
            if len(out) < 3 or rng.random() < 0.35:
                b = alphabet[rng.randrange(len(alphabet))]
                tokens.append(b)
                out.append(b)
                continue
            length = rng.choice((3, 4, 5, 10, 11, 18, 31, 34, 66, 130, 131, 227, 257, 258, rng.randint(3, 258)))
            if dist == "one":
                d = 1
            elif dist == "short":
                d = rng.randint(1, 64)
            elif dist == "far":
                d = rng.choice((32768, 32768, 32767, 24577, 16385, rng.randint(1, 32768)))
            else:   # dependent: far, then short ones that overlap what was just written
                d = rng.choice((32768, rng.randint(1, 3), rng.randint(1, length)))
            d = min(d, len(out), 32768)
            tokens.append((length, d))
            _copy(out, length, d)
        if kind == "fixed":
            blocks.append(Fixed(tokens, final=False))
        else:
            blk = Dynamic(tokens, final=False)
            if skew == "deep":
                fl, fd = _frequencies(tokens, True)
                order = list(range(286))
                rng.shuffle(order)
                for r, s in enumerate(order):      # geometric phantom counts: a deep tree over every symbol
                    fl[s] = fl[s] + (1 << max(0, 40 - r))
                dorder = list(range(30))
                rng.shuffle(dorder)
                for r, s in enumerate(dorder):
                    fd[s] = fd[s] + (1 << max(0, 30 - r))
                blk.ll_lens = _trim(huffman_lengths(fl, 15), 257)
                blk.d_lens = _trim(huffman_lengths(fd, 15), 1)
            blocks.append(blk)
    blocks.append(Fixed([], final=True))
    return blocks


# ---------------------------------------------------------------------- the catalogue
OK, UNCOMPRESS, END_OF_BUFFER, BLOCK_HEADER, INVALID_SYMBOL = 0, 3, 5, 7, 8


@dataclass
class Case:
    """One raw DEFLATE stream and the reference's verdict on it: `want` is the output (valid) or
    the reference's error code.  `zlib` is False where zlib disagrees with the reference (`why`)."""
    name: str
    data: bytes
    want: object
    zlib: bool = True
    why: str = ""


def _lits(s):
    return list(s.encode() if isinstance(s, str) else s)


def _chain_block(tokens, ll_order, d_order, final=None):
    return Dynamic(tokens, ll_lens=_trim(chain_lengths(ll_order, 286), 257), d_lens=_trim(chain_lengths(d_order, 30), 1),
                   final=final)


def deep_token_blocks(prefix_bits, length=227 + 29, dist=32768, history=None):
    """A stored block of 32768+ bytes, then a dynamic block whose literal/length code is a chain
    (symbol 65 has 1 bit, the length symbol 284 and EOB 15 bits) and whose distance code is a chain
    (distance symbol 29 at 15 bits): `prefix_bits` one-bit literals, then the match -- a 48-bit token
    (15 + 5 + 15 + 13 bits) starting `prefix_bits` bits later -- then two more of them, back to back."""
    hist = history if history is not None else bytes((i * 131 + (i >> 7)) & 0xff for i in range(32768 + 100))
    ll_order = [65, 285, 66, 257, 67, 258, 68, 259, 69, 260, 70, 261, 262, 263, 284, 256]
    d_order = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 28, 29]
    ls, _ = length_symbol(length)
    assert ls == 284 and dist > 24576
    toks = [65] * prefix_bits + [(length, dist), (length, dist - 1), 66, (length, dist), 65]
    return [Stored(hist, final=False), _chain_block(toks, ll_order, d_order)]


def catalogue():
    """Named streams at the decoder's edges.  Codes are the reference's (pinned against the oracle)."""
    cases = []

    def add(name, blocks_or_bytes, want=None, zlib=True, why=""):
        data = blocks_or_bytes if isinstance(blocks_or_bytes, bytes) else raw(blocks_or_bytes)
        if want is None:
            want = replay(blocks_or_bytes)
        cases.append(Case(name, data, want, zlib, why))

    rng = random.Random(1951)
    # ---- block headers and stored blocks
    add("fixed_empty", [Fixed([])])
    add("btype_3", bytes([0x07]), BLOCK_HEADER)
    add("empty_input", b"", END_OF_BUFFER)
    add("nonfinal_block_then_end", [Fixed(_lits("abc"), final=False)], END_OF_BUFFER)
    add("stored_nlen_wrong", [Stored(b"abc", nlen=0)], UNCOMPRESS)
    add("stored_len_past_end", [Stored(b"abc", len_=10)], END_OF_BUFFER)
    add("stored_header_cut", raw([Stored(b"abcd")])[:3], END_OF_BUFFER)
    add("stored_0_after_unaligned_fixed", [Fixed(_lits("ABC"), final=False), Stored(b"")])
    big = rng.randbytes(65535)
    add("stored_65535_after_unaligned_dynamic", [Dynamic(_lits("hello hello") + [(5, 6)], final=False), Stored(big),
                                                 Fixed(_lits("z"))])
    add("stored_0_and_65535_after_stored", [Stored(b"", final=False), Stored(big, final=False), Stored(b"")])
    # ---- dynamic headers
    good = Dynamic(_lits("abcabcabc") + [(6, 3)])
    ll, dl = dynamic_header(good)
    add("dynamic_small", [good])
    for h in (287, 288):
        add("hlit_%d" % h, [Dynamic(good.tokens, ll + [0] * (h - len(ll)))], UNCOMPRESS)
    for h in (31, 32):
        add("hdist_%d" % h, [Dynamic(good.tokens, ll, dl + [0] * (h - len(dl)))], UNCOMPRESS)
    add("clc_oversubscribed", [Dynamic(good.tokens, cl_lens=[1] * 19)], UNCOMPRESS)
    add("clc_empty", [Dynamic(good.tokens, hclen=4, cl_lens=[0] * 19, rle=[])] , INVALID_SYMBOL)
    clc_one = [0] * 19
    clc_one[8] = 1                      # one code-length symbol ('8'), one bit: '0'; '1' matches nothing
    add("clc_undecodable", [Dynamic(good.tokens, cl_lens=clc_one, rle=[(8, 0), Bits(1, 1)])], INVALID_SYMBOL)
    add("repeat16_first", [Dynamic(good.tokens, ll, dl, rle=[(16, 0)] + rle_encode(ll + dl))], UNCOMPRESS)
    tail_zero = ll + dl
    n = len(tail_zero)
    add("repeat17_past_total", [Dynamic(good.tokens, ll, dl, rle=rle_encode(tail_zero[:n - 2]) + [(17, 0)])],
        UNCOMPRESS)
    add("repeat18_past_total", [Dynamic(good.tokens, ll, dl, rle=rle_encode(tail_zero[:n - 10]) + [(18, 0)])],
        UNCOMPRESS)
    add("repeat16_past_total", [Dynamic(good.tokens, ll, dl, rle=rle_encode(tail_zero[:n - 2]) + [(16, 0)])],
        UNCOMPRESS)
    # a 16 that starts in the literal/length lengths and ends in the distance lengths (RFC 1951 3.2.7 allows it)
    ll_x = [0] * 258
    ll_x[65], ll_x[66], ll_x[67], ll_x[256], ll_x[257] = 1, 3, 3, 3, 3
    d_x = [3, 3, 3, 3, 2, 2]
    blk = Dynamic(_lits("ABC") + [(3, 1), (3, 2), (3, 4), 65], ll_x, d_x)
    assert any(op[0] == 16 for op in rle_encode(ll_x + d_x))
    add("repeat16_across_lit_dist_boundary", [blk])
    d_z = [1, 1] + [0] * 20
    add("repeat18_ends_at_total", [Dynamic(_lits("xyxy") + [(4, 2), (3, 1)], d_lens=d_z)])
    ll_o = list(ll)
    ll_o[ord("a")] = ll_o[ord("b")] = ll_o[ord("c")] = 1
    add("ll_oversubscribed", [Dynamic(good.tokens, ll_o, dl)], UNCOMPRESS)
    add("dist_oversubscribed", [Dynamic(good.tokens, ll, [1, 1, 1])], UNCOMPRESS)
    ll_i = [0] * 257
    ll_i[65] = ll_i[66] = ll_i[256] = 2   # 3/4 of the code space
    add("ll_incomplete", [Dynamic(_lits("ABBA"), ll_i, [0])], zlib=False, why="zlib rejects incomplete codes")
    clc_inc = [0] * 19
    clc_inc[0], clc_inc[2], clc_inc[18] = 2, 2, 2  # 3/4 of the code space
    add("clc_incomplete", [Dynamic(_lits("ABBA"), ll_i, [0], cl_lens=clc_inc)], zlib=False,
        why="zlib rejects an incomplete code-length code")
    add("ll_undecodable", [Dynamic(_lits("AB") + [Bits(3, 2)], ll_i, [0])], UNCOMPRESS)
    add("single_distance_code", [Dynamic(_lits("abc") + [(5, 3), (3, 3)], d_lens=[0, 0, 1])])
    add("empty_distance_tree_literals_only", [Dynamic(_lits("only literals here"), d_lens=[0])])
    ll_e = [0] * 258
    ll_e[65] = ll_e[256] = 2
    ll_e[257] = 1
    add("empty_distance_tree_with_match", [Dynamic([65, Sym(257), 65], ll_e, [0])], UNCOMPRESS)
    # ---- fixed blocks: symbols and distances that have a code but no meaning
    for s in (286, 287):
        add("fixed_symbol_%d" % s, [Fixed(_lits("ab") + [Sym(s)] + _lits("cd"))], UNCOMPRESS)
    for d in (30, 31):
        add("fixed_distance_%d" % d, [Fixed(_lits("ab") + [Sym(257, 0, d)] + _lits("cd"))], UNCOMPRESS)
    all_lengths = [(L, 1 + (L * 7) % 40) for L in range(3, 259)]
    add("fixed_every_length", [Fixed(_lits(bytes(range(40))) + all_lengths)])
    add("fixed_every_distance", [Stored(rng.randbytes(32768), final=False),
                                 Fixed([(3 + k % 200, DIST_BASE[k] + (k * 997) % (1 << DIST_EXTRA[k])) for k in range(30)]
                                       + [(258, 32768), (3, 32768)])])
    # ---- distances at the edge of the output
    add("distance_equals_produced", [Fixed(_lits("abcde") + [(10, 5), (3, 15)])])
    add("distance_produced_plus_1", [Fixed(_lits("abcde") + [(10, 6)])], UNCOMPRESS)
    add("distance_on_first_token", [Fixed([(3, 1)])], UNCOMPRESS)
    h32 = rng.randbytes(32768)
    add("distance_32768_exact", [Stored(h32, final=False), Fixed([(258, 32768), (3, 32768), (4, 32767)])])
    add("distance_32768_one_short", [Stored(h32[:32767], final=False), Fixed([(258, 32768)])], UNCOMPRESS)
    add("distance_32768_in_second_block", [Stored(h32[:20000], final=False), Fixed(_lits(h32[:12768]), final=False),
                                           Fixed([(258, 32768), (200, 32768)])])
    # ---- where the input ends (bits past the end read as zero)
    add("truncated_dynamic_header_gap", bytes.fromhex("edfd81400000000020f8fb575555555501"), END_OF_BUFFER,
        why="HLIT 286, HDIST 30, code-length code {18:1, 1:2, 8:2}; input ends during the lengths")
    add("length_extra_past_end_empty_distance_tree", bytes.fromhex("e5e00109000000800064b37f298348"), UNCOMPRESS,
        why="code {65, 256, 284} at 2 bits, one distance length 0; 284's extra bits lie past the end")
    # the last repeat code of a header ends on the last byte; its 7 extra bits lie past the end:
    # read as zeros the repeat is 11 (fits, then the next symbol is past the end), read as ones 138 (too long)
    clc_r = [0] * 19
    clc_r[18], clc_r[1], clc_r[8] = 1, 2, 2
    hdr = Dynamic([], [0] * 286, [0] * 30, cl_lens=clc_r, rle=[(18, 127), (18, 127)] + [(1, 0)] * 20 + [(18, 0)], eob=False)
    add("repeat_extra_bits_past_end", raw([hdr])[:16], END_OF_BUFFER)
    hdr2 = Dynamic([], [0] * 286, [0] * 30, cl_lens=clc_r, rle=[(18, 127), (18, 127)] + [(1, 0)] * 24 + [(18, 0)], eob=False)
    add("repeat_extra_bits_past_end_overshoots", raw([hdr2])[:17] + b"\x00", UNCOMPRESS)
    # a fixed length code that ends on the last byte: its distance code lies past the end (zeros: distance 1)
    cut = raw([Fixed([0x90] * 6 + [(3, 1)] + _lits("tail"))])
    add("distance_code_past_end", cut[:8], END_OF_BUFFER)
    cut = raw([Fixed([0x90] * 4 + [(131, 1)] + _lits("tail"))])   # symbol 281 (8-bit code) + 5 extra bits
    add("length_extra_past_end_fixed", cut[:(3 + 36 + 8 + 7) // 8], END_OF_BUFFER)
    add("fixed_symbol_286_past_end", raw([Fixed([0x90] * 5 + [Sym(286)])])[:6], END_OF_BUFFER)
    add("fixed_symbol_286_at_end", raw([Fixed([0x90] * 5 + [Sym(286)], eob=False)]), UNCOMPRESS)
    add("missing_end_of_block", raw([Fixed(_lits("abc"), eob=False)]), END_OF_BUFFER)
    s = raw([Fixed(_lits("abcdefgh") * 3 + [(20, 8)])])
    add("truncated_mid_tokens", s[:len(s) // 2], END_OF_BUFFER)
    add("distance_too_far_with_extra_past_end", raw([Fixed(_lits("abc") + [(3, 100)])])[:5], END_OF_BUFFER)
    # ---- 48-bit tokens (15-bit length code + 5 extra + 15-bit distance code + 13 extra)
    for p in (0, 1, 17, 31):
        add("deep_token_phase_%d" % p, deep_token_blocks(p))
    return cases


def placements_cut(data):
    """Every byte cut of `data` (the truncated streams a placement test puts next to other bytes)."""
    return [data[:k] for k in range(len(data))]
