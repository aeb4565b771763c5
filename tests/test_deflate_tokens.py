"""CPU tests of the DEFLATE token reader (tests/deflate_tokens.py): the tokens it reads must rebuild exactly
what zlib decodes, on zlib's own streams of every strategy and on the hand-built streams of deflate_writer,
and it must refuse every malformed stream of that catalogue."""
import random
import zlib

import pytest

from tests import deflate_tokens as dt
from tests import deflate_writer as dw
from tests import util


@pytest.fixture(scope="module")
def samples(corpus):
    rng = random.Random(1951)
    T = util.text_corpus(corpus)
    return {
        "text": T[:300000],
        "html": corpus["html"],
        "random": rng.randbytes(70000),
        "runs": util.run_length_blob(random.Random(7), 150000),
        "zeros": b"\x00" * 100000,
        "empty": b"",
        "one": b"x",
        "short": b"hello, hello, hello",
    }


def _zraw(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flush_every=None):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy)
    if flush_every is None:
        return c.compress(data) + c.flush()
    out = b""
    for i in range(0, len(data), flush_every):
        out += c.compress(data[i:i + flush_every]) + c.flush(zlib.Z_FULL_FLUSH)
    return out + c.flush()


def _check(raw, want):
    blocks = dt.parse(raw)
    assert dt.rebuild(blocks) == want
    assert blocks[-1].final and not any(b.final for b in blocks[:-1])
    for a, b in zip(blocks, blocks[1:]):
        assert a.bit_end == b.bit_start
    for b in blocks:
        for t in b.tokens:
            assert isinstance(t, int) and 0 <= t < 256 or 3 <= t[0] <= 258 and 1 <= t[1] <= 32768
    return blocks


@pytest.mark.parametrize("level", [0, 1, 6, 9])
def test_zlib_levels(samples, level):
    for name, x in samples.items():
        blocks = _check(_zraw(x, level), x)
        if level == 0:
            assert all(b.btype == 0 for b in blocks), name
        elif name == "text":
            assert any(b.btype == 2 and any(not isinstance(t, int) for t in b.tokens) for b in blocks)


@pytest.mark.parametrize("strategy", ["fixed", "huffman_only", "rle"])
def test_zlib_strategies(samples, strategy):
    st = {"fixed": zlib.Z_FIXED, "huffman_only": zlib.Z_HUFFMAN_ONLY, "rle": zlib.Z_RLE}[strategy]
    for name, x in samples.items():
        blocks = _check(_zraw(x, 6, st), x)
        toks = [t for b in blocks for t in b.tokens]
        if strategy == "fixed" and x:
            assert {b.btype for b in blocks} <= {0, 1} and 1 in {b.btype for b in blocks} or name == "random", name
        if strategy == "huffman_only":
            assert all(isinstance(t, int) for t in toks), name
        if strategy == "rle":
            assert all(isinstance(t, int) or t[1] == 1 for t in toks), name


def test_full_flush_streams(samples):
    x = samples["text"]
    for every in (1, 1000, 65536):
        blocks = _check(_zraw(x[:120000], 6, flush_every=every), x[:120000])
        joints = [b for b in blocks if b.btype == 0 and not b.tokens and not b.final]
        assert len(joints) >= (120000 + every - 1) // every


def test_writer_catalogue():
    """Every valid stream of the catalogue rebuilds to its definition; every invalid one is refused."""
    valid = invalid = 0
    for case in dw.catalogue():
        if isinstance(case.want, bytes):
            blocks = dt.parse(case.data)
            assert dt.rebuild(blocks) == case.want, case.name
            if case.zlib:
                assert zlib.decompress(case.data, -15) == case.want, case.name
            valid += 1
        else:
            with pytest.raises(dt.Malformed):
                dt.parse(case.data)
            invalid += 1
    assert valid >= 20 and invalid >= 30


def test_writer_tokens_read_back():
    """The reader returns exactly the tokens a stream was written with, block by block, with each block's
    bit extent."""
    rng = random.Random(5)
    for seed in range(12):
        hist = rng.randbytes(40000)
        toks = list(b"abcdefgh") + [(3, 1), (258, 8), (4, 32768 if seed % 2 else 9)] + list(rng.randbytes(20))
        toks += [(rng.randrange(3, 259), rng.randrange(1, 30000)) for _ in range(200)]
        blocks = [dw.Stored(hist, final=False), dw.Dynamic(toks, final=False), dw.Fixed(toks[::-1][:50] + [65])]
        raw = dw.raw(blocks)
        got = dt.parse(raw)
        assert [b.btype for b in got] == [0, 2, 1]
        assert got[0].tokens == list(hist) and got[1].tokens == toks and got[2].tokens == toks[::-1][:50] + [65]
        starts, end = dw.block_bits(blocks)
        assert [b.bit_start for b in got] == starts and got[-1].bit_end == end
        assert dt.rebuild(got) == dw.replay(blocks)


def test_member_chunk_layout():
    """The layout of a member this library writes: one fixed or dynamic block per 64 KiB chunk, each but the
    last followed by the 00 00 ff ff joint; stored chunks as stored blocks of at most 65535 bytes."""
    rng = random.Random(9)
    text = bytes(rng.choice(b"abcd efgh") for _ in range(65536))
    lit = list(text)
    rnd = rng.randbytes(65536)
    joint = dw.Stored(b"", final=False)
    blocks = [dw.Dynamic(lit, final=False), joint,
              dw.Stored(rnd[:65535], final=False), dw.Stored(rnd[65535:], final=False),
              dw.Fixed(lit, final=False), joint,
              dw.Fixed(list(b"tail") + [(4, 4)])]
    raw = dw.raw(blocks)
    assert raw.count(b"\x00\x00\xff\xff") >= 2
    chunks = dt.member_chunks(dt.parse(raw))
    assert [c.btype for c in chunks] == [2, 0, 1, 1]
    assert chunks[0].tokens == lit and chunks[1].tokens == list(rnd) and chunks[2].tokens == lit
    assert chunks[3].tokens == list(b"tail") + [(4, 4)]
    # a short chunk that is not the member's last, and a compressed chunk without its joint, are refused
    for bad in ([dw.Fixed(lit[:-1], final=False), joint, dw.Fixed([65])],
                [dw.Fixed(lit, final=False), dw.Fixed([65])],
                [dw.Stored(rnd[:1000], final=False), dw.Fixed([65])]):
        with pytest.raises(dt.Malformed):
            dt.member_chunks(dt.parse(dw.raw(bad)))
    # the same layout from zlib: full flushes every 64 KiB
    x = (text + rnd) * 2
    blocks = dt.parse(_zraw(x, 6, flush_every=65536))
    assert dt.rebuild(blocks) == x


def test_malformed_streams_are_refused():
    good = dw.raw([dw.Dynamic(list(b"abcabcabc") + [(6, 3)])])
    for bad in (good[:len(good) // 2], b"", b"\x07", bytes([0x01, 0x03, 0x00, 0xfc, 0xff, 0x61])):
        with pytest.raises(dt.Malformed):
            dt.parse(bad)
    with pytest.raises(dt.Malformed):
        dt.parse(dw.raw([dw.Fixed([(3, 1)])]))
