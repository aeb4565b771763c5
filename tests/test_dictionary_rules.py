"""The preset-dictionary rules the GPU tests rely on, checked on the CPU alone.

Decoding a raw stream S against a dictionary D is defined as decoding stored(W) || S and dropping the first |W|
output bytes (W: the last min(32768, |D|) bytes of D; stored(W): one non-final stored block).  Here that
definition is checked against zlib's own inflateSetDictionary (Python zlib's zdict), and the CPU oracle's verdict
on stored(W) || S is shown to be an expected verdict for any stream, corrupted ones included."""
import random
import zlib

import pytest

from oracle import oracle as o
from tests import util

WINDOWS = [1, 100, 8191, 8193, 32767, 32768, 100000]


def window(d):
    return d[-32768:]


def stored(w):
    n = len(w)
    return bytes([0, n & 255, n >> 8, ~n & 255, (~n >> 8) & 255]) + w


@pytest.fixture(scope="module")
def text():
    return util.text_corpus(util.load_corpus())


def _dict_and_msg(text, dlen, seed):
    rng = random.Random(seed)
    a = rng.randrange(0, len(text) - dlen - 70000)
    return text[a:a + dlen], text[a + dlen - 5000:a + dlen - 5000 + 20000]


@pytest.mark.parametrize("dlen", WINDOWS)
@pytest.mark.parametrize("level", [1, 6, 9])
def test_definition_matches_zlib(text, dlen, level):
    d, m = _dict_and_msg(text, dlen, dlen * 10 + level)
    co = zlib.compressobj(level, zlib.DEFLATED, -15, zdict=d)
    s = co.compress(m) + co.flush()
    w = window(d)
    do = zlib.decompressobj(-15, zdict=d)
    assert do.decompress(s) == m
    assert zlib.decompress(stored(w) + s, -15)[len(w):] == m
    # the oracle decodes the definition too
    assert o.uncompress(stored(w) + s, o.dfDeflate)[len(w):] == m


def test_dictid_is_adler_of_whole_dictionary(text):
    d = text[:100000]
    co = zlib.compressobj(6, zlib.DEFLATED, 15, zdict=d)
    z = co.compress(b"hello hello") + co.flush()
    assert z[:2] == b"\x78\xbb" and z[1] & 0x20
    assert int.from_bytes(z[2:6], "big") == zlib.adler32(d)
    assert (0x7820 % 31) == 0  # the header this library writes: FDICT, FLEVEL 0


def oracle_status(data):
    try:
        o.uncompress(data, o.dfDeflate)
        return 0
    except o.ZippyError as e:
        return e.code


def test_oracle_verdict_of_definition_is_total(text):
    """Every corrupted stream gets a verdict from the oracle on stored(W) || S (the GPU tests' expected table);
    zlib agrees wherever both accept."""
    d, m = _dict_and_msg(text, 32768, 7)
    w = window(d)
    co = zlib.compressobj(6, zlib.DEFLATED, -15, zdict=d)
    s = co.compress(m[:3000]) + co.flush()
    rng = random.Random(3)
    seen = set()
    for k in range(300):
        b = bytearray(s)
        kind = k % 3
        if kind == 0:
            i = rng.randrange(len(b) * 8)
            b[i // 8] ^= 1 << (i % 8)
        elif kind == 1:
            b = b[:rng.randrange(len(b))]
        else:
            b += bytes(rng.randrange(256) for _ in range(rng.randrange(1, 9)))
        st = oracle_status(stored(w) + bytes(b))
        assert 0 <= st <= 18
        seen.add(st)
        if st == 0:
            out = o.uncompress(stored(w) + bytes(b), o.dfDeflate)[len(w):]
            try:
                zo = zlib.decompressobj(-15, zdict=d)
                assert zo.decompress(bytes(b)) == out
            except zlib.error:
                pass
    assert 0 in seen and len(seen) > 2
