"""The chunk checksums of the level 0 / -2 / 1 compressor (k_lz) are computed only for the format that needs
them: CRC-32 for gzip, Adler-32 for zlib, neither for raw DEFLATE.  These tests pin the trailers that come out
of each format against zlib's own checksums, on the edge inputs and on members of many chunks with ragged last
chunks, and check that raw DEFLATE (no checksum) still inflates to the input."""
import random
import struct
import zlib

import pytest

from tests import util

pytestmark = pytest.mark.gpu

LEVELS = [0, -2, 1]


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


def _inputs():
    rng = random.Random(77)
    corpus = util.load_corpus()
    T = util.text_corpus(corpus)
    xs = util.edge_inputs()
    # members of several 64 KiB chunks, 4 KiB pieces and phases, with ragged ends
    for n in (65536 * 3, 65536 * 5 + 4097, 65536 * 2 + 1, 300000 + 31):
        o = rng.randrange(len(T) - n)
        xs.append(T[o:o + n])
    xs.append(bytes(rng.randrange(256) for _ in range(140001)))
    return xs


@pytest.mark.parametrize("level", LEVELS)
def test_gzip_trailer_is_zlib_crc32(z, level):
    xs = _inputs()
    comp = z.compress_batch(xs, level, z.dfGzip)
    for x, c in zip(xs, comp):
        crc, isize = struct.unpack("<II", c[-8:])
        assert crc == zlib.crc32(x) and isize == len(x) & 0xffffffff
        assert zlib.decompress(c, 31) == x


@pytest.mark.parametrize("level", LEVELS)
def test_zlib_trailer_is_zlib_adler32(z, level):
    xs = _inputs()
    comp = z.compress_batch(xs, level, z.dfZlib)
    for x, c in zip(xs, comp):
        assert struct.unpack(">I", c[-4:])[0] == zlib.adler32(x)
        assert zlib.decompress(c) == x


@pytest.mark.parametrize("level", LEVELS)
def test_raw_deflate_has_no_trailer(z, level):
    xs = _inputs()
    comp = z.compress_batch(xs, level, z.dfDeflate)
    for x, c in zip(xs, comp):
        d = zlib.decompressobj(-15)
        assert d.decompress(c) + d.flush() == x and d.eof and d.unused_data == b""


def test_one_batch_mixes_nothing_across_formats(z):
    """The same inputs through the three formats in turn on one context: each trailer is the format's own."""
    xs = _inputs()[-6:]
    ctx_g = z.compress_batch(xs, 1, z.dfGzip)
    ctx_r = z.compress_batch(xs, 1, z.dfDeflate)
    ctx_z = z.compress_batch(xs, 1, z.dfZlib)
    for x, g, r, zz in zip(xs, ctx_g, ctx_r, ctx_z):
        # the DEFLATE payload does not depend on the format
        assert g[-8 - len(r):-8] == r and zz[2:-4] == r
        assert struct.unpack("<I", g[-8:-4])[0] == zlib.crc32(x)
        assert struct.unpack(">I", zz[-4:])[0] == zlib.adler32(x)
