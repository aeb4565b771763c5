"""The packer (k_pack) is a pure function of the parse's tokens and the chunk's codebook.  These tests pin the exact
bytes it writes: SHA-256 digests of whole batches, taken from the packer before it became a branch-free emitter
fed from shared memory, for levels 1, -2, 0 and Default (k_lz2's records go through the same packer) in all three
formats.  Every member must also round-trip through the oracle, zlib and the GPU inflate.

The batches hold C2-style text blocks, urls and html windows, random bytes (stored blocks), run-length blobs (long
matches, windows whose matches hit the lane cap) and very short inputs (fixed blocks); chunk lengths that are not
multiples of 32 bytes or of 8 KiB, members shorter than 8 KiB (packer warps with no sub-chunk), members of several
chunks (sync joints), sources at every address alignment mod 4, and, in gzip, FNAME lengths 0 to 25 in one batch so
that members start at every output byte alignment mod 4."""
import hashlib
import random
import zlib

import pytest

from tests import util

pytestmark = pytest.mark.gpu

LEVELS = {"l1": 1, "l-2": -2, "l0": 0, "default": -1}
FORMATS = ("gzip", "zlib", "deflate")

# digests of b"".join(len(member).to_bytes(8) + member) for each batch
DIGESTS = {
    "l1/gzip": "7992917c124de32aa262a5cbad87220bca36dad54fcdf700ca8d5e7566f2dc5c",
    "l1/zlib": "659eb803cdd19998beda319781449bd3ee774f33928d1eabe4e4eccf1587bd07",
    "l1/deflate": "d9e6a71ad7c5444bea4ba7e83946c662a18d4b3416cd0000da53a7b2eb1257c0",
    "l-2/gzip": "47b1c5248c4e277cb804492e7eb1e08d487f894f84584eecaaf793be0e13b9f8",
    "l-2/zlib": "fce7de64da3c0d062f18027fd65b663ae550a5d29ceb57374a513d58fa1e978e",
    "l-2/deflate": "825a4204222042c2c13ecdbc3837f7f7d1222aab11ad0560b7a1f87df06fc411",
    "l0/gzip": "e78cfbb9fe8a13c2fabc9f7ca4b16b5c736420a31c963288ace5f6ecc87ed6b9",
    "l0/zlib": "31c1cc2f0720d406198c8842394d242f1c4815c3405e3cf613b27c9846e78bd7",
    "l0/deflate": "ea44b940d330d2e28dee8b468c124e273f6f1a4abbcfabd69d648420e22af00c",
    "default/gzip": "4353215f6650ba35c8347a4c77bc06998353aed779d2b10d7c363d514c012224",
    "default/zlib": "c480d57443206a19316db4c28a871d133143b3f1230aa899ca149b8563a563ef",
    "default/deflate": "a78f8fc99d97f8006687b2a88fe3ff950c0c0d59d5c2db6a50f0813920bbd693",
}


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


def _inputs():
    rng = random.Random(0x9AC4)
    corpus = util.load_corpus()
    T = util.text_corpus(corpus)
    urls, html = corpus["urls.10K"], corpus["html"]
    xs = [util.c2_block(T, i) for i in range(6)]
    for n in (65536, 40000 + 3, 8191, 5000 + 1, 33, 1, 2):  # text windows at ragged lengths
        o = rng.randrange(len(urls) - n)
        xs.append(urls[o:o + n])
        o = rng.randrange(len(html) - n)
        xs.append(html[o:o + n])
    for n in (65536 * 3 + 777, 65536 * 2 + 12345, 65536 + 1, 65536 * 4):  # several chunks: sync joints
        o = rng.randrange(len(T) - n)
        xs.append(T[o:o + n])
    xs.append(bytes(rng.randrange(256) for _ in range(70001)))  # stored
    xs.append(bytes(rng.randrange(256) for _ in range(3000)))
    for _ in range(4):
        xs.append(util.run_length_blob(rng, 150000))
    xs += [b"\x00" * 65537, b"ab" * 3001, b"abc" * 700 + b"x"]
    xs += [b"", b"a", b"hi", b"abcd", b"hello, hello, hello", bytes(range(64))]  # fixed blocks
    # sources at every alignment mod 4: the inputs are packed back to back
    for k in range(4):
        xs.append(b"z" * (k + 1))
        o = rng.randrange(len(T) - 20000)
        xs.append(T[o:o + 20000 + k])
    return xs


def _fname_lens(n):
    return [(0, 25, 1, 2, 3)[i % 5] for i in range(n)]


def _compress(z, xs, level, fmt):
    df = {"gzip": z.dfGzip, "zlib": z.dfZlib, "deflate": z.dfDeflate}[fmt]
    return z.compress_batch(xs, level, df, _fname_lens(len(xs)) if fmt == "gzip" else None)


def _digest(comp):
    h = hashlib.sha256()
    for c in comp:
        h.update(len(c).to_bytes(8, "little"))
        h.update(bytes(c))
    return h.hexdigest()


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("level", list(LEVELS))
def test_packer_output_is_pinned(z, level, fmt):
    comp = _compress(z, _inputs(), LEVELS[level], fmt)
    assert _digest(comp) == DIGESTS["%s/%s" % (level, fmt)]


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("level", list(LEVELS))
def test_packer_output_round_trips(z, level, fmt):
    from oracle import oracle as o
    xs = _inputs()
    comp = _compress(z, xs, LEVELS[level], fmt)
    wbits = {"gzip": 31, "zlib": 15, "deflate": -15}[fmt]
    odf = {"gzip": o.dfGzip, "zlib": o.dfZlib, "deflate": o.dfDeflate}[fmt]
    zdf = {"gzip": z.dfGzip, "zlib": z.dfZlib, "deflate": z.dfDeflate}[fmt]
    back = z.uncompress_batch(comp, zdf)
    for x, c, b in zip(xs, comp, back):
        d = zlib.decompressobj(wbits)
        assert d.decompress(c) + d.flush() == x and d.eof and d.unused_data == b""
        assert o.uncompress(c, odf) == x
        assert b == x


def test_gzip_members_start_at_every_alignment(z):
    """The FNAME lengths put the first chunks of the gzip batch's members at every byte offset mod 4."""
    comp = _compress(z, _inputs(), 1, "gzip")
    fl = _fname_lens(len(comp))
    starts, off = set(), 0
    for c, k in zip(comp, fl):
        assert c[3] == 8 and c[10:10 + k] == bytes(range(97, 97 + k)) and c[10 + k] == 0
        starts.add((off + 11 + k) % 4)
        off += len(c)
    assert starts == {0, 1, 2, 3}
