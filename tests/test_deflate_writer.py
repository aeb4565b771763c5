"""Pins tests/deflate_writer.py (the independent DEFLATE writer the GPU edge tests are built on) against
system zlib and the CPU oracle, so that a GPU failure on one of its streams points at the kernel and not
at the helper.  CPU only."""
import zlib

import pytest

from tests import deflate_writer as w


@pytest.fixture(scope="module")
def o():
    from oracle import oracle
    return oracle


def _oracle(o, data, fmt=3):
    try:
        return o.uncompress(data, fmt) if fmt != 3 else o.inflate(data)
    except o.ZippyError as e:
        return e.code


CASES = w.catalogue()


def test_catalogue_names_are_unique():
    names = [c.name for c in CASES]
    assert len(names) == len(set(names))
    assert sum(isinstance(c.want, int) for c in CASES) >= 30 and sum(isinstance(c.want, bytes) for c in CASES) >= 15


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_catalogue_case(o, case):
    """Valid cases: zlib and the oracle give the replay bytes (or zlib rejects, where the catalogue says the
    reference accepts what zlib does not).  Invalid cases: the oracle returns exactly the catalogued code."""
    got = _oracle(o, case.data)
    assert got == case.want, (case.name, got if isinstance(got, int) else len(got))
    try:
        z = zlib.decompress(case.data, -15)
    except zlib.error:
        z = None
    if isinstance(case.want, bytes) and case.zlib:
        assert z == case.want
    else:   # rejected by zlib: an invalid stream, or a valid one whose disagreement the catalogue names
        assert z is None, "zlib accepts a stream the reference rejects (or the catalogue is stale)"
        assert isinstance(case.want, int) or case.why
    if isinstance(case.want, bytes):   # the wrappers around it decode the same way
        assert _oracle(o, w.zlib_wrap(case.data, case.want), 1) == case.want
        assert _oracle(o, w.gzip_wrap(case.data, case.want, fname=b"x"), 2) == case.want


def test_wrong_trailers(o):
    data = b"trailer test " * 50
    blocks = [w.Fixed(list(data[:13]) + [(254, 13), (258, 13), (125, 13)])]
    s = w.raw(blocks)
    assert w.replay(blocks) == data
    assert _oracle(o, w.zlib_wrap(s, data), 1) == data
    assert _oracle(o, w.zlib_wrap(s, data, adler=w.adler32(data) ^ 1), 1) == 14
    assert _oracle(o, w.gzip_wrap(s, data, crc=w.crc32(data) ^ 1), 2) == 14
    assert _oracle(o, w.gzip_wrap(s, data, isize=len(data) + 1), 2) == 18
    assert w.crc32(data) == zlib.crc32(data) and w.adler32(data) == zlib.adler32(data)
    big = bytes(range(256)) * 9000
    assert w.adler32(big) == zlib.adler32(big)


@pytest.mark.parametrize("skew", ["flat", "deep"])
@pytest.mark.parametrize("dist", ["one", "short", "far", "dependent"])
def test_random_streams(o, skew, dist):
    """The seeded generator: every knob, zlib and the oracle agree with the replay."""
    n15 = 0
    for seed in range(12):
        blocks = w.random_stream(seed, skew=skew, dist=dist, phase=(seed * 7) % 32,
                                 history=32768 + 17 if dist in ("far", "dependent") else 0,
                                 kinds=("dynamic", "fixed", "stored") if seed % 3 else ("dynamic",))
        s = w.raw(blocks)
        want = w.replay(blocks)
        assert zlib.decompress(s, -15) == want, seed
        assert o.inflate(s) == want, seed
        for b in blocks:
            if isinstance(b, w.Dynamic):
                ll, d = w.dynamic_header(b)
                n15 += max(ll) == 15 and max(d) == 15
    assert (n15 > 0) == (skew == "deep")


def test_phase_block_sets_the_bit_phase():
    for p in range(32):
        pos, _ = w.block_bits([w.phase_block(p), w.Fixed([])])
        assert pos[1] % 32 == p


def test_deep_tokens_are_48_bits():
    blocks = w.deep_token_blocks(0)
    ll, d = w.dynamic_header(blocks[1])
    assert ll[284] == 15 and d[29] == 15 and w.LEN_EXTRA[284 - 257] == 5 and w.DIST_EXTRA[29] == 13
    one = w.Dynamic([65], ll, d)
    two = w.Dynamic([65, (256, 32768)], ll, d)
    assert w.block_bits([two])[1] - w.block_bits([one])[1] == 48
