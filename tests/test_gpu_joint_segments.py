"""Large members of this library's levels -1 and 2..9 decode as parallel marker segments at their sync joints
(zb_api.cu: inflate_member_joints; zb_inflate.cu: the parallel window resolve).  Every case checks the bytes
against the input or the oracle, and the exact launch count, which shows that the member took the new path and
did not fall back to the speculative segments or the serial decode."""
import zipfile

import numpy as np
import pytest

from tests import util

pytestmark = pytest.mark.gpu

CHUNK = 65536
# launches per single-member uncompress_batch call: the ordinary launch + 2 verify kernels, the joint search and
# the optimistic pass; then per window a marker prefill, the marker decode and 4 resolve kernels; 1 per count pass
BASE, PER_WINDOW = 5, 6


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


@pytest.fixture(scope="module")
def o():
    from oracle import oracle
    return oracle


def _ctx(z, monkeypatch, big=100000, window=None, joints=True):
    monkeypatch.setenv("ZB200_BIG_MEMBER_BYTES", str(big))
    if window:
        monkeypatch.setenv("ZB200_MARK_WINDOW_SEGS", str(window))
    if not joints:
        monkeypatch.setenv("ZB200_JOINT_MARKERS", "0")
    ctx = z.Context()
    for k in ("ZB200_BIG_MEMBER_BYTES", "ZB200_MARK_WINDOW_SEGS", "ZB200_JOINT_MARKERS"):
        monkeypatch.delenv(k, raising=False)
    return ctx


def _one(ctx, blob, fmt, sizes=None):
    base = np.frombuffer(blob, dtype=np.uint8)
    offs = np.array([0, len(blob)], dtype=np.uint64)
    out, do, lens, st = ctx.uncompress_batch(base, offs, fmt, sizes=sizes)
    got = out[int(do[0]):int(do[0]) + int(lens[0])].tobytes() if st[0] == 0 else None
    return got, int(st[0]), ctx.timing()["kernel_launches"]


def _comp(ctx, z, raw, level, fmt):
    c = ctx.compress_batch(np.frombuffer(raw, dtype=np.uint8), np.array([0, len(raw)], dtype=np.uint64), level, fmt)
    return c[0][:int(c[1][1])].tobytes()


def _data(corpus, kind, n, seed=1):
    rng = np.random.default_rng(seed)
    T = util.text_corpus(corpus)
    if kind == "text":
        return (T * (1 + n // len(T)))[:n]
    if kind == "runs":
        runs = rng.integers(1, 300, n // 50 + 1)
        return np.repeat(rng.integers(0, 256, len(runs), dtype=np.uint8), runs)[:n].tobytes()
    if kind == "zeros":
        return bytes(n)
    if kind == "random":
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    # mix: text, runs and random pieces that do not line up with the 64 KiB chunks
    parts, k = [], 0
    while sum(map(len, parts)) < n:
        m = int(rng.integers(20000, 300000))
        parts.append(_data(corpus, ("text", "runs", "random")[k % 3], m, seed + k))
        k += 1
    return b"".join(parts)[:n]


def _windows(nseg, w):
    return (nseg + w - 1) // w


@pytest.mark.parametrize("level", [-1, 2, 6, 9])
@pytest.mark.parametrize("kind", ["text", "runs", "zeros"])
def test_own_members_all_wrappers(z, corpus, monkeypatch, level, kind):
    """64 KiB of output per joint: the guess holds, no count pass.  Zero runs make every chunk refer into the
    previous one, so reference chains go through every segment."""
    ctx = _ctx(z, monkeypatch, big=1000)   # (zero runs compress to a few KiB)
    raw = _data(corpus, kind, 3_000_000 + 12345)
    nseg = (len(raw) + CHUNK - 1) // CHUNK
    for fmt in (z.dfGzip, z.dfZlib, z.dfDeflate):
        blob = _comp(ctx, z, raw, level, fmt)
        got, st, launches = _one(ctx, blob, fmt)
        assert st == 0 and got == raw, (fmt, st)
        assert launches == BASE + PER_WINDOW * _windows(nseg, 8192), (fmt, launches)
    ctx.close()


@pytest.mark.parametrize("level", [-1, 6])
def test_mixed_and_random_members(z, o, corpus, monkeypatch, level):
    """Stored chunks (random bytes) carry no joint after them, so segments differ from 64 KiB: the optimistic pass
    says so and one count pass in marker mode sizes them.  Random bytes alone have no joints at all and keep the
    existing path (see DESIGN section 8)."""
    ctx = _ctx(z, monkeypatch)
    raw = _data(corpus, "mix", 4_000_000, seed=level + 5)
    for fmt in (z.dfGzip, z.dfZlib, z.dfDeflate):
        blob = _comp(ctx, z, raw, level, fmt)
        got, st, launches = _one(ctx, blob, fmt)
        assert st == 0 and got == raw, (fmt, st)
        assert launches == BASE + 1 + PER_WINDOW, (fmt, launches)
    rnd = _data(corpus, "random", 2_000_000)
    got, st, _ = _one(ctx, _comp(ctx, z, rnd, level, z.dfGzip), z.dfGzip)
    assert st == 0 and got == rnd
    ctx.close()


def test_multi_window_members(z, corpus, monkeypatch):
    ctx = _ctx(z, monkeypatch, big=1000, window=7)
    for kind in ("text", "zeros", "mix"):
        raw = _data(corpus, kind, 5_000_000 + 999)
        nseg = (len(raw) + CHUNK - 1) // CHUNK
        for fmt in (z.dfGzip, z.dfDeflate):
            blob = _comp(ctx, z, raw, z.DefaultCompression, fmt)
            got, st, launches = _one(ctx, blob, fmt)
            assert st == 0 and got == raw, (kind, fmt, st)
            if kind != "mix":
                assert launches == BASE + PER_WINDOW * _windows(nseg, 7), (kind, launches)
            else:
                assert launches >= BASE + 1 + 2 * PER_WINDOW, launches
    ctx.close()


def test_sizes_and_single_calls(z, corpus, monkeypatch):
    ctx = _ctx(z, monkeypatch)
    raw = _data(corpus, "text", 2_500_000)
    for fmt in (z.dfZlib, z.dfDeflate):
        blob = _comp(ctx, z, raw, z.DefaultCompression, fmt)
        sizes = ctx.uncompressed_sizes(np.frombuffer(blob, dtype=np.uint8), np.array([0, len(blob)], dtype=np.uint64), fmt)
        assert int(np.asarray(sizes[0])[0]) == len(raw), sizes
    assert ctx.decode_one(_comp(ctx, z, raw, z.DefaultCompression, z.dfZlib)) == raw
    assert ctx.inflate(_comp(ctx, z, raw, z.DefaultCompression, z.dfDeflate)) == raw
    ctx.close()


def test_false_joints_are_repaired(z, o, corpus, monkeypatch):
    """00 00 ff ff inside stored chunks (random bytes with the pattern planted) is a false joint: the segments on
    both sides fail the count pass, the joint is dropped and the member still decodes in parallel."""
    ctx = _ctx(z, monkeypatch)
    rng = np.random.default_rng(9)
    T = _data(corpus, "text", 1_500_000)
    rnd = bytearray(rng.integers(0, 256, 6 * CHUNK, dtype=np.uint8).tobytes())
    for p in (1000, CHUNK + 30000, 3 * CHUNK + 5, 5 * CHUNK + 60000):
        rnd[p:p + 4] = b"\x00\x00\xff\xff"
    raw = T[:700000] + bytes(rnd) + T[700000:]
    for fmt in (z.dfGzip, z.dfZlib, z.dfDeflate):
        blob = _comp(ctx, z, raw, z.DefaultCompression, fmt)
        got, st, launches = _one(ctx, blob, fmt)
        assert st == 0 and got == raw, (fmt, st)
        # the 64 KiB guess (prefill + decode) fails, a count pass fails, the repaired one passes
        assert launches == BASE + 2 + 2 + PER_WINDOW, (fmt, launches)
    ctx.close()


def test_corrupt_and_truncated_members_get_the_oracles_status(z, o, corpus, monkeypatch):
    ctx = _ctx(z, monkeypatch)
    raw = _data(corpus, "mix", 2_000_000, seed=3)
    good = _comp(ctx, z, raw, z.DefaultCompression, z.dfGzip)
    rng = np.random.default_rng(11)
    for k in range(16):
        bad = bytearray(good)
        pos = int(rng.integers(20, len(bad)))
        bad[pos] ^= 1 << int(rng.integers(0, 8))
        got, st, _ = _one(ctx, bytes(bad), z.dfDetect)
        try:
            want = o.uncompress(bytes(bad))
        except o.ZippyError as e:
            assert st == e.code, (k, pos, st, e.code)
            continue
        assert st == 0 and got == want, k
    for cut in (len(good) // 3, len(good) - 9, len(good) - 1):
        got, st, _ = _one(ctx, good[:cut], z.dfDetect)
        try:
            o.uncompress(good[:cut])
            raise AssertionError("the oracle accepted a truncated member")
        except o.ZippyError as e:
            assert st == e.code, (cut, st, e.code)
    ctx.close()


def test_off_hook_gives_the_same_bytes(z, corpus, monkeypatch):
    ctx = _ctx(z, monkeypatch, joints=False)
    raw = _data(corpus, "text", 1_000_000)
    blob = _comp(ctx, z, raw, z.DefaultCompression, z.dfGzip)
    got, st, launches = _one(ctx, blob, z.dfGzip)
    # the parent's sequence: the count pass fails, the speculative segments (block search, count, prefill + marker
    # decode, two resolve kernels) take the member
    assert st == 0 and got == raw and launches == BASE + 2 + 6, launches
    ctx.close()


def test_tarball_and_zip_archive_read_back(z, corpus, tmp_path):
    """Default-level members through the archive readers at the library's default thresholds."""
    import zippy_b200.tarballs as tb
    import zippy_b200.ziparchives as za
    contents = {"d": tb.TarballEntry("dir")}
    big = _data(corpus, "mix", 9_000_000, seed=21)
    contents["d/big.bin"] = tb.TarballEntry("file", big, 1700000000, 0o644)
    contents["d/t.txt"] = tb.TarballEntry("file", _data(corpus, "text", 3_000_000), 1700000001, 0o644)
    t = tb.Tarball()
    t.contents = contents
    path = str(tmp_path / "a.tar.gz")
    t.write_tarball(path)
    back = tb.Tarball()
    back.open(path)
    assert back.contents["d/big.bin"].contents == big
    src = tmp_path / "src"
    (src / "in").mkdir(parents=True)
    (src / "in" / "big.bin").write_bytes(big)
    a = za.ZipArchive()
    a.add_dir(str(src / "in"))
    zpath = str(tmp_path / "a.zip")
    a.write_zip_archive(zpath)
    with zipfile.ZipFile(zpath) as zf:
        assert zf.read(zf.namelist()[-1]) == big
    r = za.ZipArchive()
    r.open(zpath)
    assert [e.contents for e in r.contents.values() if e.kind == "file"] == [big]


def test_member_of_more_than_4_gib(z, monkeypatch):
    """One Default member whose output is 4 GiB + 1 MiB: beyond the serial path's 32-bit positions."""
    n = (4 << 30) + (1 << 20)
    rng = np.random.default_rng(4)
    words = rng.integers(0, 256, (4096, 64), dtype=np.uint8)
    pick = rng.integers(0, 4096, n // 64 + 1)
    raw = words[pick].reshape(-1)[:n]
    ctx = z.Context()
    c = ctx.compress_batch(raw, np.array([0, n], dtype=np.uint64), z.DefaultCompression, z.dfZlib)
    blob = c[0][:int(c[1][1])]
    out, do, lens, st = ctx.uncompress_batch(blob, np.array([0, len(blob)], dtype=np.uint64), z.dfZlib,
                                             sizes=np.array([n], dtype=np.uint64))
    assert int(st[0]) == 0 and int(lens[0]) == n
    assert np.array_equal(out[int(do[0]):int(do[0]) + n], raw)
    ctx.close()
