"""The parallel joint decode (zb_api.cu: inflate_member_joints; zb_inflate.cu: k_resolve_groups, k_resolve_compose,
k_resolve_tails_par, k_resolve_rest) on segment shapes this library's own members never have: foreign zlib
streams sync-flushed every 100 bytes to every 200 000, hand-built members with segments of a few hundred bytes,
zero-output segments, segments that start at output byte 32767 or 32768, windows of 1..17 segments with
partial groups, segments larger than a window's element budget, and a 64 KiB guess that fails in a later window.

Every valid member must come out bit-exact, with the exact launch count the host code reports for its path
(tests/segment_streams.py: plan), and with the same bytes when the joint decode is off and when the serial
decode takes the member.  Every invalid member must get the oracle's exact status."""
import zlib

import numpy as np
import pytest

from tests import deflate_writer as dw
from tests import segment_streams as ss
from tests import util

pytestmark = pytest.mark.gpu

BIG = 100            # every member of 100 bytes or more takes the large-member paths
SERIAL = 1 << 50     # no member does: the ordinary launch decodes it serially


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


@pytest.fixture(scope="module")
def o():
    from oracle import oracle
    return oracle


@pytest.fixture(scope="module")
def T(corpus):
    return util.text_corpus(corpus)


@pytest.fixture(scope="module")
def ctxs(z):
    """Contexts by (window, joints, big, gated), created with the hooks set as test_gpu_joint_segments._ctx does."""
    made = {}

    def get(window=None, joints=True, big=BIG, gated=None):
        key = (window, joints, big, gated)
        if key not in made:
            with pytest.MonkeyPatch.context() as mp:
                mp.setenv("ZB200_BIG_MEMBER_BYTES", str(big))
                if window:
                    mp.setenv("ZB200_MARK_WINDOW_SEGS", str(window))
                if not joints:
                    mp.setenv("ZB200_JOINT_MARKERS", "0")
                if gated is not None:
                    mp.setenv("ZB200_UNC_GATED", gated)
                made[key] = z.Context()
        return made[key]
    yield get
    for c in made.values():
        c.close()


def _one(ctx, blob, fmt, sizes=None):
    base = np.frombuffer(blob, dtype=np.uint8)
    offs = np.array([0, len(blob)], dtype=np.uint64)
    out, do, lens, st = ctx.uncompress_batch(base, offs, fmt, sizes=sizes)
    got = out[int(do[0]):int(do[0]) + int(lens[0])].tobytes() if st[0] == 0 else None
    return got, int(st[0]), ctx.timing()["kernel_launches"]


def verdict(o, blob, fmt):
    try:
        return o.uncompress(blob, fmt)
    except o.ZippyError as e:
        return e.code


def check_valid(ctxs, m, window=None, path="joint", name=""):
    """The joint decode's bytes and launch count, then the same bytes with the joint decode off and from the
    serial decode.  -> the plan."""
    p = ss.plan(m, window=window or 8192)
    assert p.path == path, (name, p)
    got, st, launches = _one(ctxs(window), m.blob, m.fmt)
    assert st == 0 and got == m.raw, (name, st)
    assert launches == p.launches, (name, launches, p)
    for ctx in (ctxs(window, joints=False), ctxs(big=SERIAL)):
        g2, s2, _ = _one(ctx, m.blob, m.fmt)
        assert s2 == 0 and g2 == m.raw, (name, s2)
    return p


def check_invalid(ctxs, o, blob, fmt, window=None, name=""):
    """Status (and bytes, when the oracle accepts the stream) equal to the oracle's, on all three paths."""
    want = verdict(o, blob, fmt)
    for ctx in (ctxs(window), ctxs(window, joints=False), ctxs(big=SERIAL)):
        got, st, _ = _one(ctx, blob, fmt)
        if isinstance(want, int):
            assert st == want, (name, st, want)
        else:
            assert st == 0 and got == want, (name, st)


# ---------------------------------------------------------------------------------------------- 1. foreign
@pytest.mark.parametrize("f", range(3))
@pytest.mark.parametrize("i", range(len(ss.INTERVALS)))
def test_foreign_sync_flushed_members(ctxs, T, i, f):
    name, m, _ = ss.foreign_case(T, i, f)
    p = check_valid(ctxs, m, name=name)
    if ss.INTERVALS[i] == ss.CHUNK:     # this library's shape: the guess holds and no count pass runs
        assert p.counts == 0 and p.launches == ss.BASE + ss.OPTIMISTIC + 6, p


@pytest.mark.parametrize("seed", range(3))
def test_foreign_random_intervals(ctxs, T, seed):
    name, m, _ = ss.random_case(T, seed)
    check_valid(ctxs, m, name=name)


def test_more_than_8192_segments(ctxs, T):
    m, _ = ss.many_segments_case(T)
    p = check_valid(ctxs, m)
    assert len(m.segs) > 16384 and p.windows[0] == 8192 and len(p.windows) == 3, p.windows


def test_dense_joints_fall_back(ctxs, T):
    """Above the density cap the joints are not taken: the same launches as with the joint decode off, and
    those of the speculative segments."""
    for name, m, _ in ss.dense_cases(T):
        assert ss.plan(m).path == "fallback" and m.dense
        got, st, launches = _one(ctxs(), m.blob, m.fmt)
        assert st == 0 and got == m.raw, name
        g2, s2, l2 = _one(ctxs(joints=False), m.blob, m.fmt)
        assert s2 == 0 and g2 == m.raw and l2 == launches, (name, launches, l2)
        assert launches - ss.BASE in ss.SPECULATIVE, (name, launches)


# ---------------------------------------------------------------------------------------------- 2./3. hand-built
WINDOW_CASES = [   # (segments after segment 0, window, big segment indices)
    (3, None, ()), (4, None, ()), (8, None, ()), (9, None, ()), (15, None, ()), (16, None, ()),
    (4, 1, ()), (6, 2, ()), (9, 3, ()), (16, 7, ()), (40, 8192, ()),
    (6, 2, (2, 4)), (6, 3, (2, 5)), (5, None, (1, 3)),
]


@pytest.mark.parametrize("n,window,big", WINDOW_CASES)
def test_windows_and_groups(ctxs, n, window, big):
    """Copies from the first and the last byte of every group's incoming window and across every segment start;
    windows of 1..17 segments; a 200 000-byte segment alone in its window."""
    for fmt in (ss.RAW, ss.GZIP):
        m = ss.joint_member(ss.edge_segments(n, seed=n, big=big), fmt)
        p = check_valid(ctxs, m, window, name=(n, window, big))
        assert sum(p.windows) == n + 1


@pytest.mark.parametrize("dist", [1, 32768, None])
@pytest.mark.parametrize("window", [None, 7])
def test_chains_through_every_segment(ctxs, dist, window):
    """One literal or 40 000 random bytes, then 600 segments of one 258-byte match each: every byte resolves
    through every segment, group and window before it."""
    m = ss.joint_member(ss.chain_segments(600, dist, seed=3), ss.ZLIB)
    check_valid(ctxs, m, window, name=dist)


def test_joints_below_the_density_cap_fall_back(ctxs):
    m = ss.joint_member(ss.chain_segments(3000, 32768, seed=4), ss.RAW, pad=0)
    assert m.dense and ss.plan(m).path == "fallback"
    got, st, launches = _one(ctxs(), m.blob, m.fmt)
    assert st == 0 and got == m.raw
    g2, s2, l2 = _one(ctxs(joints=False), m.blob, m.fmt)
    assert s2 == 0 and g2 == m.raw and l2 == launches


ZERO_CASES = {
    "first": ([[]] + ss.edge_segments(5, 1)[0:1] + [ss.edge_tokens(k) for k in range(4)], None),
    "middle": (ss.edge_segments(3, 2) + [[], ss.edge_tokens(9), []] + [ss.edge_tokens(k) for k in range(3)], None),
    "back_to_back": (ss.edge_segments(3, 3) + [None, None, ss.edge_tokens(5), None] + [ss.edge_tokens(7)], None),
    "last_empty_fixed": (ss.edge_segments(6, 4), "fixed"),
    "last_empty_stored": (ss.edge_segments(6, 5), "stored"),
    "last_empty_segment": (ss.edge_segments(6, 6) + [[]], None),
}


@pytest.mark.parametrize("case", sorted(ZERO_CASES))
def test_zero_output_segments(ctxs, case):
    segs, tail = ZERO_CASES[case]
    for fmt in (ss.RAW, ss.ZLIB):
        m = ss.joint_member(segs, fmt, tail=tail)
        assert any(s.n == 0 for s in m.segs) or tail == "stored"   # (stored: the payload ends on a joint)
        for window in (None, 2):
            check_valid(ctxs, m, window, name=case)


# ---------------------------------------------------------------------------------------------- 4. 32 KiB start rule
@pytest.mark.parametrize("tiny", [0, 40])
@pytest.mark.parametrize("start", [32767, 32768])
def test_32k_start_rule(ctxs, o, start, tiny):
    """A segment starting at output byte 32767 or 32768 whose first match reaches exactly byte 0 (valid) or
    byte -1 (invalid; a distance of 32769 does not exist, so only after 32767 bytes)."""
    m = ss.joint_member(ss.start_rule_segments(start, start, tiny), ss.RAW)
    for window in (None, 1):
        check_valid(ctxs, m, window, name=(start, tiny))
    if start + 1 <= ss.WIN:
        blocks = ss.joint_blocks(ss.start_rule_segments(start, start + 1, tiny))
        blob = dw.raw(blocks)
        assert isinstance(verdict(o, blob, ss.RAW), int)
        for fmt in (ss.RAW, ss.GZIP):
            check_invalid(ctxs, o, ss.wrap(blob, b"", fmt), fmt, name=(start, tiny, fmt))


# ---------------------------------------------------------------------------------------------- 5. late guess failure
@pytest.mark.parametrize("odd", [40000, 100000])
def test_guess_fails_in_a_later_window(ctxs, T, odd):
    m, _ = ss.late_failure_member(T, odd)
    p = check_valid(ctxs, m, 3)
    # two windows under the guess, the third fails, one count pass, then the rest with counted sizes
    assert p.guess_failed == 2 and p.counts == 1, p
    assert p.launches == ss.BASE + ss.OPTIMISTIC + 2 * 6 + 2 + 1 + 6 * (len(p.windows) - 2), p


def false_joint_member(fmt=ss.RAW):
    """A 5000-byte stored segment with 00 00 ff ff planted in its data, then 60 short segments: the count drops
    the false joint, then joins the segments that start before output byte 32768."""
    rng = np.random.default_rng(12)
    rnd = bytearray(rng.integers(0, 256, 5000, dtype=np.uint8).tobytes())
    rnd[2000:2004] = ss.MARK
    segs = [[dw.Stored(bytes(rnd), final=False)]] + [ss.edge_tokens(k) for k in range(60)]
    segs[1] = [0x41] * 300 + [(258, 300)] * 120         # (32768 bytes before the first edge_tokens)
    blocks = ss.joint_blocks(segs)
    raw = dw.replay(blocks)
    blob = ss.wrap(dw.raw(blocks), raw, fmt)
    at = blob.find(bytes(rnd[:64])) + 2004
    return ss.analyse(blob, fmt, raw, [at])


def test_false_joint_repair_and_join_in_one_count(ctxs):
    for fmt in (ss.RAW, ss.GZIP):
        m = false_joint_member(fmt)
        p = check_valid(ctxs, m)
        assert p.counts == 3, p


# ---------------------------------------------------------------------------------------------- 6. sizes and single calls
def _single_members(T):
    out = [ss.foreign_case(T, 1, 0)[1], ss.foreign_case(T, 4, 1)[1], ss.random_case(T, 1)[1]]
    out.append(ss.joint_member(ss.edge_segments(12, 8), ss.RAW))
    out.append(ss.joint_member(ss.chain_segments(300, 1, 9), ss.ZLIB))
    return out


def test_sizes_capacity_and_single_calls(ctxs, T):
    on, serial = ctxs(), ctxs(big=SERIAL)
    for k, m in enumerate(_single_members(T)):
        n = len(m.raw)
        if m.fmt != ss.GZIP:   # (gzip sizes come from ISIZE)
            sz, st = on.uncompressed_sizes(np.frombuffer(m.blob, dtype=np.uint8), np.array([0, len(m.blob)], dtype=np.uint64), m.fmt)
            assert int(st[0]) == 0 and int(sz[0]) == n, (k, sz, st)
        got, st, launches = _one(on, m.blob, m.fmt, sizes=np.array([n], dtype=np.uint64))
        assert st == 0 and got == m.raw and launches == ss.plan(m).launches, (k, st, launches)
        # one byte short: the joint decode reports the slot too small, the member is decoded again alone
        short = np.array([n - 1], dtype=np.uint64)
        assert ss.plan(m, mcap=n - 1).path == "too_small"
        assert _one(on, m.blob, m.fmt, sizes=short)[:2] == _one(serial, m.blob, m.fmt, sizes=short)[:2], k
        assert on.decode_one(m.blob, m.fmt) == m.raw, k
        if m.fmt == ss.RAW:
            assert on.inflate(m.blob) == m.raw, k


# ---------------------------------------------------------------------------------------------- 7. corruption
def _flip_positions(m, rng, count):
    pos = [int(p) for p in rng.integers(m.pos, m.end, count)]
    for j in m.joints[1:len(m.joints):max(1, len(m.joints) // 6)]:
        pos += [j - 4, j - 3, j - 2, j - 1, j]          # the joint's bytes and the first block header after it
    return pos


@pytest.mark.parametrize("kind", ["short_segments", "multi_window"])
def test_corrupt_and_truncated_members(ctxs, o, T, kind):
    rng = np.random.default_rng(17)
    if kind == "short_segments":
        m, window = ss.foreign_case(T, 1, 0)[1], None           # raw: no trailer check can catch a bad resolve
    else:
        m, window = ss.joint_member(ss.edge_segments(40, 10), ss.GZIP), 7
    for k, p in enumerate(_flip_positions(m, rng, 20)):
        bad = bytearray(m.blob)
        bad[p] ^= 1 << int(rng.integers(0, 8))
        check_invalid(ctxs, o, bytes(bad), m.fmt, window, name=(kind, k, p))
    for j in m.joints[2:len(m.joints):max(1, len(m.joints) // 3)]:
        for cut in (j - 1, j, j + 1):
            check_invalid(ctxs, o, m.blob[:cut], m.fmt, window, name=(kind, "cut", cut))


# ---------------------------------------------------------------------------------------------- 8. batches
def _batch(z, o, T, ctx):
    ms = [ss.foreign_case(T, 1, 2)[1], ss.foreign_case(T, 3, 1)[1], ss.random_case(T, 2)[1],
          ss.joint_member(ss.edge_segments(20, 11), ss.GZIP)]
    items = [(m.blob, m.raw) for m in ms]
    for r in (T[:5000], b"", T[100:180]):
        items.append((o.compress(r, 6, o.dfZlib), r))
    own = T[:900000]
    c = ctx.compress_batch(np.frombuffer(own, dtype=np.uint8), np.array([0, len(own)], dtype=np.uint64),
                           z.DefaultCompression, z.dfGzip)
    items.append((c[0][:int(c[1][1])].tobytes(), own))
    order = [4, 0, 5, 1, 7, 2, 6, 3]
    return [items[i] for i in order]


@pytest.mark.parametrize("gated", ["1", "0"])
def test_batch_next_to_small_and_own_members(z, o, ctxs, T, gated):
    ctx = ctxs(gated=gated)
    items = _batch(z, o, T, ctx)
    base = np.frombuffer(b"".join(b for b, _ in items), dtype=np.uint8)
    offs = np.zeros(len(items) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(b) for b, _ in items])
    out, do, lens, st = ctx.uncompress_batch(base, offs, z.dfDetect)
    for i, (_, want) in enumerate(items):
        assert int(st[i]) == 0 and out[int(do[i]):int(do[i]) + int(lens[i])].tobytes() == want, (gated, i, int(st[i]))


def test_device_batch_from_a_misaligned_source(z, o, ctxs, T):
    torch = pytest.importorskip("torch")
    ctx = ctxs()
    items = _batch(z, o, T, ctx)
    blob = b"".join(b for b, _ in items)
    offs = np.zeros(len(items) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(b) for b, _ in items])
    doffs = np.zeros(len(items) + 1, dtype=np.uint64)
    doffs[1:] = np.cumsum([len(w) for _, w in items])
    for shift in (1, 3):
        d_src = torch.zeros(len(blob) + 8, dtype=torch.uint8, device="cuda")
        d_src[shift:shift + len(blob)] = torch.from_numpy(np.frombuffer(blob, dtype=np.uint8).copy()).cuda()
        d_dst = torch.zeros(int(doffs[-1]) + 8, dtype=torch.uint8, device="cuda")
        lens, st = ctx.uncompress_batch_device(d_src.data_ptr() + shift, offs, z.dfDetect, d_dst.data_ptr(), doffs)
        host = d_dst.cpu().numpy()
        for i, (_, want) in enumerate(items):
            assert int(st[i]) == 0 and int(lens[i]) == len(want), (shift, i, int(st[i]))
            assert host[int(doffs[i]):int(doffs[i]) + len(want)].tobytes() == want, (shift, i)


def test_inflate_batch_crc32_on_sync_flushed_raw_members(ctxs, T):
    ctx = ctxs()
    ms = [ss.foreign_case(T, i, 0)[1] for i in (0, 2, 6)] + [ss.joint_member(ss.edge_segments(9, 13), ss.RAW)]
    base = np.frombuffer(b"".join(m.blob for m in ms), dtype=np.uint8)
    offs = np.zeros(len(ms) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(m.blob) for m in ms])
    out, do, lens, crcs, st = ctx.inflate_batch_crc32(base, offs, np.array([len(m.raw) for m in ms], dtype=np.uint64))
    for i, m in enumerate(ms):
        assert int(st[i]) == 0 and out[int(do[i]):int(do[i]) + int(lens[i])].tobytes() == m.raw, i
        assert int(crcs[i]) == zlib.crc32(m.raw), i


# ---------------------------------------------------------------------------------------------- 9. speculative
def speculative_member(T, seed):
    """A zlib stream at memLevel 1 (blocks of about 128 symbols) and no sync flush: the speculative segments,
    cut 2 KiB of input apart for a single member, are shorter than 32 KiB."""
    d = ss.data(T, ("text", "mix")[seed], 1_200_000, seed=80 + seed)
    c = zlib.compressobj(6, zlib.DEFLATED, 15, 1)
    return c.compress(d) + c.flush(), d


@pytest.mark.parametrize("seed", range(2))
def test_short_speculative_segments(ctxs, o, T, seed):
    blob, d = speculative_member(T, seed)
    got, st, launches = _one(ctxs(), blob, ss.ZLIB)
    # block search, count, prefill + marker decode, k_resolve_tails + k_resolve_rest
    assert st == 0 and got == d and launches == ss.BASE + 6, (st, launches)
    rng = np.random.default_rng(seed)
    for k in range(6):
        bad = bytearray(blob)
        p = int(rng.integers(2, len(bad) - 4))
        bad[p] ^= 1 << int(rng.integers(0, 8))
        want = verdict(o, bytes(bad), ss.ZLIB)
        g, s, _ = _one(ctxs(), bytes(bad), ss.ZLIB)
        assert (s == want) if isinstance(want, int) else (s == 0 and g == want), (k, p, s)
