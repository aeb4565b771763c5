"""CPU checks of the stream builders and the launch-count model of tests/segment_streams.py, which the GPU tests
in test_gpu_segment_shapes.py rely on: joints exactly where intended, the intended segment sizes, segments that
really refer back across their joint, hand-built streams that zlib and the oracle decode to their replay, and a
model that reproduces the launch counts test_gpu_joint_segments.py pins."""
import zlib

import numpy as np
import pytest

from tests import deflate_writer as dw
from tests import segment_streams as ss
from tests import test_gpu_segment_shapes as g
from tests import util


@pytest.fixture(scope="module")
def T(corpus):
    return util.text_corpus(corpus)


@pytest.fixture(scope="module")
def o():
    from oracle import oracle
    return oracle


def _pieces(m):
    return [m.blob[a:b] for a, b in zip(m.bounds, m.bounds[1:])]


def check_foreign(m, cuts):
    """zlib flushed exactly at `cuts`: one joint per flush, segment sizes are the intervals, and a segment that
    refers back fails alone with zlib's 'invalid distance too far back'."""
    assert len(m.joints) == len(cuts) and not m.false
    assert [s.n for s in m.segs] == list(np.diff([0] + cuts + [len(m.raw)]))
    for i, (s, piece) in enumerate(zip(m.segs, _pieces(m))):
        assert ss.refers_back(piece) == (s.back is not None), i
        assert i > 0 or s.back is None


@pytest.mark.parametrize("f", range(3))
@pytest.mark.parametrize("i", range(len(ss.INTERVALS)))
def test_foreign_builders(T, i, f):
    name, m, cuts = ss.foreign_case(T, i, f)
    check_foreign(m, cuts)
    assert zlib.decompress(m.blob, ss.WBITS[m.fmt]) == m.raw
    assert not m.dense
    assert sum(s.back is not None for s in m.segs) >= len(m.segs) // 2, name   # most segments refer back


def test_foreign_random_many_and_dense_builders(T):
    for s in range(3):
        name, m, cuts = ss.random_case(T, s)
        check_foreign(m, cuts)
        assert min(np.diff(cuts)) >= 1 and max(np.diff(cuts)) <= 150000
    m, cuts = ss.many_segments_case(T)
    check_foreign(m, cuts)
    assert len(ss.join([s.n for s in m.segs])) > 8192 * 2
    for name, m, cuts in ss.dense_cases(T):
        check_foreign(m, cuts)
        assert m.dense, name
    m, cuts = ss.late_failure_member(T, 40000)
    check_foreign(m, cuts)


def check_hand_built(o, m, segments, tail=None):
    """Joints behind every segment (and before a final empty fixed block), nothing else; sizes as built; zlib
    and the oracle give the replay."""
    want = [ss.seg_len(s) for s in segments] + ([0] if tail == "fixed" else [])
    assert [s.n for s in m.segs] == want
    assert len(m.joints) == len(want) - 1 + (1 if tail == "stored" else 0) + m.false
    assert zlib.decompress(m.blob, ss.WBITS[m.fmt]) == m.raw
    assert o.uncompress(m.blob, m.fmt) == m.raw
    for i, s in enumerate(m.segs):
        if s.back is not None:   # (segments split by a false joint are not decodable alone)
            assert ss.refers_back(m.blob[m.bounds[i]:m.bounds[i + 1]]) or m.false


@pytest.mark.parametrize("n,window,big", g.WINDOW_CASES)
def test_window_builders_and_shapes(o, n, window, big):
    segs = ss.edge_segments(n, seed=n, big=big)
    m = ss.joint_member(segs, ss.RAW)
    check_hand_built(o, m, segs)
    assert all(s.back == 0 for s in m.segs[1:]) and not m.dense
    p = ss.plan(m, window=window or 8192)
    assert p.path == "joint" and sum(p.windows) == n + 1
    if big:
        assert any(s.n > 2 * (ss.WIN + ss.CHUNK) - ss.WIN for s in m.segs)


def test_windows_cover_every_shape():
    """Windows of 1, 2, 3, 4, 5, 9, 10, 16 and 17 segments (squares, one either side, partial last groups), a
    window of a budget-sized segment alone, windows that end on the budget, and first segments under 32 KiB."""
    seen, alone, budget = set(), False, False
    for n, window, big in g.WINDOW_CASES:
        m = ss.joint_member(ss.edge_segments(n, seed=n, big=big), ss.RAW)
        w = window or 8192
        p = ss.plan(m, window=w)
        seen |= set(p.windows)
        a = 0
        for k in p.windows:
            alone = alone or (k == 1 and m.segs[a].n + ss.WIN > w * (ss.WIN + ss.CHUNK))
            budget = budget or (k < w and a + k < len(m.segs))
            a += k
    assert {1, 2, 3, 4, 5, 9, 10, 16, 17} <= seen and alone and budget, seen
    assert ss.group_shape(17) == (5, 4) and ss.group_shape(16) == (4, 4) and ss.group_shape(10) == (4, 3)


def test_chain_and_dense_builders(o):
    for dist in (1, 32768, None):
        segs = ss.chain_segments(600, dist, seed=3)
        m = ss.joint_member(segs, ss.ZLIB)
        check_hand_built(o, m, segs)
        assert ss.plan(m).path == "joint" and not m.dense
    segs = ss.chain_segments(3000, 32768, seed=4)
    m = ss.joint_member(segs, ss.RAW, pad=0)
    check_hand_built(o, m, segs)
    assert m.dense and ss.plan(m).path == "fallback"


@pytest.mark.parametrize("case", sorted(g.ZERO_CASES))
def test_zero_output_builders(o, case):
    segs, tail = g.ZERO_CASES[case]
    m = ss.joint_member(segs, ss.RAW, tail=tail)
    check_hand_built(o, m, segs, tail)
    assert any(s.n == 0 for s in m.segs) or tail == "stored"
    if case == "back_to_back":
        assert m.blob.count(ss.MARK + b"\x00" + ss.MARK) == 2
    if tail == "stored":
        assert m.joints[-1] == m.end
    assert ss.plan(m).path == "joint"


@pytest.mark.parametrize("tiny", [0, 40])
@pytest.mark.parametrize("start", [32767, 32768])
def test_start_rule_builders(o, start, tiny):
    segs = ss.start_rule_segments(start, start, tiny)
    m = ss.joint_member(segs, ss.RAW)
    check_hand_built(o, m, segs)
    first = 1 + tiny
    assert sum(s.n for s in m.segs[:first]) == start and m.segs[first].back == 0
    if start + 1 <= ss.WIN:
        blob = dw.raw(ss.joint_blocks(ss.start_rule_segments(start, start + 1, tiny)))
        with pytest.raises(zlib.error, match="invalid distance too far back"):
            zlib.decompress(blob, -15)
        assert g.verdict(o, blob, ss.RAW) == 3


def test_late_failure_and_false_joint_plans(T, o):
    for odd in (40000, 100000):
        m, _ = ss.late_failure_member(T, odd)
        assert m.segs[6].n == odd and m.segs[6].back < ss.CHUNK
        p = ss.plan(m, window=3)
        assert p.guess_failed == 2 and p.counts == 1
    m = g.false_joint_member()
    assert m.false == 1 and len(m.joints) == 61
    assert zlib.decompress(m.blob, -15) == m.raw and o.uncompress(m.blob, ss.RAW) == m.raw
    assert ss.plan(m).counts == 3


def test_speculative_members_have_no_joints(T):
    for seed in range(2):
        blob, d = g.speculative_member(T, seed)
        assert ss.MARK not in blob and zlib.decompress(blob) == d


def test_plan_reproduces_the_joint_segment_tests():
    """The launch counts test_gpu_joint_segments.py pins, from segment lists of the same shape."""
    def own(n, backs=True):
        segs = [ss.Seg(min(ss.CHUNK, n - k), (0 if backs and k else None)) for k in range(0, n, ss.CHUNK)]
        m = ss.Member(b"", ss.GZIP, b"", 0, 10 ** 9, [1] * (len(segs) - 1), segs=segs)
        m.bounds = [0] * (len(segs) + 1)
        return m
    m = own(3_012_345)
    assert ss.plan(m).launches == 5 + 6
    m = own(5_000_999)
    assert ss.plan(m, window=7).launches == 5 + 6 * 11
    # level 1 (independent chunks): the optimistic pass is all it takes
    assert ss.plan(own(3_012_345, backs=False)) == ss.Plan("independent", 5)
    # stored chunks carry no joint after them: a 128 KiB segment makes the guess wrong, one count pass
    m = own(1_000_000)
    m.segs[3:5] = [ss.Seg(2 * ss.CHUNK, ss.CHUNK + 5)]   # random bytes first: the first reference is past 64 KiB
    m.bounds, m.joints = m.bounds[:-1], m.joints[:-1]
    assert ss.plan(m).launches == 5 + 1 + 6
    # the speculative fallback with the joint decode off
    assert ss.plan(own(1_000_000), joints=False).path == "fallback"
