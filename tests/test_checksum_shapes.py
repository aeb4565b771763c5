"""CPU checks of tests/checksum_shapes.py: the geometry parsed from the sources is the one the shape classes are
written for, and the size sweep of tests/test_gpu_checksum_shapes.py reaches every path of the checksum kernels."""
import zlib

import pytest

from tests import checksum_shapes as cs


def test_parsed_constants_are_the_assumed_geometry():
    # a change to any of these changes which sizes reach which path: review the classes, then update this test
    assert cs.PIECE == 32768
    assert cs.BIG_PIECES == 2048
    assert (cs.CK_THREADS, cs.CK_THREADS_ADLER, cs.CKB_THREADS) == (512, 256, 1024)
    assert cs.CHUNK == 65536
    assert cs.ADLER_MOD == 65521
    assert cs.share_bytes(False) == 2048 and cs.share_bytes(True) == 4096
    assert cs.CHUNK % cs.PIECE == 0


@pytest.mark.parametrize("kind,adler_only", [("crc32", False), ("adler32", False), ("adler32", True)])
def test_sweep_hits_every_shape_class(kind, adler_only):
    hit = set()
    for n in cs.SWEEP + cs.HUGE:
        hit |= cs.shape_classes(n, kind, adler_only)
    missing = cs.required_shape_classes(kind, adler_only) - hit
    assert not missing, missing


def test_shape_classes_examples():
    assert cs.shape_classes(0, "crc32") == {"empty"}
    assert "short" in cs.shape_classes(3, "crc32")
    assert "exactly_chunk" in cs.shape_classes(65536, "crc32")
    assert "ragged_share_multiple" in cs.shape_classes(2048 * 17, "crc32")
    assert "ragged_share_multiple" not in cs.shape_classes(2048 * 17, "adler32", adler_only=True)
    assert "ragged_share_multiple" in cs.shape_classes(2048 * 18, "adler32", adler_only=True)
    assert "lane_ge32_ragged" in cs.shape_classes(32 * 32768 + 1, "crc32")
    assert "exactly_big_pieces" in cs.shape_classes(2048 * 32768, "crc32")
    assert "big_fold" in cs.shape_classes(2048 * 32768 + 1, "crc32")
    assert "big_fold_ragged_ge_threads" in cs.shape_classes(3072 * 32768 - 1, "crc32")
    assert "mod_p_m1" in cs.shape_classes(17 * 65521 - 1, "adler32")


def test_sweep_contains_the_listed_sizes():
    s = set(cs.SWEEP)
    want = set(range(9)) | {127, 128, 129, 2047, 2048, 2049, 4095, 4096, 4097, 32767, 32768, 32769,
                            65535, 65536, 65537, 131072, (1 << 20) - 1, (1 << 20) + 1}
    want |= {2048 * j for j in range(17, 32)}
    want |= {32768 * k + d for k in (2, 15, 16, 31, 32, 33, 63, 64, 65) for d in (0, 1, 3, 2048, 6144)}
    want |= {2048 * 32768 + d for d in (-1, 0, 1)} | {3072 * 32768 + d for d in (-1, 1)}
    assert want <= s, sorted(want - s)


def test_member_sweep_hits_every_member_class():
    hit = set()
    for n in cs.MEMBER_SWEEP:
        hit |= cs.member_classes(n)
    assert not cs.REQUIRED_MEMBER_CLASSES - hit, cs.REQUIRED_MEMBER_CLASSES - hit
    assert "ge_4GiB" in cs.member_classes(cs.HUGE_MEMBER)
    # the carry-in of a compress stream's launches: the running totals of the write cuts
    carry, tot = set(), 0
    for w in cs.STREAM_CUTS:
        carry |= cs.member_classes(tot)
        tot += w
    assert {"exactly_chunk", "whole_chunks", "ragged_last_chunk", "chunks_2_32", "chunks_33_63"} <= carry


def test_member_classes_examples():
    assert cs.member_classes(65536 * 33) >= {"chunks_33_63", "whole_chunks"}
    assert "chunks_multiple_of_32" in cs.member_classes(65536 * 64)
    assert "chunks_gt_1024" in cs.member_classes(1025 * 65536 + 3)
    assert cs.member_classes(131072) >= {"exactly_two_chunks", "chunks_2_32"}


@pytest.mark.parametrize("base_shift", range(16))
def test_placement_gives_every_full_piece_misalignment(base_shift):
    lengths = [n for n in cs.SMALL_SWEEP if n >= cs.PIECE]
    mis = [i % 16 for i in range(len(lengths))]
    offs, which = cs.place(lengths, mis, base_shift)
    for n, j, m in zip(lengths, which, mis):
        assert (base_shift + int(offs[j])) % 16 == m and int(offs[j + 1] - offs[j]) == n
    assert cs.full_piece_misalignments(lengths, mis, base_shift) == set(range(16))


@pytest.mark.parametrize("base_shift", range(16))
def test_device_layout_gives_every_full_piece_misalignment(base_shift):
    """the layout the checksum_batch_device sweep uses, at each of its base shifts"""
    lengths, mis, offs, which = cs.device_layout()
    for n, j, m in zip(lengths, which, mis):
        assert int(offs[j]) % 16 == m and int(offs[j + 1] - offs[j]) == n
    seen = {(base_shift + int(offs[j]) + k * cs.PIECE) % 16 for n, j in zip(lengths, which) for k in range(n // cs.PIECE)}
    assert seen == set(range(16))


def test_pipeline_batch_stays_below_the_big_member_threshold(corpus):
    """Host decodes of this batch go through the host pipeline only while every member is shorter than
    big_member_bytes (zb_api.cu); its outputs still span many pieces."""
    from tests import util
    items = cs.pipeline_members(util.text_corpus(corpus))
    assert cs.BIG_MEMBER_BYTES == 512 << 10
    assert max(len(x[1]) for x in items) < cs.BIG_MEMBER_BYTES
    assert max(x[3] for x in items) > cs.COMBINE_LANES * cs.PIECE
    hit = set()
    for n in cs.PIPE_SWEEP:
        hit |= cs.shape_classes(n, "crc32")
    assert {"ragged_share_multiple", "exactly_chunk", "exactly_two_chunks", "lane_ge32_ragged", "empty"} <= hit
    for name, m, out, n in items:
        if out is not None:
            assert zlib.decompress(m, 31 if name.startswith("gzip") else 15) == out


def test_content_generators():
    assert cs.content("random", 1000, seed=3).tobytes() == cs.content("random", 1000, seed=3).tobytes()
    assert cs.content("ff", 5).tobytes() == b"\xff" * 5 and cs.content("zeros", 3).tobytes() == b"\0" * 3
    assert cs.content("text", 7, text=b"abc").tobytes() == b"abcabca"
    # the largest Adler sums: all-0xff buffers reach the modular reduction in every piece
    assert zlib.adler32(cs.content("ff", 5552 + 1).tobytes()) != 1
