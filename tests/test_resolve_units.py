"""CPU-only tests of the parallel window resolve's per-element rules (zippy_b200/csrc/zb_resolve.h).

tests/native/resolve_units.cpp runs the three steps of the GPU resolve (group walk, group composition, parallel
tails + the rest) on the CPU with the header's functions; every case must give the bytes and the bad flag of a
plain sequential resolve."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "resolve_units.cpp")
HDR = os.path.join(HERE, "..", "zippy_b200", "csrc", "zb_resolve.h")
WIN = 32768


@pytest.fixture(scope="module")
def ru(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("resolve_units") / "libresolve_units.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, SRC])
    L = ctypes.CDLL(so)
    u16, u32, u8 = (np.ctypeslib.ndpointer(t, flags="C_CONTIGUOUS") for t in (np.uint16, np.uint32, np.uint8))
    L.t_resolve_seq.argtypes = [u16, u32, ctypes.c_uint32, ctypes.c_uint64, u8, u8]
    L.t_resolve_groups.argtypes = [u16, u32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64, u8, u8]
    return L


def _check(ru, sym, sizes, w0, prev, gszs=(1, 2, 3, 7, 64)):
    n = np.asarray(sizes, dtype=np.uint32)
    sym = np.ascontiguousarray(sym, dtype=np.uint16)
    assert len(sym) == int(n.sum())
    want = np.zeros(len(sym), dtype=np.uint8)
    bad = ru.t_resolve_seq(sym, n, len(n), w0, prev, want)
    for g in gszs:
        got = np.zeros(len(sym), dtype=np.uint8)
        assert ru.t_resolve_groups(sym, n, len(n), g, w0, prev, got) == bad, g
        assert np.array_equal(got, want), g
    return bad, want


def _random_case(rng, sizes, p_marker):
    total = int(sum(sizes))
    sym = rng.integers(0, 256, total).astype(np.uint16)
    m = rng.random(total) < p_marker
    sym[m] = 0x8000 | rng.integers(0, WIN, int(m.sum()))
    return sym


def test_random_marker_arrays(ru):
    rng = np.random.default_rng(1)
    for t in range(12):
        sizes = rng.integers(40000, 70000, rng.integers(2, 20))
        w0 = int(rng.integers(WIN, 1 << 40)) if t % 2 else WIN + int(rng.integers(0, 5))
        prev = rng.integers(0, 256, WIN).astype(np.uint8)
        bad, _ = _check(ru, _random_case(rng, sizes, [0.01, 0.3, 0.9][t % 3]), sizes, w0, prev)
        assert bad == 0


def test_chains_through_every_segment(ru):
    """Every symbol after the window's first bytes is a marker to the byte 32768 back (a zero run, or a copy at
    the maximum distance): each segment's bytes come from the one before, through all of them."""
    rng = np.random.default_rng(2)
    prev = rng.integers(0, 256, WIN).astype(np.uint8)
    for sizes in ([65536] * 17, [32768] * 9 + [100], [70001, 32767, 40000, 1, 65536, 65536]):
        total = sum(sizes)
        sym = np.empty(total, dtype=np.uint16)
        o = 0
        for n in sizes:   # marker k of every segment: position p0 - 32768 + k, i.e. 32768 bytes back
            j = np.arange(n)
            sym[o:o + n] = np.where(j < WIN, 0x8000 | (j % WIN), 0x8000)   # beyond 32768: distance-1 runs of marker 0 too
            o += n
        bad, out = _check(ru, sym, sizes, 5 * WIN, prev)
        assert bad == 0
        assert np.array_equal(out[:WIN], prev[:min(WIN, total)])   # the first 32 KiB are the incoming window


def test_segments_shorter_than_the_window(ru):
    rng = np.random.default_rng(3)
    for t in range(10):
        sizes = rng.integers(1, 9000, rng.integers(5, 60))
        prev = rng.integers(0, 256, WIN).astype(np.uint8)
        bad, _ = _check(ru, _random_case(rng, sizes, 0.5), sizes, 3 * WIN + t, prev)
        assert bad == 0
    sizes = [1] * 200   # single-byte segments: every group map is mostly the incoming window, shifted
    _check(ru, _random_case(rng, sizes, 1.0), sizes, WIN, rng.integers(0, 256, WIN).astype(np.uint8))


def test_markers_before_the_stream_start(ru):
    rng = np.random.default_rng(4)
    zeros = np.zeros(WIN, dtype=np.uint8)
    # the member's first window: a marker in the first 32 KiB of output can reach before position 0
    sizes = [70000, 20000, 65536]
    sym = _random_case(rng, sizes, 0.0)
    sym[100] = 0x8000 | 50                          # position 100 - 32768 + 50 < 0
    assert _check(ru, sym, sizes, 0, zeros)[0] == 1
    sym = _random_case(rng, sizes, 0.0)
    sym[69990] = 0x8000 | 3                         # in the first segment's tail: found by the group walk
    assert _check(ru, sym, sizes, 0, zeros)[0] == 1
    sym = _random_case(rng, sizes, 0.0)
    sym[70000 + 5] = 0x8000 | 100                   # second segment, position 70005 - 32768 + 100 >= 0: fine
    assert _check(ru, sym, sizes, 0, zeros)[0] == 0
    # a window that starts less than 32 KiB into the member
    sizes = [5000] * 10
    sym = _random_case(rng, sizes, 0.0)
    sym[2] = 0x8000 | 10
    assert _check(ru, sym, sizes, 1000, zeros)[0] == 1
    sym[2] = 0x8000 | (WIN - 1000 + 1)             # position 1000 + 2 - 32768 + 31769 = 3: inside the member
    assert _check(ru, sym, sizes, 1000, zeros)[0] == 0
