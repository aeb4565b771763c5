"""The parse of a member compressed against its own dictionary under zlib's window size n (zb200_compress_batch_dicts,
levels -1 and 2..9): the windowed schedule model (tests/native/lz2_window_model.c) run on W || M with a chunk
boundary at |W|, no reset and the distance limit 2^n.  The CPU part checks that model on W || M by itself: the tokens
rebuild M from W, no distance exceeds 2^n, and some match reaches exactly 2^n back into W.  The GPU part
(tests/test_gpu_dictionaries.py) requires k_lz2's tokens to be the model's."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from tests import util
from tests.test_dictionary_rules import window
from tests.test_gpu_lz2_model import decode

NATIVE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "native")
CHUNK = 65536
WINDOW_BITS = [9, 12, 15]
LEVELS = [-1, 2, 6, 9]


class WindowedSchedule:
    """lz2_window_model under an explicit chunk schedule (bounds / hist_from, as lz2_model_schedule takes them)."""

    def __init__(self, so):
        self.L = ctypes.CDLL(so)
        P, U64, U32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
        self.f = self.L.lz2_window_model
        self.f.argtypes = [ctypes.c_char_p, U64, ctypes.c_int, ctypes.c_int, U32, P, P, U64, P, U64, P, P, P]
        self.f.restype = ctypes.c_int64

    def member(self, w, m, level, n):
        """-> (M's chunks' encoded tokens, matches at exactly 2^n): the parse of W || M with a boundary at |W|."""
        x = w + m
        bounds = [0, len(w)] + list(range(len(w) + CHUNK, len(x), CHUNK)) + [len(x)]
        if bounds[-1] == bounds[-2] and len(bounds) > 3:
            bounds.pop()
        nch = len(bounds) - 1
        b = np.array(bounds, dtype=np.uint64)
        h = np.zeros(nch, dtype=np.uint64)
        tok = np.zeros(len(x) + 16, dtype=np.uint32)
        per = np.zeros(nch, dtype=np.uint32)
        cnt = np.zeros(32, dtype=np.uint64)
        edge = ctypes.c_uint64(0)
        got = self.f(bytes(x), len(x), level, 4, 1 << n, b.ctypes.data, h.ctypes.data, nch, tok.ctypes.data, tok.size,
                     per.ctypes.data, cnt.ctypes.data, ctypes.byref(edge))
        assert got >= 0, got
        edges = np.concatenate([[0], np.cumsum(per.astype(np.int64))])
        return [tok[edges[i]:edges[i + 1]] for i in range(1, nch)], edge.value


@pytest.fixture(scope="module")
def wmodel(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lz2w") / "liblz2_window_model.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(NATIVE, "lz2_window_model.c")])
    return WindowedSchedule(so)


def edge_case(n, seed=0):
    """A 32 KiB dictionary D and a member M whose first 300 bytes repeat W from exactly 2^n bytes before its end:
    the only earlier copy of them lies 2^n back, in W (the rest of D is random, the rest of M text)."""
    rng = random.Random(seed * 31 + n)
    text = util.text_corpus(util.load_corpus())
    d = rng.randbytes(32768)
    a = rng.randrange(len(text) - 140000)
    m = d[32768 - (1 << n):][:300] + text[a:a + 140000]
    return d, m


def replay(w, chunks):
    """-> (the bytes the tokens rebuild after W, the largest distance, a match reaching exactly len into W seen)"""
    out = bytearray(w)
    far, into_w_at = 0, set()
    for arr in chunks:
        for t in decode(arr):
            if isinstance(t, int):
                out.append(t)
            else:
                ln, dist = t
                far = max(far, dist)
                if dist > len(out) - len(w):
                    into_w_at.add(dist)
                for _ in range(ln):
                    out.append(out[-dist])
    return bytes(out[len(w):]), far, into_w_at


@pytest.mark.parametrize("n", WINDOW_BITS)
def test_model_on_window_and_member(wmodel, n):
    d, m = edge_case(n)
    w = window(d)
    for level in LEVELS:
        chunks, at_edge = wmodel.member(w, m, level, n)
        back, far, into_w = replay(w, chunks)
        assert back == m, (n, level)
        assert far <= 1 << n, (n, level, far)
        assert (1 << n) in into_w and at_edge >= 1, (n, level)
