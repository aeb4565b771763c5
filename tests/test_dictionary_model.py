"""The dictionary parse of levels -1 and 2..9 against the schedule model (tests/native/lz2_schedule_model.c):
a member M compressed against a window W is the schedule model run on W || M with a chunk boundary at |W| and no
reset, so every chunk of M sees min(32 KiB, bytes before it in W || M) of history.  The CPU part checks the model
on W || M by itself; the GPU part requires k_lz2's tokens (read back through stored(W) || member) to be the model's."""
import random

import numpy as np
import pytest

from tests import deflate_tokens as dt
from tests import util
from tests.test_dictionary_rules import stored, window
from tests.test_gpu_lz2_model import decode, encode
from tests.test_gpu_stream_flush import model  # noqa: F401  (the schedule model fixture)

CHUNK = 65536
WINDOWS = [1, 100, 8191, 8193, 32767, 32768, 100000]
LEVELS = [-1, 2, 6, 9]


@pytest.fixture(scope="module")
def text():
    return util.text_corpus(util.load_corpus())


def _case(text, dlen):
    rng = random.Random(dlen)
    a = rng.randrange(len(text) - dlen - 300000)
    d = text[a:a + dlen]
    pre = d[-min(dlen, 3000):]
    m = pre * (1 + 8 // len(pre)) + text[a + dlen + 5000:a + dlen + 5000 + 140000]   # starts with a repeat of W's end
    return d, m


def schedule(model, w, m, level):
    """-> the model's tokens of M's chunks, run on W || M with a boundary at |W| and no reset."""
    x = w + m
    bounds = [0, len(w)] + list(range(len(w) + CHUNK, len(x), CHUNK)) + [len(x)]
    if bounds[-1] == bounds[-2] and len(bounds) > 3:
        bounds.pop()
    return model.run_schedule(x, level, bounds, [0] * (len(bounds) - 1))[1:]


@pytest.mark.parametrize("dlen", WINDOWS)
def test_schedule_on_window_and_member(model, text, dlen):
    d, m = _case(text, dlen)
    w = window(d)
    for level in LEVELS:
        chunks = schedule(model, w, m, level)
        out = bytearray(w)
        into_w = False
        for arr in chunks:
            for t in decode(arr):
                if isinstance(t, int):
                    out.append(t)
                else:
                    ln, dist = t
                    into_w |= dist > len(out) - len(w)
                    for _ in range(ln):
                        out.append(out[-dist])
        assert bytes(out[len(w):]) == m, (dlen, level)
        assert into_w, (dlen, level)


@pytest.mark.gpu
@pytest.mark.parametrize("dlen", WINDOWS)
def test_kernel_tokens_equal_the_schedule(model, text, dlen):
    import zippy_b200 as z
    d, m = _case(text, dlen)
    w = window(d)
    for level in LEVELS:
        c = z.compress(m, level, z.dfDeflate, dictionary=d)
        blocks = dt.parse(stored(w) + c)
        got = dt.member_chunks(blocks[1:])
        want = schedule(model, w, m, level)
        assert len(got) == len(want), (dlen, level)
        compared = 0
        for k, (g, wt) in enumerate(zip(got, want)):
            if g.btype == 0:
                continue
            compared += 1
            assert np.array_equal(encode(g.tokens), wt), (dlen, level, k)
        assert compared >= 1
