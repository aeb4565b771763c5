"""The compress call's host plan: one pass over the members writes the chunk descriptors into the context's pinned
buffer, which every call reuses (zb_api.cu, compress_locked).

A call that fails part way through, or a batch of another shape, must not leave anything behind in that buffer that
changes the next call's bytes; offsets that decrease anywhere in the batch are rejected before any launch; and the
host time up to the first launch is reported as `plan_ms`."""
import random

import numpy as np
import pytest

from tests import util

pytestmark = pytest.mark.gpu

ERR_DST_TOO_SMALL = 19
ERR_ARG = 22


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


@pytest.fixture(scope="module")
def members(corpus):
    rng = random.Random(0x91A)
    T = util.text_corpus(corpus)
    out = []
    for n in (70001, 0, 1, 65536, 131073, 4096, 65535, 200000, 12, 65537):
        o = rng.randrange(len(T) - n)
        out.append(T[o:o + n])
    return out


@pytest.fixture
def group1_ctx(z, monkeypatch):
    monkeypatch.setenv("ZB200_GROUP_CHUNKS", "1")   # one launch group per member: many groups, many plan entries
    ctx = z.Context()
    yield ctx
    ctx.close()


def _raw_compress(z, ctx, items, level, df, cap):
    L = z._native.lib()
    base, offs = z._pack(items)
    out = np.empty(max(cap, 4), dtype=np.uint8)
    oo = np.zeros(len(items) + 1, dtype=np.uint64)
    st = np.zeros(max(len(items), 1), dtype=np.int32)
    return L.zb200_compress_batch(ctx._h, base.ctypes.data, offs.ctypes.data, len(items), level, df, None,
                                  out.ctypes.data, cap, oo.ctypes.data, st.ctypes.data)


@pytest.mark.parametrize("level", [1, -1])
def test_calls_after_a_failed_call_give_the_same_bytes(z, members, group1_ctx, level):
    """A host-buffer call that runs out of destination after several launch groups, then batches of other shapes
    through the host and device calls, equal each member compressed alone on a fresh context."""
    torch = pytest.importorskip("torch")
    ref = [z.compress_batch([m], level, z.dfGzip)[0] for m in members]
    ctx = group1_ctx
    assert _raw_compress(z, ctx, members, level, z.dfGzip, 4096) == ERR_DST_TOO_SMALL
    for idx in (list(range(len(members))), [7, 3, 1], [4], list(range(len(members)))[::-1]):
        items = [members[i] for i in idx]
        out, oo = ctx.compress_batch(*z._pack(items), level, z.dfGzip)
        assert [bytes(out[int(oo[k]):int(oo[k + 1])]) for k in range(len(idx))] == [ref[i] for i in idx]
        base, offs = z._pack(items)
        d_src = torch.from_numpy(base.copy()).cuda() if len(base) else torch.zeros(1, dtype=torch.uint8, device="cuda")
        cap = int(sum(z._native.lib().zb200_compress_bound(len(m), z.dfGzip) + 64 for m in items))
        d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
        oo = ctx.compress_batch_device(d_src.data_ptr(), offs, level, z.dfGzip, d_dst.data_ptr(), cap)
        host = d_dst[:int(oo[-1])].cpu().numpy()
        assert [bytes(host[int(oo[k]):int(oo[k + 1])]) for k in range(len(idx))] == [ref[i] for i in idx]


def test_decreasing_offsets_are_rejected(z, group1_ctx):
    """Offsets that decrease after a long member (more chunks than the batch's byte span allows), at the end, or
    in the middle, are ERR_ARG; the context then compresses as before."""
    L = z._native.lib()
    base = np.frombuffer(bytes(range(256)) * 4096, dtype=np.uint8)   # 1 MiB
    out = np.empty(1 << 22, dtype=np.uint8)
    for ctx in (group1_ctx, z.default_context()):
        for offs in ([0, 1 << 20, 0], [0, 1 << 20, 5], [0, 10, 5, 20], [100, 200, 50], [0, 300000, 200000, 1 << 20]):
            o = np.array(offs, dtype=np.uint64)
            n = len(offs) - 1
            oo = np.zeros(n + 1, dtype=np.uint64)
            rc = L.zb200_compress_batch(ctx._h, base.ctypes.data, o.ctypes.data, n, 1, z.dfGzip, None,
                                        out.ctypes.data, out.size, oo.ctypes.data, None)
            assert rc == ERR_ARG, offs
        item = bytes(base[:300000])
        got, oo = ctx.compress_batch(*z._pack([item, b"", item]), 1, z.dfGzip)
        assert bytes(got[:int(oo[1])]) == z.compress_batch([item], 1, z.dfGzip)[0]


def test_plan_time_is_reported(z, corpus):
    torch = pytest.importorskip("torch")
    T = util.text_corpus(corpus)
    n = 256
    src = np.frombuffer(b"".join(util.c2_block(T, i) for i in range(n)), dtype=np.uint8)
    d_src = torch.from_numpy(src.copy()).cuda()
    offs = np.arange(n + 1, dtype=np.uint64) * 65536
    cap = n * (65536 + 96) + 4096
    d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    ctx = z.Context()
    try:
        ctx.compress_batch_device(d_src.data_ptr(), offs, 1, z.dfGzip, d_dst.data_ptr(), cap)
        tm = ctx.timing()
        assert tm["plan_ms"] > 0.0 and tm["n_chunks"] == n
        assert tm["plan_ms"] < 1000.0
    finally:
        ctx.close()
