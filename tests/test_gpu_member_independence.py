"""A member's compressed bytes depend on the member alone (DESIGN.md section 4).

Where a member sits must not show in its bytes: alone or in a batch, followed by a member that continues its
tail or by one that does not, after many chunks of 'a's or 'b's (what the persistent CTAs then hold in shared
memory from the chunks before), read from a device source at any offset mod 16, through the host, device and
host-to-device entry points, in launch groups of 1 and 3 chunks, on a fresh or the default context, and through
MultiGpu.  Every level -2..9, all three formats.  The members are the lazy traps of test_gpu_lz2_model.py
(whose parse turns on bytes just past the member if any rule reads them) and a few corpus and edge members."""
import random

import numpy as np
import pytest

from tests import util
from tests.test_gpu_lz2_model import trap_member

pytestmark = pytest.mark.gpu

LEVELS = list(range(-2, 10))
FORMATS = ("gzip", "zlib", "deflate")


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


@pytest.fixture(scope="module")
def members(corpus):
    rng = random.Random(0x1D)
    T = util.text_corpus(corpus)
    o = rng.randrange(len(T) - 100000)
    return [trap_member(False)[0], trap_member(True)[0], T[o:o + 70001], corpus["html"][:12345],
            bytes(rng.choice(b"abcdefgh ") for _ in range(8193)), b"abcaaaa", b""]


def _df(z, fmt):
    return {"gzip": z.dfGzip, "zlib": z.dfZlib, "deflate": z.dfDeflate}[fmt]


def _body(c, fmt):
    """A member without its gzip header (compress() gives it a random FNAME)."""
    c = bytes(c)
    if fmt != "gzip":
        return c
    assert c[:3] == b"\x1f\x8b\x08"
    i = 10
    if c[3] & 8:
        i = c.index(b"\x00", 10) + 1
    return c[i:]


def _split(out, oo, idx):
    return [bytes(out[int(oo[i]):int(oo[i + 1])]) for i in idx]


def _pack(items):
    import zippy_b200
    return zippy_b200._pack(items)


def _batch(ctx, items, level, df):
    base, offs = _pack(items)
    return ctx.compress_batch(base, offs, level, df)


@pytest.fixture(scope="module")
def contexts(z):
    mp = pytest.MonkeyPatch()
    ctxs = {}
    try:
        for g in ("1", "3"):
            mp.setenv("ZB200_GROUP_CHUNKS", g)
            ctxs["group" + g] = z.Context()
        mp.delenv("ZB200_GROUP_CHUNKS")
        ctxs["fresh"] = z.Context()
    finally:
        mp.undo()
    yield ctxs
    for c in ctxs.values():
        c.close()


@pytest.fixture(scope="module")
def poison(z):
    """Enough full chunks of 'a' (or 'b') that every CTA of a launch parses one before the members."""
    torch = pytest.importorskip("torch")
    n = 2 * torch.cuda.get_device_properties(0).multi_processor_count
    return {c: [c * 65536] * n for c in (b"a", b"b")}


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("level", LEVELS)
def test_member_bytes_do_not_depend_on_neighbours(z, members, contexts, poison, level, fmt):
    torch = pytest.importorskip("torch")
    df = _df(z, fmt)
    ref = [z.compress_batch([m], level, df)[0] for m in members]   # each member in a batch of its own
    seen = {}

    def expect(setting, got, body=False):
        for i, (g, r) in enumerate(zip(got, ref)):
            if (_body(g, fmt) if body else g) != (_body(r, fmt) if body else r):
                seen.setdefault(setting, []).append(i)

    # alone through compress(), on the default context
    expect("compress", [z.compress(m, level, df) for m in members], body=True)
    # one batch; each member followed by one that continues its tail, or by one that does not
    k = len(members)
    out, oo = _batch(z.default_context(), members, level, df)
    expect("batch", _split(out, oo, range(k)))
    for tail in (b"a" * 300, b"Zq" * 150):
        items = [x for m in members for x in (m, tail)]
        out, oo = _batch(z.default_context(), items, level, df)
        expect("followed_by_%r" % tail[:2], _split(out, oo, range(0, 2 * k, 2)))
    # after a full launch of 'a' / 'b' chunks, each member followed by 'a's
    for c, pre in poison.items():
        items = pre + [x for m in members for x in (m, b"a" * 300)]
        out, oo = _batch(z.default_context(), items, level, df)
        expect("after_%r_chunks" % c, _split(out, oo, range(len(pre), len(items), 2)))
    # launch groups of 1 and 3 chunks, and a fresh context
    for name in ("group1", "group3", "fresh"):
        items = poison[b"a"][:4] + [x for m in members for x in (m, b"a" * 40)]
        out, oo = _batch(contexts[name], items, level, df)
        expect(name, _split(out, oo, range(4, len(items), 2)))
    # device source at every offset mod 16, and host in / device out
    ctx = contexts["fresh"]
    ctx.set_stream(ctx.LEGACY_DEFAULT_STREAM)
    items = [x for m in members for x in (m, b"a" * 64)]
    base, offs = _pack(items)
    cap = int(offs[-1]) * 2 + 65536 * len(items)
    d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    d_all = torch.full((len(base) + 64,), ord("a"), dtype=torch.uint8, device="cuda")
    host_src = torch.from_numpy(base.copy())
    for shift in range(16):
        d_all[shift:shift + len(base)] = host_src.cuda()
        torch.cuda.synchronize()
        o2 = ctx.compress_batch_device(d_all.data_ptr() + shift, offs, level, df, d_dst.data_ptr(), cap)
        host = d_dst.cpu().numpy()
        expect("device_shift%d" % shift, _split(host, o2, range(0, 2 * k, 2)))
    pinned = host_src.pin_memory()
    o3 = ctx.compress_batch_h2d(pinned.data_ptr(), offs, level, df, d_dst.data_ptr(), cap)
    back = np.empty(int(o3[-1]), dtype=np.uint8)
    ctx.download(d_dst.data_ptr(), back.ctypes.data, back.size)
    expect("h2d", _split(back, o3, range(0, 2 * k, 2)))
    ctx.set_stream(0)
    assert not seen, "members whose bytes changed, by setting: %s" % seen


@pytest.mark.parametrize("fmt", FORMATS)
def test_multi_gpu_member_bytes(z, members, poison, fmt):
    """MultiGpu shards a batch over contexts (device 0 listed twice on one GPU): every member as one context
    compresses it, at Default."""
    from zippy_b200 import _native
    nd = _native.lib().zb200_device_count()
    df = _df(z, fmt)
    items = poison[b"a"][:8] + [x for m in members for x in (m, b"a" * 300)] * 3
    base, offs = _pack(items)
    ctx = z.Context()
    out, oo = ctx.compress_batch(base, offs, z.DefaultCompression, df)
    ctx.close()
    mg = z.MultiGpu(list(range(nd)) if nd > 1 else [0, 0])
    out2, oo2 = mg.compress_batch(base, offs, z.DefaultCompression, df)
    mg.close()
    alone = {m: z.compress_batch([m], z.DefaultCompression, df)[0] for m in set(items)}
    for i, m in enumerate(items):
        a = bytes(out[int(oo[i]):int(oo[i + 1])])
        b = bytes(out2[int(oo2[i]):int(oo2[i + 1])])
        assert a == b == alone[m], i
