"""The inflate kernel on hand-built DEFLATE streams (tests/deflate_writer.py): every catalogue case and a
seeded sweep through every decode path -- the batch call with and without caller sizes, the device batch,
the sizing pass, the single calls -- at member alignments 0..3, next to other members and bytes, at all 32
bit phases of a 48-bit token, through the host pipeline and through the large-member segment paths.  Every
member must give the replay's bytes or the oracle's exact error code."""
import random

import numpy as np
import pytest

from tests import deflate_writer as w

pytestmark = pytest.mark.gpu

RAW, ZLIB, GZIP = 3, 1, 2


@pytest.fixture(scope="module")
def z():
    import zippy_b200
    return zippy_b200


@pytest.fixture(scope="module")
def o():
    from oracle import oracle
    return oracle


def verdict(o, data, fmt, pos=0):
    """The oracle's answer: output bytes or error code (pos > 0: a raw stream from byte pos)."""
    try:
        return o.inflate(data, pos) if pos else o.uncompress(data, fmt)
    except o.ZippyError as e:
        return e.code


def wrap(data, want, fmt):
    body = want if isinstance(want, bytes) else b""
    return data if fmt == RAW else w.zlib_wrap(data, body) if fmt == ZLIB else w.gzip_wrap(data, body, fname=b"m")


def sweep():
    """Seeded valid streams over every knob of the generator."""
    out = []
    for seed in range(24):
        dist = ("one", "short", "far", "dependent")[seed % 4]
        blocks = w.random_stream(100 + seed, skew=("flat", "deep")[(seed // 4) % 2], dist=dist, phase=seed % 32,
                                 history=32768 + seed if dist in ("far", "dependent") else 0,
                                 kinds=(("dynamic",), ("dynamic", "fixed", "stored"), ("fixed", "stored"))[seed % 3],
                                 nblocks=2 + seed % 3, block_tokens=(1, 60 + 20 * seed))
        out.append(("sweep_%d" % seed, w.raw(blocks), w.replay(blocks)))
    return out


def members(fmt):
    """[(name, member bytes)] for the catalogue and the sweep, wrapped for `fmt`."""
    items = [(c.name, wrap(c.data, c.want, fmt)) for c in w.catalogue()]
    items += [(n, wrap(d, want, fmt)) for n, d, want in sweep()]
    return items


def pack(items, fill=0xA5):
    """Members at byte alignments 0..3 of the buffer: 0..3 filler bytes (a member of their own) go
    before member i so that it starts at offset = i mod 4."""
    blob, offs, names = bytearray(), [0], []
    for i, (name, m) in enumerate(items):
        pad = (i - len(blob)) % 4
        if pad:
            blob += bytes([fill]) * pad
            offs.append(len(blob))
            names.append("filler")
        blob += m
        offs.append(len(blob))
        names.append(name)
    return np.frombuffer(bytes(blob), dtype=np.uint8), np.array(offs, dtype=np.uint64), names


def check(names, base, offs, fmt, o, out, do, lens, st, tag):
    for i, name in enumerate(names):
        m = base[int(offs[i]):int(offs[i + 1])].tobytes()
        want = verdict(o, m, fmt)
        if isinstance(want, int):
            assert int(st[i]) == want, (tag, name, int(st[i]), want)
        else:
            assert int(st[i]) == 0, (tag, name, int(st[i]))
            assert out[int(do[i]):int(do[i]) + int(lens[i])].tobytes() == want, (tag, name)


@pytest.mark.parametrize("fmt", [RAW, ZLIB, GZIP])
def test_batch_three_ways(z, o, fmt):
    torch = pytest.importorskip("torch")
    base, offs, names = pack(members(fmt))
    n = len(names)
    ctx = z.Context()
    out, do, lens, st = ctx.uncompress_batch(base, offs, fmt)
    check(names, base, offs, fmt, o, out, do, lens, st, "batch")
    # caller sizes: the decode pass's own verdict (no sizing pass in front of it)
    wants = [verdict(o, base[int(offs[i]):int(offs[i + 1])].tobytes(), fmt) for i in range(n)]
    sizes = np.array([len(v) if isinstance(v, bytes) else 1 << 16 for v in wants], dtype=np.uint64)
    out, do, lens, st = ctx.uncompress_batch(base, offs, fmt, sizes=sizes)
    check(names, base, offs, fmt, o, out, do, lens, st, "sized")
    # device batch, caller offsets
    dsz = np.array([len(v) + 64 if isinstance(v, bytes) else 1 << 16 for v in wants], dtype=np.uint64)
    doffs = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(dsz, out=doffs[1:])
    d_src = torch.from_numpy(base.copy()).cuda()
    d_dst = torch.zeros(int(doffs[-1]) + 64, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    lens, st = ctx.uncompress_batch_device(d_src.data_ptr(), offs, fmt, d_dst.data_ptr(), doffs)
    check(names, base, offs, fmt, o, d_dst.cpu().numpy(), doffs, lens, st, "device")
    if fmt != GZIP:   # the sizing pass decodes zlib and raw members (gzip answers from ISIZE)
        for tag, (sz, sst) in (("sizes", ctx.uncompressed_sizes(base, offs, fmt)),
                               ("sizes_device", ctx.uncompressed_sizes_device(d_src.data_ptr(), offs, fmt))):
            for i, name in enumerate(names):
                m = base[int(offs[i]):int(offs[i + 1])].tobytes()
                want = verdict(o, m, fmt) if fmt == RAW or len(m) < 6 else verdict(o, m, fmt, pos=2)
                if isinstance(verdict(o, m, fmt), int) and verdict(o, m, fmt) in (9, 10, 11, 12, 13):
                    want = verdict(o, m, fmt)   # a wrapper error, reported before any decoding
                if isinstance(want, int):
                    assert int(sst[i]) == want, (tag, name, int(sst[i]), want)
                else:
                    assert int(sst[i]) == 0 and int(sz[i]) == len(want), (tag, name, int(sst[i]), int(sz[i]))
    ctx.close()


def test_single_calls(z, o):
    ctx = z.Context()
    for c in w.catalogue():
        for fmt in (RAW, ZLIB):
            m = wrap(c.data, c.want, fmt)
            want = verdict(o, m, fmt)
            for call in (lambda: z.uncompress(m, fmt), lambda: ctx.decode_one(m, fmt)):
                if isinstance(want, int):
                    with pytest.raises(z.ZippyError) as e:
                        call()
                    assert e.value.code == want, (c.name, fmt, e.value.code, want)
                else:
                    assert call() == want, (c.name, fmt)
        for k in (1, 3, 6):
            m = bytes(range(200, 200 + k)) + c.data
            want = verdict(o, m, RAW, pos=k)
            if isinstance(want, int):
                with pytest.raises(z.ZippyError) as e:
                    ctx.inflate(m, pos=k)
                assert e.value.code == want, (c.name, k, e.value.code, want)
            else:
                assert ctx.inflate(m, pos=k) == want, (c.name, k)
    ctx.close()


def truncations():
    """Byte cuts of streams whose every part matters: headers, 15-bit codes, fixed and stored blocks."""
    cat = {c.name: c for c in w.catalogue()}
    srcs = [cat["dynamic_small"].data, cat["repeat16_across_lit_dist_boundary"].data, cat["fixed_every_length"].data[:90],
            w.raw(w.random_stream(7, skew="deep", dist="short", nblocks=2, block_tokens=(20, 40))),
            w.raw([w.Fixed(list(b"abcdefgh"), final=False), w.Stored(b"stored!", final=False), w.Fixed([(200, 3)])])]
    return [s[:k] for s in srcs for k in range(len(s))]


def test_truncated_members_next_to_other_bytes(z, o):
    """A truncated member followed by zeros, by ones, by another member, or last in the buffer: bits past
    its end are zeros for the reference whatever the buffer holds after it."""
    ctx = z.Context()
    cuts = truncations()
    good = w.raw([w.Fixed(list(b"neighbour") + [(30, 9)])])
    for follow in ("zeros", "ones", "member", "last"):
        items = []
        for k, c in enumerate(cuts):
            items.append(("cut%d" % k, c))
            if follow == "zeros":
                items.append(("z", b"\x00" * 5))
            elif follow == "ones":
                items.append(("f", b"\xff" * 5))
            elif follow == "member":
                items.append(("good", good))
        if follow == "last":
            items = items[::-1]
        base, offs, names = pack(items, fill=0xff if follow == "ones" else 0)
        out, do, lens, st = ctx.uncompress_batch(base, offs, RAW)
        check(names, base, offs, RAW, o, out, do, lens, st, follow)
        if follow == "last":   # the last member of the buffer, alone
            for c in cuts[-40:]:
                b1 = np.frombuffer(c, dtype=np.uint8)
                out, do, lens, st = ctx.uncompress_batch(b1, np.array([0, len(c)], dtype=np.uint64), RAW)
                check(["last"], b1, np.array([0, len(c)], dtype=np.uint64), RAW, o, out, do, lens, st, "alone")
    ctx.close()


def test_lockstep_members_stop_at_different_tokens(z, o):
    """Four members share a warp and decode in lockstep: put every valid case between failing members in
    several arrangements, failing after 0..31 tokens of a flush batch."""
    rng = random.Random(32)
    cat = w.catalogue()
    valid = [(c.name, c.data) for c in cat if isinstance(c.want, bytes)] + [(n, d) for n, d, _ in sweep()]
    failing = []
    for t in range(0, 40):
        toks = list(b"0123456789abcdefghijklmnopqrstuvwxyz")[:max(t, 0)] + [w.Sym(286)]
        failing.append(("fail_at_%d" % t, w.raw([w.Fixed(toks)])))
        failing.append(("far_at_%d" % t, w.raw([w.Fixed(list(range(65, 65 + t)) + [(5, t + 1)])])))
    ctx = z.Context()
    for arrangement in range(4):
        items = []
        for v in valid:
            for _ in range(arrangement % 3 + 1):
                items.append(rng.choice(failing))
            items.append(v)
        rng.shuffle(items) if arrangement == 3 else None
        base, offs, names = pack(items)
        out, do, lens, st = ctx.uncompress_batch(base, offs, RAW)
        check(names, base, offs, RAW, o, out, do, lens, st, "arrangement%d" % arrangement)
    ctx.close()


def test_48_bit_tokens_at_every_bit_phase(z, o):
    """The 48-bit token at all 32 start phases of the bit window and at every position of an 8-word line,
    at member alignments 0..3; the replay is the expected output."""
    items, wants = [], {}
    hist = bytes(random.Random(48).randbytes(32768 + 100))
    for p in range(0, 288, 1):
        blocks = w.deep_token_blocks(p, length=227 + (p % 31), dist=32768 - (p % 3), history=hist)
        items.append(("phase%d" % p, w.raw(blocks)))
        wants["phase%d" % p] = w.replay(blocks)
    base, offs, names = pack(items)
    ctx = z.Context()
    out, do, lens, st = ctx.uncompress_batch(base, offs, RAW)
    for i, name in enumerate(names):
        if name in wants:
            assert int(st[i]) == 0 and out[int(do[i]):int(do[i]) + int(lens[i])].tobytes() == wants[name], name
    for p in (0, 5, 31, 200):
        blob = items[p][1]
        assert ctx.inflate(blob) == wants["phase%d" % p]
        assert o.inflate(blob) == wants["phase%d" % p]
    ctx.close()


@pytest.mark.parametrize("gated", ["0", "1"])
def test_host_pipeline(z, o, monkeypatch, gated):
    monkeypatch.setenv("ZB200_UNC_GATED", gated)
    monkeypatch.setenv("ZB200_UNC_GROUP_BYTES", "4096")
    ctx = z.Context()
    monkeypatch.delenv("ZB200_UNC_GATED")
    monkeypatch.delenv("ZB200_UNC_GROUP_BYTES")
    for fmt in (ZLIB, GZIP):
        base, offs, names = pack(members(fmt))
        out, do, lens, st = ctx.uncompress_batch(base, offs, fmt)
        check(names, base, offs, fmt, o, out, do, lens, st, "gated" + gated)
    ctx.close()


def big_stream(seed, corrupt=None):
    """A multi-block member of a few hundred KB: dynamic blocks (15-bit codes and flat), fixed and stored
    blocks between them, matches at distance 32768 and long distance-1 runs across many blocks.
    corrupt: None, "middle" or "last" -- one invalid token in a middle block or in the last one."""
    rng = random.Random(seed)
    blocks = [w.Stored(rng.randbytes(40000), final=False)]
    out = bytearray(blocks[0].data)
    for k in range(90):
        kind = ("dynamic", "fixed", "dynamic", "stored", "dynamic")[k % 5]
        if kind == "stored":
            blocks.append(w.Stored(rng.randbytes(rng.choice((0, 5, 3000))), final=False))
            out += blocks[-1].data
            continue
        toks = []
        for _ in range(rng.randint(200, 900)):
            r = rng.random()
            if r < 0.3:
                toks.append(rng.randrange(256))
                out.append(toks[-1])
            elif r < 0.55:
                toks.append((rng.choice((258, 227, 131)), 32768))
                w._copy(out, toks[-1][0], 32768)
            elif r < 0.75:
                toks.append((258, 1))
                w._copy(out, 258, 1)
            else:
                d = rng.randint(1, 32768)
                toks.append((rng.randint(3, 258), d))
                w._copy(out, toks[-1][0], d)
        if kind == "fixed":
            blocks.append(w.Fixed(toks, final=False))
        else:
            blk = w.Dynamic(toks, final=False)
            if k % 2:
                fl, fd = w._frequencies(toks, True)
                order = list(range(286))
                rng.shuffle(order)
                for r_, s in enumerate(order):
                    fl[s] += 1 << max(0, 40 - r_)
                blk.ll_lens = w._trim(w.huffman_lengths(fl, 15), 257)
                dord = list(range(30))
                rng.shuffle(dord)
                for r_, s in enumerate(dord):
                    fd[s] += 1 << max(0, 30 - r_)
                blk.d_lens = w._trim(w.huffman_lengths(fd, 15), 1)
            blocks.append(blk)
    blocks.append(w.Fixed(list(b"end"), final=True))
    out += b"end"
    if corrupt:
        idx = len(blocks) // 2 if corrupt == "middle" else len(blocks) - 1
        while not isinstance(blocks[idx], w.Fixed):
            idx += 1
        blocks[idx].tokens.insert(len(blocks[idx].tokens) // 2, w.Sym(286))
        return w.raw(blocks), None
    assert w.replay(blocks) == bytes(out)
    return w.raw(blocks), bytes(out)


def test_large_members_through_segments(z, o, monkeypatch):
    monkeypatch.setenv("ZB200_BIG_MEMBER_BYTES", "60000")
    ctx = z.Context()
    monkeypatch.delenv("ZB200_BIG_MEMBER_BYTES")

    def one(m, fmt):
        b1 = np.frombuffer(m, dtype=np.uint8)
        offs = np.array([0, len(m)], dtype=np.uint64)
        out, do, lens, st = ctx.uncompress_batch(b1, offs, fmt)
        got = out[int(do[0]):int(do[0]) + int(lens[0])].tobytes() if st[0] == 0 else int(st[0])
        return got, ctx.timing()["kernel_launches"]

    _, small = one(wrap(w.raw([w.Fixed(list(b"x"))]), b"x", GZIP), GZIP)
    for seed in (1, 2):
        s, want = big_stream(seed)
        assert len(s) > 150000
        assert o.inflate(s) == want
        for fmt in (RAW, GZIP):
            got, launches = one(wrap(s, want, fmt), fmt)
            assert got == want, (seed, fmt, got if isinstance(got, int) else len(got))
            assert launches > small, (launches, small)   # not the serial path
        assert ctx.decode_one(w.zlib_wrap(s, want), ZLIB) == want
        for corrupt in ("middle", "last"):
            bad, _ = big_stream(seed, corrupt)
            for fmt in (RAW, ZLIB):
                m = wrap(bad, b"", fmt)
                got, _ = one(m, fmt)
                assert got == verdict(o, m, fmt), (seed, corrupt, fmt, got)
        rng = random.Random(seed)
        for _ in range(4):   # truncated: the cut falls in some segment
            cut = s[:rng.randrange(len(s) // 4, len(s))]
            got, _ = one(cut, RAW)
            assert got == verdict(o, cut, RAW), (seed, len(cut), got)
    ctx.close()
