"""k_huff (zippy_b200/csrc/zb_huff_warp.cuh), the warp-per-chunk codebook builder, against the host builder
zb_build_codebook (zb_huff.h): the whole ZbCodebook, byte for byte, on seeded histograms.

The kernel is compiled into a test-only library (tests/native/huff_warp.cu) that launches it on given
histograms.  The host builder writes into a zero-filled struct; the fields it leaves alone (ll, dd and hdr of a
stored block, hdr past the header's last byte) must come out 0 from the kernel, whose output buffer starts as
0xa5 bytes.  The cases cover 0, 1, 2 and all used literal/length and distance symbols, depth-forcing frequencies
that hit the 15-bit limit and the code-length code's 7-bit limit, counts summing to 65 537, chunk lengths 0, 1 and
65 536, both BFINAL values, level 0 (stored forced) and the block choice at one byte either side of a tie."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HOST_UNITS = os.path.join(HERE, "native", "host_units.cpp")
HUFF_WARP = os.path.join(HERE, "native", "huff_warp.cu")
CSRC = os.path.join(ROOT, "zippy_b200", "csrc")
WORDS = 418
LEN_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
FIXED_LL = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 6
CLCL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


class Host:
    def __init__(self, so):
        self.L = ctypes.CDLL(so)
        self.nbytes = self.L.t_codebook_size()
        assert self.nbytes == 4 * WORDS

    def build(self, h, ln, fin, force):
        cb = ctypes.create_string_buffer(self.nbytes)
        self.L.t_build_codebook(h.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), int(ln), int(fin), int(force), cb)
        return cb.raw

    def lengths(self, freq, limit):
        f = np.ascontiguousarray(freq, dtype=np.uint32)
        out = np.zeros(len(f), dtype=np.uint8)
        self.L.t_huff_lengths(f.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), len(f), limit,
                              out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)))
        return out.astype(np.int64)

    def coded_bits(self, h):
        """(dynamic, fixed) block bits of a histogram, from the host builder's code lengths."""
        tot = h.astype(np.int64).sum(axis=0)
        llf, df = tot[:286].copy(), tot[286:]
        llf[256] = 1   # end-of-block, once
        lll, ldl = self.lengths(llf, 15), self.lengths(df, 15)
        extra = int((llf[257:] * LEN_EXTRA).sum() + (df * DIST_EXTRA).sum())
        nll = max([257] + [s + 1 for s in range(286) if lll[s]])
        nd = max([1] + [s + 1 for s in range(30) if ldl[s]])
        seq = list(lll[:nll]) + list(ldl[:nd])
        rsym, i = [], 0
        while i < len(seq):
            v, run = seq[i], 1
            while i + run < len(seq) and seq[i + run] == v:
                run += 1
            left = run
            if v == 0:
                while left >= 11:
                    r = min(left, 138)
                    rsym.append(18)
                    left -= r
                if left >= 3:
                    rsym.append(17)
                    left = 0
                rsym += [0] * left
            else:
                rsym.append(v)
                left -= 1
                while left >= 3:
                    r = min(left, 6)
                    rsym.append(16)
                    left -= r
                rsym += [v] * left
            i += run
        cll = self.lengths(np.bincount(rsym, minlength=19), 7)
        hclen = max([4] + [i + 1 for i in range(19) if cll[CLCL_ORDER[i]]])
        hdr = 17 + 3 * hclen + sum(int(cll[r]) + {16: 2, 17: 3, 18: 7}.get(r, 0) for r in rsym)
        dyn = hdr + int((llf * lll).sum() + (df * ldl).sum()) + extra
        fix = 3 + int((llf * FIXED_LL[:286]).sum() + 5 * df.sum()) + extra
        return dyn, fix


def block_bytes(bits, fin):
    return (bits + 7) // 8 if fin else (bits + 3 + 7) // 8 + 4


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("huff_host") / "libhost_units.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, HOST_UNITS])
    return Host(so)


@pytest.fixture(scope="module")
def kernel(tmp_path_factory):
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    so = str(tmp_path_factory.mktemp("huff_warp") / "libhuff_warp.so")
    subprocess.check_call([os.environ.get("NVCC", "nvcc")] + g.NVCC_FLAGS + ["-o", so, HUFF_WARP], cwd=CSRC)
    L = ctypes.CDLL(so)
    assert L.t_codebook_size() == 4 * WORDS

    def run(hists, lens, finals, level):
        n = len(hists)
        h = np.ascontiguousarray(np.stack(hists), dtype=np.uint16)
        ln = np.ascontiguousarray(lens, dtype=np.uint32)
        fi = np.ascontiguousarray(finals, dtype=np.int32)
        out = np.zeros(n * 4 * WORDS, dtype=np.uint8)
        rc = L.t_huff_warp(h.ctypes.data_as(ctypes.c_void_p), ln.ctypes.data_as(ctypes.c_void_p),
                           fi.ctypes.data_as(ctypes.c_void_p), n, level, out.ctypes.data_as(ctypes.c_void_p))
        assert rc == 0, "CUDA error %d" % rc
        return [out[i * 4 * WORDS:(i + 1) * 4 * WORDS].tobytes() for i in range(n)]
    return run


def split8(rng, tot):
    """counts per symbol [316] -> the eight sub-chunk histograms, 8 x 316 u16"""
    tot = np.asarray(tot, dtype=np.int64)
    h = np.zeros((8, 316), dtype=np.int64)
    for s in np.nonzero(tot)[0]:
        h[:, s] = rng.multinomial(int(tot[s]), [1 / 8] * 8)
    assert h.max() <= 65535
    return np.ascontiguousarray(h, dtype=np.uint16)


def pick(rng, n, k, avoid=()):
    return rng.choice([s for s in range(n) if s not in avoid], k, replace=False)


def gen_cases(rng):
    """-> list of (name, hist 8 x 316, chunk_len, is_final)"""
    cases = []

    def add(name, tot, ln=None):
        h = split8(rng, tot)
        if ln is None:
            ln = int(rng.choice([0, 1, 65536, int(rng.integers(2, 65536))]))
        cases.append((name, h, ln, int(rng.integers(0, 2))))

    def dist_counts(kind):
        d = np.zeros(30, dtype=np.int64)
        if kind == "none":
            return d
        k = {"one": 1, "two": 2, "all": 30, "some": int(rng.integers(3, 30))}[kind]
        d[pick(rng, 30, k)] = rng.integers(1, 3000, k)
        return d

    dkinds = ["none", "one", "two", "all", "some"]
    for t in range(300):   # 0, 1, 2 or all literal/length symbols besides end-of-block
        k = [0, 1, 2, 285, int(rng.integers(3, 285))][t % 5]
        ll = np.zeros(286, dtype=np.int64)
        if k:
            ll[pick(rng, 286, k, avoid=(256,))] = rng.integers(1, 2000, k)
        add("ll%d" % k, np.concatenate([ll, dist_counts(dkinds[(t // 5) % 5])]))
    for t in range(500):   # text-like: skewed literals, matches
        ll = np.zeros(286, dtype=np.int64)
        ntok = int(rng.integers(1, 60000))
        p = rng.dirichlet(np.full(96, 0.3))
        ll[32:128] = rng.multinomial(ntok, p)
        nm = int(rng.integers(0, 8000))
        ll[257:286] += rng.multinomial(nm, rng.dirichlet(np.full(29, 0.5)))
        d = rng.multinomial(nm, rng.dirichlet(np.full(30, 0.5)))
        add("text", np.concatenate([ll, d]))
    for t in range(400):   # heavy-tailed counts: code lengths spread widely, the code-length code at its 7-bit limit
        tot = np.zeros(316, dtype=np.int64)
        used = rng.random(316) > rng.uniform(0.1, 0.7)
        tot[used] = np.minimum(8 * 65535, np.maximum(1, rng.lognormal(3, 2, used.sum()).astype(np.int64)))
        add("lognormal", tot)
    for t in range(200):   # depth-forcing frequencies (w[i] = w[i-1] + w[i-2] + 1): the 15-bit limit
        tot = np.zeros(316, dtype=np.int64)
        k = int(rng.integers(16, 20))
        a, b = 2, 3
        for s in pick(rng, 286, k, avoid=(256,)):
            tot[s] = a
            a, b = b, a + b + 1
        if t % 2:
            kd = int(rng.integers(2, 19))
            a, b = 1, 2
            for s in pick(rng, 30, kd):
                tot[286 + s] = a
                a, b = b, a + b + 1
        add("fib", np.minimum(tot, 8 * 65535))
    for t in range(200):   # a full 64 KiB chunk of literals: 65 536 + end-of-block = 65 537 tokens
        tot = np.zeros(316, dtype=np.int64)
        k = int(rng.choice([1, 2, 16, 256]))
        tot[pick(rng, 256, k)] = rng.multinomial(65536, rng.dirichlet(np.full(k, 1.0)))
        add("full", tot, 65536)
    for t in range(100):   # uniform random bytes
        tot = np.zeros(316, dtype=np.int64)
        tot[:256] = rng.multinomial(65536, np.full(256, 1 / 256))
        add("random", tot, 65536)
    for t in range(100):   # long runs of equal code lengths (RLE codes 16, 17, 18)
        tot = np.zeros(316, dtype=np.int64)
        lo = int(rng.integers(0, 200))
        tot[lo:lo + int(rng.integers(1, 86))] = int(rng.integers(1, 50))
        tot[286 + int(rng.integers(0, 30))] = int(rng.integers(0, 5))
        add("runs", tot)
    return cases


def margin_cases(host, rng, n):
    """Histograms whose block choice is decided by one byte: fixed vs dynamic (found by search), and stored vs
    the better coded block (the chunk length set against it): -> list of (name, hist, chunk_len, is_final)."""
    out, found = [], {"fix_by_1": 0, "dyn_by_1": 0, "fix_dyn_tie": 0}
    tries = 0
    while min(found.values()) < n // 6 and tries < 20000:
        tries += 1
        tot = np.zeros(316, dtype=np.int64)
        k = int(rng.integers(1, 40))
        tot[pick(rng, 286, k, avoid=(256,))] = rng.integers(1, 12, k)
        kd = int(rng.integers(0, 6))
        if kd:
            tot[286 + pick(rng, 30, kd)] = rng.integers(1, 6, kd)
        h = split8(rng, tot)
        dyn, fix = host.coded_bits(h)
        for fin in (0, 1):
            db, fb = block_bytes(dyn, fin), block_bytes(fix, fin)
            name = {db - 1: "fix_by_1", db + 1: "dyn_by_1", db: "fix_dyn_tie"}.get(fb)
            if name and found[name] < n // 6:
                found[name] += 1
                out.append((name, h, 65536, fin))
    assert min(found.values()) >= n // 6, found
    for t in range(n // 2):   # stored wins by one byte, ties (stored wins), loses by one byte
        tot = np.zeros(316, dtype=np.int64)
        k = int(rng.integers(1, 200))
        tot[pick(rng, 286, k, avoid=(256,))] = rng.integers(1, 300, k)
        h = split8(rng, tot)
        fin = int(rng.integers(0, 2))
        dyn, fix = host.coded_bits(h)
        coded = min(block_bytes(dyn, fin), block_bytes(fix, fin))
        d = [-1, 0, 1][t % 3]
        ln = coded + d - 5
        if 0 <= ln <= 65535:
            out.append(("stored%+d" % d, h, ln, fin))
    return out


def header_field(raw, bit, n):
    bits = np.unpackbits(np.frombuffer(raw[4 * 334:], dtype=np.uint8), bitorder="little")
    return int(sum(int(bits[bit + i]) << i for i in range(n)))


@pytest.mark.gpu
def test_k_huff_matches_host_builder(host, kernel):
    rng = np.random.default_rng(20261017)
    cases = gen_cases(rng) + margin_cases(host, rng, 300)
    assert len(cases) >= 2000
    for level, force in ((1, -1), (0, 0)):
        got = kernel([c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases], level)
        seen = set()
        for (name, h, ln, fin), g in zip(cases, got):
            want = host.build(h, ln, fin, force)
            if g != want:
                a, b = np.frombuffer(g, dtype=np.uint32), np.frombuffer(want, dtype=np.uint32)
                bad = np.nonzero(a != b)[0]
                pytest.fail("%s (len %d, final %d, level %d): %d words differ, first at word %d: %#x != %#x"
                            % (name, ln, fin, level, len(bad), bad[0], a[bad[0]], b[bad[0]]))
            u32 = np.frombuffer(want, dtype=np.uint32)
            btype = int(u32[320])
            seen.add(("type", btype))
            if name.startswith(("fix_", "dyn_", "stored")):
                seen.add((name, btype))
            if btype == 2:
                seen.add(("ll15", int((u32[:286] >> 16).max()) == 15))
                hclen = header_field(want, 13, 4) + 4
                seen.add(("cl7", max(header_field(want, 17 + 3 * i, 3) for i in range(hclen)) == 7))
            if force == -1 and btype == 2:   # the size model the margin search uses agrees with the builder
                # eob_bit_start: the tokens of the histograms (their end-of-block counts too) before end-of-block
                l256 = int(u32[256] >> 16)
                assert host.coded_bits(h)[0] == int(u32[330]) + l256 * (1 - int(h[:, 256].astype(np.int64).sum())), name
            if ln in (0, 1, 65536):
                seen.add(("len", ln))
            seen.add(("final", fin))
        if force == 0:
            assert seen >= {("type", 0)} and ("type", 2) not in seen
            continue
        assert {("type", 0), ("type", 1), ("type", 2), ("ll15", True), ("cl7", True), ("len", 0), ("len", 1),
                ("len", 65536), ("final", 0), ("final", 1), ("fix_by_1", 1), ("dyn_by_1", 2), ("fix_dyn_tie", 2),
                ("stored-1", 0), ("stored+0", 0)} <= seen
        assert ("stored+1", 1) in seen or ("stored+1", 2) in seen
