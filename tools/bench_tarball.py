"""Time one large tarball through the GPU: the tar image compressed as one gzip member at DefaultCompression
(zippy_b200.compress, what Tarball.write_tarball does for .tar.gz) and read back (read_tarball: the member
inflated by the GPU path, then the header walk), plus the same two steps through files
(write_tarball / extract_all in a temporary directory).  Prints one JSON line.

    python tools/bench_tarball.py [--mib 1024] [--repeats 3] [--seed 7]

The tree is seeded and held in memory: text windows of the test corpus, byte runs and random bytes in
files of 0..8 MiB.  Each call is timed on the host clock; every call returns after its device work has
finished and its output is in host memory."""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def seeded_contents(total, seed):
    from tests import util
    import zippy_b200.tarballs as tb
    T = util.text_corpus(util.load_corpus())
    rng = np.random.default_rng(seed)
    contents, done, i = {}, 0, 0
    while done < total:
        n = int(min(rng.integers(0, 8 << 20), total - done))
        kind = i % 3
        if kind == 0:
            o = int(rng.integers(0, len(T)))
            data = (T * (2 + n // len(T)))[o:o + n]
        elif kind == 1:
            runs = rng.integers(1, 256, n // 64 + 1)
            data = np.repeat(rng.integers(0, 256, len(runs), dtype=np.uint8), runs)[:n].tobytes()
        else:
            data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        d = "big/d%d/e%d" % (i % 7, i % 3)
        for p in ("big", "big/d%d" % (i % 7), d):
            contents.setdefault(p, tb.TarballEntry("dir"))
        contents["%s/f%d.bin" % (d, i)] = tb.TarballEntry("file", data, 1700000000 + i, 0o644)
        done += len(data)
        i += 1
    return contents


def timed(fn, repeats):
    ts, out = [], None
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return out, ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    import zippy_b200 as z
    import zippy_b200.tarballs as tb
    contents = seeded_contents(a.mib << 20, a.seed)
    image = tb.tar_image(contents)
    gib = len(image) / (1 << 30)
    z.uncompress(z.compress(image[:64 << 20], z.DefaultCompression, z.dfGzip))  # warm-up: module load, scratch
    member, c_ms = timed(lambda: z.compress(image, z.DefaultCompression, z.dfGzip), a.repeats + 1)
    n_chunks = z.default_context().timing()["n_chunks"]
    back, r_ms = timed(lambda: tb.read_tarball(member), a.repeats + 1)
    assert [e[1] for e in back] == list(contents) and z.uncompress(member) == image
    t = tb.Tarball()
    t.contents = contents
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "big.tar.gz")
        _, w_ms = timed(lambda: t.write_tarball(path), a.repeats)
        dests = iter(range(a.repeats))
        _, x_ms = timed(lambda: tb.extract_all(path, os.path.join(tmp, "out%d" % next(dests))), a.repeats)
    med = lambda ts: statistics.median(ts[-a.repeats:])  # noqa: E731  (the first call is a warm-up)
    print(json.dumps({
        "tar_image_gib": round(gib, 4), "member_bytes": len(member), "ratio": round(len(member) / len(image), 4),
        "n_chunks": n_chunks,
        "compress_ms": round(med(c_ms), 1), "compress_gibs": round(gib / med(c_ms) * 1e3, 2),
        "read_back_ms": round(med(r_ms), 1), "read_back_gibs": round(gib / med(r_ms) * 1e3, 2),
        "write_tarball_ms": round(med(w_ms), 1), "extract_all_ms": round(med(x_ms), 1),
        "all_ms": {"compress": [round(x, 1) for x in c_ms], "read_back": [round(x, 1) for x in r_ms],
                   "write_tarball": [round(x, 1) for x in w_ms], "extract_all": [round(x, 1) for x in x_ms]},
    }))


if __name__ == "__main__":
    main()
