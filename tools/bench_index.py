"""Random access through zippy_b200.Index.  Prints one JSON line per member with the card's name and power limit.

    python tools/bench_index.py [--mib 1024] [--small-mib 256] [--reads 4096] [--members all]

Members: --mib MiB of the C2 text (tests/util.c2_block) at level 1 and at Default, --small-mib MiB of it through
Python zlib at level 6, and --small-mib MiB of random bytes at level 1.  For each:
- build_s against uncompress_s (median of 3 each, after one warm-up);
- the index size in memory (points and raw windows) and exported;
- one_read_ms: one 4 KiB read at a random offset, median of 100;
- batch_gibs: --reads random 4 KiB reads in one extract_batch call, GiB/s of output, and the bytes uploaded per read;
- whole_gibs: extract(0, size) against uncompress, GiB/s of output.
Every read is checked against uncompress."""
import argparse
import json
import os
import random
import statistics
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_ziparchive import card  # noqa: E402


def corpus_text(mib):
    from tests import util
    T = util.text_corpus(util.load_corpus())
    return b"".join(util.c2_block(T, i) for i in range(mib * 16))


def timed(f, repeats=3):
    f()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def measure(z, ctx, name, data, out, reads):
    size = len(out)
    res = {"member": name, "compressed_bytes": len(data), "output_bytes": size}
    res["uncompress_s"] = timed(lambda: z.uncompress(data))
    res["build_s"] = timed(lambda: z.Index.build(data, ctx=ctx).close())
    idx = z.Index.build(data, ctx=ctx)
    pts = idx.points
    nwin = int(((pts["window"] == 1) & (pts["out"] > 0)).sum())
    res["points"] = int(len(pts["out"]))
    res["index_bytes_memory"] = int(len(pts["out"]) * 24 + nwin * 32768)
    res["index_bytes_exported"] = len(idx.to_bytes())
    rng = random.Random(1)
    lat = []
    for _ in range(101):
        a = rng.randrange(size - 4096)
        t0 = time.perf_counter()
        got = idx.extract(data, a, 4096)
        lat.append(time.perf_counter() - t0)
        assert got == out[a:a + 4096]
    res["one_read_ms"] = statistics.median(lat[1:]) * 1e3
    offs = [rng.randrange(size - 4096) for _ in range(reads)]
    lens = [4096] * reads
    idx.extract_batch(data, offs, lens)
    t0 = time.perf_counter()
    got, goff, st = idx.extract_batch(data, offs, lens)
    dt = time.perf_counter() - t0
    assert (st == 0).all()
    for i in range(0, reads, 97):
        assert got[int(goff[i]):int(goff[i + 1])].tobytes() == out[offs[i]:offs[i] + 4096]
    res["batch_reads"] = reads
    res["batch_gibs"] = reads * 4096 / dt / 2 ** 30
    res["batch_h2d_bytes_per_read"] = ctx.timing()["h2d_bytes"] / reads
    whole = timed(lambda: idx.extract_batch(data, [0], [size]))
    assert idx.extract(data, 0, size) == out
    res["whole_gibs"] = size / whole / 2 ** 30
    res["uncompress_gibs"] = size / res["uncompress_s"] / 2 ** 30
    idx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--small-mib", type=int, default=256)
    ap.add_argument("--reads", type=int, default=4096)
    ap.add_argument("--members", default="all")
    a = ap.parse_args()
    import zippy_b200 as z
    ctx = z.Context()
    info = card()
    big = corpus_text(a.mib)
    small = big[:a.small_mib << 20]
    rnd = np.random.default_rng(7).integers(0, 256, a.small_mib << 20, dtype=np.uint8).tobytes()
    members = [
        ("c2_text_level1_%dmib" % a.mib, lambda: z.compress(big, 1, z.dfGzip), big),
        ("c2_text_default_%dmib" % a.mib, lambda: z.compress(big, z.DefaultCompression, z.dfGzip), big),
        ("c2_text_python_zlib6_%dmib" % a.small_mib, lambda: zlib.compress(small, 6), small),
        ("random_level1_%dmib" % a.small_mib, lambda: z.compress(rnd, 1, z.dfGzip), rnd),
    ]
    for name, make, out in members:
        if a.members != "all" and not any(k in name for k in a.members.split(",")):
            continue
        r = measure(z, ctx, name, make(), out, a.reads)
        r["gpu"], r["power_limit"] = info
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
