"""Per-member preset dictionaries (zb200_*_dicts): what one call with a dictionary table costs.

Batches of --n C2-text messages of 1 KiB and 4 KiB (slices of the SURVEY 8(d) text at seeded offsets), Default level,
zlib, three tables:
* k = 1: one 32 KiB dictionary shared by every message (dictionaries=[d] * n);
* k = 64: 64 tenant dictionaries of 32 KiB, message i against tenant i % 64, against 64 _dict calls over the same
  members (one per tenant);
* k = n: every message against the 32 KiB of text in front of it (RFC 7692 context takeover), distinct per message.
For each: compress and decode host-to-host time, the device kernel time (zb200_last_timing) and the compressed total
against zlib level 6 with the same zdicts (every 8th message).  For k = n also the time of one upload of the table's
bytes alone (a pageable host-to-device copy of the same size), the part of the call that kernel time does not show.
Times are medians of --reps runs after a warm-up.  Prints the card's name and power limit first.

    python tools/bench_dictionaries.py [--reps 3] [--n 65536] [--tables k=1,k=64,k=n]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def med(f, reps):
    f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = f()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=65536)
    ap.add_argument("--tables", default="k=1,k=64,k=n", help="the tables to run, comma-separated")
    args = ap.parse_args()
    import torch
    import zippy_b200 as z
    from tests import util
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    T = util.text_corpus(util.load_corpus())
    tarr = np.frombuffer(T, np.uint8)
    ctx = z.Context()
    rng = np.random.default_rng(0xD1C75)
    n, level = args.n, z.DefaultCompression
    tenants = [T[o:o + 32768] for o in rng.integers(0, len(T) - 32768, 64)]
    for size in (1024, 4096):
        starts = rng.integers(32768, len(T) - size, n)
        base = np.concatenate([tarr[s:s + size] for s in starts])
        offs = np.arange(n + 1, dtype=np.uint64) * size
        tables = {"k=1": [tenants[0]] * n, "k=64": [tenants[i % 64] for i in range(n)],
                  "k=n": [T[s - 32768:s] for s in starts]}
        for name, dl in tables.items():
            if name not in args.tables.split(","):
                continue
            tc, (out, oo) = med(lambda: ctx.compress_batch(base, offs, level, z.dfZlib, dictionaries=dl), args.reps)
            tm = ctx.timing()
            kc = tm["lz_ms"] + tm["huff_ms"] + tm["scan_ms"] + tm["pack_ms"]
            td, res = med(lambda: ctx.uncompress_batch(out, oo, z.dfZlib, dictionaries=dl), args.reps)
            tmu = ctx.timing()
            assert (res[3] == 0).all() and np.array_equal(res[0], base)
            zl = ours = 0
            for i in range(0, n, 8):
                co = zlib.compressobj(6, zlib.DEFLATED, 15, zdict=dl[i])
                zl += len(co.compress(bytes(base[i * size:(i + 1) * size])) + co.flush())
                ours += int(oo[i + 1] - oo[i])
            print("%d x %d B %-5s | compress %.1f ms (kernels %.2f ms) | decode %.1f ms (kernels %.2f ms) | "
                  "every 8th message %d B, zlib-6 with zdict %d B (%.3f)" %
                  (n, size, name, tc, kc, td, tmu["inflate_ms"] + tmu["verify_ms"], ours, zl, ours / zl))
            if name == "k=64":
                groups = [np.arange(j, n, 64) for j in range(64)]
                parts = [(np.concatenate([base[i * size:(i + 1) * size] for i in g]),
                          np.arange(len(g) + 1, dtype=np.uint64) * size) for g in groups]

                def comp64():
                    return [ctx.compress_batch(b, o, level, z.dfZlib, dictionary=tenants[j])
                            for j, (b, o) in enumerate(parts)]
                t64c, c64 = med(comp64, args.reps)
                t64d, _ = med(lambda: [ctx.uncompress_batch(c, co, z.dfZlib, dictionary=tenants[j])
                                       for j, (c, co) in enumerate(c64)], args.reps)
                print("    64 _dict calls over the same members: compress %.1f ms, decode %.1f ms" % (t64c, t64d))
            if name == "k=n":
                blob = np.concatenate([np.frombuffer(d, np.uint8) for d in dl])
                tu, _ = med(lambda: (torch.from_numpy(blob).cuda(), torch.cuda.synchronize()), args.reps)
                print("    one upload of the table's %.0f MiB alone: %.1f ms" % (blob.size / 2**20, tu))


if __name__ == "__main__":
    main()
