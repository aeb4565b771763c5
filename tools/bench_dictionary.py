"""Preset dictionaries on the GPU: what a shared 32 KiB dictionary costs and saves.

* Batches of 65 536 x 4 KiB and 65 536 x 1 KiB C2-text messages (slices of the SURVEY 8(d) text at seeded
  offsets) with a 32 KiB dictionary taken from the same text, at levels 1 (control: no history), Default and 9:
  compress and uncompress device time (zb200_last_timing) and host-to-host time, each against the same batch without
  the dictionary, and the compressed total against zlib level 6 with the same zdict (on every 8th message).
* The message sets of the feature's motivation (urls.10K, alice29.txt, html_x_4: the first 32 KiB as dictionary,
  1 KiB messages after it): totals at Default against zlib level 6 with that zdict.
* One 1 GiB Default-level zlib member through uncompress(dictionary=) against uncompress of the member without one.
Times are medians of --reps runs after a warm-up.  Prints the card's name and power limit first.

    python tools/bench_dictionary.py [--reps 3] [--n 65536]
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
    return statistics.median(ts), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=65536)
    args = ap.parse_args()
    import zippy_b200 as z
    from tests import util
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    corpus = util.load_corpus()
    T = util.text_corpus(corpus)
    tarr = np.frombuffer(T, np.uint8)
    d = T[:32768]
    ctx = z.Context()
    rng = np.random.default_rng(0xD1C7)
    for size in (4096, 1024):
        starts = rng.integers(32768, len(T) - size, args.n)
        base = np.concatenate([tarr[s:s + size] for s in starts])
        offs = np.arange(args.n + 1, dtype=np.uint64) * size
        for level in (1, -1, 9):
            row = {}
            for tag, dd in (("plain", None), ("dict", d)):
                t, (out, oo) = med(lambda: ctx.compress_batch(base, offs, level, z.dfZlib, dictionary=dd), args.reps)
                tm = ctx.timing()
                dev_c = tm["lz_ms"] + tm["huff_ms"] + tm["scan_ms"] + tm["pack_ms"]
                lz = tm["lz_ms"]
                tu, res = med(lambda: ctx.uncompress_batch(out, oo, z.dfZlib, dictionary=dd), args.reps)
                tmu = ctx.timing()
                assert (res[3] == 0).all() and np.array_equal(res[0], base)
                row[tag] = (int(oo[-1]), t * 1e3, dev_c, lz, tu * 1e3, tmu["inflate_ms"] + tmu["verify_ms"])
            zl = 0
            for i in range(0, args.n, 8):
                co = zlib.compressobj(6, zlib.DEFLATED, 15, zdict=d)
                zl += len(co.compress(bytes(base[i * size:(i + 1) * size])) + co.flush())
            pl, dc = row["plain"], row["dict"]
            print("%d x %d B level %2d | size %d -> %d (%.3f)  | compress host %.1f -> %.1f ms, device %.2f -> %.2f ms "
                  "(k_lz %.2f -> %.2f) | uncompress host %.1f -> %.1f ms, device %.2f -> %.2f ms" %
                  (args.n, size, level, pl[0], dc[0], dc[0] / pl[0], pl[1], dc[1], pl[2], dc[2], pl[3], dc[3], pl[4],
                   dc[4], pl[5], dc[5]))
            # zlib-6 with zdict on every 8th message, against this library's dictionary members of the same messages
            sample = [bytes(base[i * size:(i + 1) * size]) for i in range(0, args.n, 8)]
            ours = sum(map(len, z.compress_batch(sample, level, z.dfZlib, dictionary=d)))
            print("    every 8th message: this library %d, zlib-6 with zdict %d (%.3f)" % (ours, zl, ours / zl))
    for name in ("urls.10K", "alice29.txt", "html_x_4"):
        data = corpus[name]
        dd, msgs = data[:32768], [data[i:i + 1024] for i in range(32768, len(data) - 1023, 1024)]
        zl = 0
        for m in msgs:
            co = zlib.compressobj(6, zlib.DEFLATED, 15, zdict=dd)
            zl += len(co.compress(m) + co.flush())
        a = sum(map(len, z.compress_batch(msgs, -1, z.dfZlib)))
        b = sum(map(len, z.compress_batch(msgs, -1, z.dfZlib, dictionary=dd)))
        print("%s, %d x 1 KiB, Default: without %d, with %d, zlib-6 with zdict %d: %.3f x zlib" %
              (name, len(msgs), a, b, zl, b / zl))
    big = (T * (1 + (1 << 30) // len(T)))[:1 << 30]
    c_plain = z.compress(big, -1, z.dfZlib)
    c_dict = z.compress(big, -1, z.dfZlib, dictionary=d)
    t0, r0 = med(lambda: z.uncompress(c_plain, z.dfZlib), args.reps)
    t1, r1 = med(lambda: z.uncompress(c_dict, z.dfZlib, dictionary=d), args.reps)
    assert r0 == big and r1 == big
    print("1 GiB member: uncompress %.1f ms (%.2f GiB/s), uncompress(dictionary=) %.1f ms (%.2f GiB/s)" %
          (t0 * 1e3, 1 / t0, t1 * 1e3, 1 / t1))


if __name__ == "__main__":
    main()
