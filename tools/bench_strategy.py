"""Compression strategies on device-resident batches of 64 KiB members: for each input class, strategy and level
(1, Default) the input GiB/s of a whole compress_batch_device call, the k_lz* kernel time (zb200_last_timing's lz_ms,
scaled to the batch) and the compressed ratio, with zlib's ratio under the same strategy on a CPU sample.  The card
name and power limit are read in the same run.

Usage: python tools/bench_strategy.py [--members 65536] [--repeats 3] [--sample 64] [--out FILE]"""
import argparse
import json
import os
import random
import subprocess
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import zippy_b200 as z  # noqa: E402
from tests import util  # noqa: E402

SIZE = 65536
STRATEGIES = {"default": z.StrategyDefault, "filtered": z.StrategyFiltered, "huffman_only": z.StrategyHuffmanOnly,
              "rle": z.StrategyRle, "fixed": z.StrategyFixed}
ZLIB_STRATEGY = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman_only": zlib.Z_HUFFMAN_ONLY,
                 "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}


def classes(n, torch):
    """-> {name: device uint8 tensor of n x 64 KiB members}"""
    T = util.text_corpus(util.load_corpus())
    out = {}
    # C2: text blocks; the distinct blocks repeat to fill the batch
    uniq = min(n, 4096)
    c2 = np.frombuffer(b"".join(util.c2_block(T, i) for i in range(uniq)), dtype=np.uint8)
    c2 = torch.from_numpy(np.tile(c2, -(-n // uniq))[:n * SIZE].copy()).cuda()
    out["c2_text"] = c2
    # C5 classes: seeded short runs, random bytes
    rng = random.Random(5)
    runs = bytearray()
    while len(runs) < uniq * SIZE:
        runs += bytes([rng.choice(b"abcd")]) * rng.randint(1, 8)
    r = np.frombuffer(bytes(runs[:uniq * SIZE]), dtype=np.uint8)
    out["c5_runs"] = torch.from_numpy(np.tile(r, -(-n // uniq))[:n * SIZE].copy()).cuda()
    g = torch.Generator(device="cuda").manual_seed(7)
    out["c5_random"] = torch.randint(0, 256, (n * SIZE,), device="cuda", dtype=torch.uint8, generator=g)
    v = torch.randn(n * SIZE // 2, device="cuda", generator=g)
    keep = torch.rand(v.numel(), device="cuda", generator=g) < 0.05
    out["sparse_fp16"] = torch.where(keep, v, torch.zeros_like(v)).to(torch.float16).view(torch.uint8)
    out["zeros"] = torch.zeros(n * SIZE, device="cuda", dtype=torch.uint8)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", type=int, default=65536)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--sample", type=int, default=64, help="members compressed by zlib on the CPU")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    n = a.members
    offs = np.arange(n + 1, dtype=np.uint64) * SIZE
    L = z._native.lib()
    cap = int(L.zb200_compress_bound(SIZE, z.dfGzip)) * n
    d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    ctx = z.Context()
    rows = []
    for cname, src in classes(n, torch).items():
        sample = src[:a.sample * SIZE].cpu().numpy().tobytes()
        for sname, strategy in STRATEGIES.items():
            for level in (1, -1):
                ctx.compress_batch_device(src.data_ptr(), offs, level, z.dfGzip, d_dst.data_ptr(), cap,
                                          strategy=strategy)   # warm-up
                best, lz = None, None
                for _ in range(a.repeats):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    oo = ctx.compress_batch_device(src.data_ptr(), offs, level, z.dfGzip, d_dst.data_ptr(), cap,
                                                   strategy=strategy)
                    dt = time.perf_counter() - t0
                    t = ctx.timing()
                    if best is None or dt < best:
                        best = dt
                        lz = t["lz_ms"]   # timed on the first launch group, scaled to the batch by chunk count
                zl = 0
                for i in range(a.sample):
                    c = zlib.compressobj(6 if level == -1 else level, zlib.DEFLATED, 31, 8, ZLIB_STRATEGY[sname])
                    zl += len(c.compress(sample[i * SIZE:(i + 1) * SIZE]) + c.flush())
                rows.append({"class": cname, "strategy": sname, "level": level,
                             "gib_s": n * SIZE / best / 2 ** 30, "call_ms": best * 1e3, "lz_ms": lz,
                             "ratio": int(oo[-1]) / (n * SIZE), "zlib_ratio_sample": zl / (a.sample * SIZE)})
                r = rows[-1]
                print("%-12s %-13s %2d  %7.2f GiB/s  call %8.2f ms  k_lz* %7.2f ms  ratio %.4f  zlib %.4f"
                      % (cname, sname, level, r["gib_s"], r["call_ms"], r["lz_ms"], r["ratio"],
                         r["zlib_ratio_sample"]), flush=True)
    res = {"gpu": smi, "members": n, "member_bytes": SIZE, "rows": rows}
    if a.out:
        json.dump(res, open(a.out, "w"), indent=1)
    print(json.dumps({"gpu": smi, "members": n}))


if __name__ == "__main__":
    main()
