"""Window sizes on device-resident batches of 64 KiB text members (C2 blocks): for each level (1, 6, 9) and window
(9, 12, 15) the k_lz* kernel time (zb200_last_timing's lz_ms), the input GiB/s of a whole compress_batch_device call
and the compressed ratio, with zlib's ratio at the same level and window on a CPU sample.  The card name and power
limit are read in the same run.

Usage: python tools/bench_window.py [--members 16384] [--repeats 5] [--sample 64] [--out FILE]"""
import argparse
import json
import os
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", type=int, default=16384)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--sample", type=int, default=64, help="members compressed by zlib on the CPU")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    n = a.members
    T = util.text_corpus(util.load_corpus())
    uniq = min(n, 4096)
    c2 = np.frombuffer(b"".join(util.c2_block(T, i) for i in range(uniq)), dtype=np.uint8)
    src = torch.from_numpy(np.tile(c2, -(-n // uniq))[:n * SIZE].copy()).cuda()
    sample = src[:a.sample * SIZE].cpu().numpy().tobytes()
    offs = np.arange(n + 1, dtype=np.uint64) * SIZE
    cap = int(z._native.lib().zb200_compress_bound(SIZE, z.dfGzip)) * n
    d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    ctx = z.Context()
    rows = []
    for level in (1, 6, 9):
        for wb in (9, 12, 15):
            ctx.compress_batch_device(src.data_ptr(), offs, level, z.dfGzip, d_dst.data_ptr(), cap,
                                      window_bits=wb)   # warm-up
            best, lz = None, None
            for _ in range(a.repeats):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                oo = ctx.compress_batch_device(src.data_ptr(), offs, level, z.dfGzip, d_dst.data_ptr(), cap,
                                               window_bits=wb)
                dt = time.perf_counter() - t0
                t = ctx.timing()
                if best is None or dt < best:
                    best, lz = dt, t["lz_ms"]
            zl = 0
            for i in range(a.sample):
                c = zlib.compressobj(level, zlib.DEFLATED, 16 + wb)
                zl += len(c.compress(sample[i * SIZE:(i + 1) * SIZE]) + c.flush())
            rows.append({"level": level, "window_bits": wb, "gib_s": n * SIZE / best / 2 ** 30, "call_ms": best * 1e3,
                         "lz_ms": lz, "ratio": int(oo[-1]) / (n * SIZE), "zlib_ratio_sample": zl / (a.sample * SIZE)})
            r = rows[-1]
            print("level %d  n %2d  %7.2f GiB/s  call %8.2f ms  k_lz* %7.2f ms  ratio %.4f  zlib %.4f"
                  % (level, wb, r["gib_s"], r["call_ms"], r["lz_ms"], r["ratio"], r["zlib_ratio_sample"]), flush=True)
    ctx.close()
    res = {"gpu": smi, "members": n, "member_bytes": SIZE, "rows": rows}
    if a.out:
        json.dump(res, open(a.out, "w"), indent=1)
    print(json.dumps({"gpu": smi, "members": n}))


if __name__ == "__main__":
    main()
