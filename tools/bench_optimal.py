"""Throughput and sizes of the optimal parse (optimal=True) against level 9, Default and Python's zlib -9.

Workloads: C2-like 64 KiB text blocks (tests/util.c2_block) and 64 KiB tiles of urls.10K.  Throughput is GiB/s of
input, device-resident (compress_batch_device, data already in HBM) and from host buffers (compress_batch), the
median of --reps timed calls after one warm-up call; sizes are the summed member bytes (zlib -9 computed on the CPU).
The GPU's name and power limit are recorded with the numbers.

    python tools/bench_optimal.py [--blocks 4096] [--reps 5] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import zlib

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zippy_b200 as z  # noqa: E402
from tests import util  # noqa: E402


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:   # the numbers still stand, without the card's description
        return "unknown (%s)" % e


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def run(name, blocks, reps):
    import torch
    ctx = z.default_context()
    base, offs = z._pack(blocks)
    nbytes = int(offs[-1])
    src = torch.from_numpy(np.frombuffer(bytes(base), dtype=np.uint8).copy()).cuda()
    cap = sum(int(z._native.lib().zb200_compress_bound(len(b), z.dfGzip)) + 64 for b in blocks) + 64
    dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    res = {"workload": name, "blocks": len(blocks), "input_bytes": nbytes}
    for label, kw in (("optimal", dict(optimal=True)), ("level9", {}), ("default", {})):
        level = z.DefaultCompression if label == "default" else 9
        oo = ctx.compress_batch_device(src.data_ptr(), offs, level, z.dfGzip, dst.data_ptr(), cap,
                                       fname_lens=[0] * len(blocks), **kw)
        res[label + "_bytes"] = int(oo[-1])
        dev = timed(lambda: ctx.compress_batch_device(src.data_ptr(), offs, level, z.dfGzip, dst.data_ptr(), cap,
                                                      fname_lens=[0] * len(blocks), **kw), reps)
        host = timed(lambda: ctx.compress_batch(base, offs, level, z.dfGzip, [0] * len(blocks), **kw), reps)
        res[label + "_device_gibs"] = nbytes / dev / 2 ** 30
        res[label + "_host_gibs"] = nbytes / host / 2 ** 30
    res["zlib9_bytes"] = sum(len(zlib.compress(b, 9)) + 12 for b in blocks)   # gzip framing: 18 bytes vs zlib's 6
    res["optimal_vs_level9"] = res["optimal_bytes"] / res["level9_bytes"]
    res["optimal_vs_zlib9"] = res["optimal_bytes"] / res["zlib9_bytes"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    corpus = util.load_corpus()
    T = util.text_corpus(corpus)
    urls = corpus["urls.10K"]
    tiles = [urls[(i * 65536) % (len(urls) - 65536):][:65536] for i in range(a.blocks)]
    out = {"gpu": gpu_info(), "results": [run("c2_text_64k", [util.c2_block(T, i) for i in range(a.blocks)], a.reps),
                                          run("urls_64k_tiles", tiles, a.reps)]}
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
