"""Throughput and sizes of rsyncable compression (rsyncable=True) against the plain 64 KiB grid.

Workloads: C2-like 64 KiB text blocks (tests/util.c2_block), one 1 GiB text member (the text corpus repeated) and
256 MiB of seeded random bytes, at level 1 and Default.  Throughput is GiB/s of input, device-resident
(compress_batch_device, data already in HBM) and from host buffers (compress_batch), the median of --reps timed calls
after one warm-up call; sizes are the summed member bytes.  For the 1 GiB member, also the uncompress time of the
rsyncable and the plain member.  --profile instead times the chunk-map kernels (k_rsync_cand, k_rsync_starts) with
torch.profiler over a 4 GiB text member, in a run of its own.  The GPU's name and power limit are recorded with the
numbers.

    python tools/bench_rsyncable.py [--blocks 16384] [--reps 3] [--json out.json] [--profile]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import zippy_b200 as z  # noqa: E402
from tests import util  # noqa: E402
from tools.bench_optimal import gpu_info, timed  # noqa: E402


def run(name, blocks, reps, uncompress=False):
    import torch
    ctx = z.default_context()
    L = z._native.lib()
    base, offs = z._pack(blocks)
    nbytes = int(offs[-1])
    src = torch.from_numpy(np.frombuffer(bytes(base), dtype=np.uint8).copy()).cuda()
    cap = sum(int(L.zb200_compress_bound_rsyncable(len(b), z.dfGzip)) + 64 for b in blocks) + 64
    dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
    fl = [0] * len(blocks)
    res = {"workload": name, "blocks": len(blocks), "input_bytes": nbytes}
    for level, lname in ((1, "l1"), (z.DefaultCompression, "default")):
        for rs in (False, True):
            label = lname + ("_rsync" if rs else "_plain")
            oo = ctx.compress_batch_device(src.data_ptr(), offs, level, z.dfGzip, dst.data_ptr(), cap, fname_lens=fl,
                                           rsyncable=rs)
            res[label + "_bytes"] = int(oo[-1])
            dev = timed(lambda: ctx.compress_batch_device(src.data_ptr(), offs, level, z.dfGzip, dst.data_ptr(), cap,
                                                          fname_lens=fl, rsyncable=rs), reps)
            host = timed(lambda: ctx.compress_batch(base, offs, level, z.dfGzip, fl, rsyncable=rs), reps)
            res[label + "_device_gibs"] = nbytes / dev / 2 ** 30
            res[label + "_host_gibs"] = nbytes / host / 2 ** 30
            if uncompress:
                member = dst[:int(oo[1])].cpu().numpy().tobytes()
                assert len(z.uncompress(member)) == nbytes
                res[label + "_uncompress_ms"] = 1e3 * timed(lambda: z.uncompress(member), reps)
        res[lname + "_size_ratio"] = res[lname + "_rsync_bytes"] / res[lname + "_plain_bytes"]
    res["chunks_plain"] = sum(max(1, -(-len(b) // 65536)) for b in blocks)
    res["chunks_rsync"] = int(sum(len(c) for c in ctx.rsyncable_chunks(base, offs)))
    return res


def profile(nbytes):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    T = util.text_corpus(util.load_corpus())
    buf = np.frombuffer((T * (nbytes // len(T) + 1))[:nbytes], dtype=np.uint8)
    ctx = z.default_context()
    ctx.rsyncable_chunks(buf, [0, nbytes])      # warm-up: staging buffers and modules
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(3):
            ctx.rsyncable_chunks(buf, [0, nbytes])
        torch.cuda.synchronize()
    out = {}
    for e in p.key_averages():
        if "k_rsync" in e.key:
            out[e.key] = {"calls": e.count, "ms_per_call": e.device_time_total / e.count / 1e3}
    return {"gpu": gpu_info(), "input_bytes": nbytes, "kernels": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=16384)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if a.profile:
        out = profile(4 << 30)
    else:
        corpus = util.load_corpus()
        T = util.text_corpus(corpus)
        big = (T * ((1 << 30) // len(T) + 1))[:1 << 30]
        rnd = np.random.default_rng(1).integers(0, 256, 256 << 20, dtype=np.uint8).tobytes()
        out = {"gpu": gpu_info(), "results": [
            run("c2_text_64k", [util.c2_block(T, i) for i in range(a.blocks)], a.reps),
            run("text_1gib_member", [big], a.reps, uncompress=True),
            run("random_256mib_member", [rnd], a.reps)]}
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
