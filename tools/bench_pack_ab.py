#!/usr/bin/env python3
"""Where a C2 step's time goes, for one or more builds of the library: kernels, host plan, and the rest.

    python tools/bench_pack_ab.py LIB.so [MORE.so ...] [--runs 3] [--steps 5] [--blocks 65536]

C2 is bench.py's flagship: N x 64 KiB text blocks, level 1, gzip, inputs and outputs on the device, one launch group
per step.  Each run loads one library (through zippy_b200._native.LIB_PATH, before the first load) in a subprocess
of its own, compresses C2 `--warmup` times, then times `--steps` calls of compress_batch_device:
  - lz_ms, huff_ms, scan_ms, pack_ms: the library's CUDA-event kernel times (ctx.timing());
  - plan_ms: the library's host time from entry to the first kernel launch (0 for a build that does not report it);
  - step_ms: two events on the library's stream around the call, so it includes the time the GPU waits for the plan;
  - wall_ms: host clock around the call (it returns after a stream synchronise);
  - gap_ms: step_ms - plan_ms - the kernel times: copies, launch gaps and the event spans' edges.
With several builds they take turns, run after run, so a drift of the card's clocks falls on all of them alike.
Every run hashes (sha256) the complete C2 output, every member's bytes and offsets; the tool exits non-zero if any
run's digest differs from the first build's.  Prints the median and range over the runs of each figure (each run
contributes the median of its steps) with the card's name and power limit, then one JSON line.  Nothing is written
into the repository tree.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = ["lz_ms", "huff_ms", "scan_ms", "pack_ms"]
FIGURES = KERNELS + ["plan_ms", "step_ms", "wall_ms", "gap_ms"]


def child(args):
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    from zippy_b200 import _native
    _native.LIB_PATH = os.path.abspath(args.child)   # before the first load
    import zippy_b200 as z
    import bench

    n = args.blocks
    os.environ["ZB200_DEV_GROUP_CHUNKS"] = str(n)   # one launch group per step, as bench.py's C2
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    d_src, _ = bench.gen_c2(types.SimpleNamespace(torch=torch, dev=dev), n, 0)
    offs = np.arange(n + 1, dtype=np.uint64) * bench.BLOCK
    cap = n * (bench.BLOCK + 96) + 4096
    d_dst = torch.empty(cap, dtype=torch.uint8, device=dev)
    ctx = z.Context(0)
    stream = torch.cuda.current_stream()
    ctx.set_stream(stream.cuda_stream or ctx.LEGACY_DEFAULT_STREAM)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(max(1, args.warmup)):
        oo = ctx.compress_batch_device(d_src.data_ptr(), offs, z.BestSpeed, z.dfGzip, d_dst.data_ptr(), cap)
    torch.cuda.synchronize()
    per = {k: [] for k in FIGURES}
    for _ in range(args.steps):
        ev0.record(stream)
        t0 = time.perf_counter()
        oo = ctx.compress_batch_device(d_src.data_ptr(), offs, z.BestSpeed, z.dfGzip, d_dst.data_ptr(), cap)
        t1 = time.perf_counter()
        ev1.record(stream)
        torch.cuda.synchronize()
        tm = ctx.timing()
        for k in KERNELS + ["plan_ms"]:
            per[k].append(tm.get(k, 0.0))
        per["step_ms"].append(ev0.elapsed_time(ev1))
        per["wall_ms"].append((t1 - t0) * 1e3)
        per["gap_ms"].append(per["step_ms"][-1] - per["plan_ms"][-1] - sum(tm[k] for k in KERNELS))
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(oo, dtype=np.uint64).tobytes())
    total = int(oo[n])
    for s in range(0, total, 1 << 28):   # the complete output, in 256 MiB slices
        h.update(d_dst[s:min(total, s + (1 << 28))].cpu().numpy().tobytes())
    out = {k: float(np.median(v)) for k, v in per.items()}
    out.update(sha256=h.hexdigest(), comp_bytes=total, gib_s=n * bench.BLOCK / float(1 << 30) / (out["step_ms"] / 1e3))
    print("RESULT " + json.dumps(out))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": pl}
    except Exception as ex:
        return {"name": None, "power_limit": None, "error": repr(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="*", help="library paths; the first is the baseline")
    ap.add_argument("--runs", type=int, default=3, help="runs per build")
    ap.add_argument("--steps", type=int, default=5, help="timed steps per run")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--blocks", type=int, default=65536)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args)
        return
    if not args.libs:
        ap.error("give at least one library")
    import numpy as np
    libs = [os.path.abspath(p) for p in args.libs]
    runs = {p: [] for p in libs}
    for r in range(args.runs):
        for p in (libs if r % 2 == 0 else libs[::-1]):   # alternate the order too
            cmd = [sys.executable, os.path.abspath(__file__), "--child", p, "--blocks", str(args.blocks),
                   "--steps", str(args.steps), "--warmup", str(args.warmup)]
            res = subprocess.run(cmd, capture_output=True, text=True)
            line = [l for l in res.stdout.splitlines() if l.startswith("RESULT ")]
            if res.returncode != 0 or not line:
                sys.stderr.write(res.stdout[-4000:] + res.stderr[-4000:])
                raise SystemExit("run of %s failed (exit %d)" % (p, res.returncode))
            runs[p].append(json.loads(line[0][7:]))
    gpu = gpu_info()
    print("%s, power limit %s; C2 = %d x 64 KiB, level 1, gzip; %d runs x %d steps per build"
          % (gpu["name"], gpu["power_limit"], args.blocks, args.runs, args.steps))
    summary = {}
    ref = runs[libs[0]][0]["sha256"]
    same = True
    for p in libs:
        s = {k: {"median": float(np.median([x[k] for x in runs[p]])), "min": min(x[k] for x in runs[p]),
                 "max": max(x[k] for x in runs[p])} for k in FIGURES + ["gib_s"]}
        digests = sorted({x["sha256"] for x in runs[p]})
        s["sha256"] = digests
        s["comp_bytes"] = runs[p][0]["comp_bytes"]
        same = same and digests == [ref]
        summary[p] = s
        print(p)
        for k in FIGURES + ["gib_s"]:
            print("  %-8s median %9.3f  range %9.3f .. %9.3f" % (k, s[k]["median"], s[k]["min"], s[k]["max"]))
        print("  sha256   %s" % " ".join(digests))
    base = summary[libs[0]]
    for p in libs[1:]:
        for k in ("pack_ms", "plan_ms", "step_ms"):
            d = summary[p][k]["median"] - base[k]["median"]
            apart = summary[p][k]["max"] < base[k]["min"] or summary[p][k]["min"] > base[k]["max"]
            print("%s vs baseline: %s %+.3f ms, ranges %s" % (os.path.basename(p), k, d, "apart" if apart else "OVERLAP"))
    print(json.dumps({"gpu": gpu, "blocks": args.blocks, "runs": args.runs, "steps": args.steps,
                      "same_output": same, "builds": summary, "per_run": runs}))
    if not same:
        raise SystemExit("the builds' C2 outputs differ")


if __name__ == "__main__":
    main()
