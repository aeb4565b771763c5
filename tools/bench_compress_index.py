"""Cost of an index written while compressing (zb200_compress_batch_index / _device_index), on one GPU.

  python tools/bench_compress_index.py [--runs 5] [--out RESULT.json]

Workloads, each timed as medians of runs that alternate the variants:
  * 1 GiB of C2 text (the BASELINE text corpus repeated), one gzip member, levels 1 and Default, device-resident
    input and output: compress alone, compress with an index (span 1 MiB), and compress + Index.build of the member;
  * C2: 65 536 x 64 KiB text members, level 1, gzip, device-resident, span 1 MiB: compress alone and with indexes;
  * the exported index size of the 1 GiB member.
Every run checks that the members with and without an index are the same bytes (sha256).  Per workload it also
times the C call with an index alone (no Python Index objects) and lists, from torch.profiler in a run of its own, the
device time of that call by kernel and copy."""
import argparse
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    a = ap.parse_args()
    import torch
    import zippy_b200 as z
    from tests import util
    ctx = z.Context()
    T = util.text_corpus(util.load_corpus())
    big = (T * ((1 << 30) // len(T) + 1))[:1 << 30]
    c2 = b"".join(util.c2_block(T, i) for i in range(65536))
    gpu = torch.cuda.get_device_name(0)
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the measurement still stands; the power limit is then reported as unknown
        smi = "unknown (%s)" % e
    res = {"gpu": gpu, "power_limit_and_max_sm_clock": smi, "runs": a.runs, "results": {}}

    def device_case(name, data, offsets, level, with_build):
        d_src = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
        n = len(offsets) - 1
        cap = int(sum(z._native.lib().zb200_compress_bound(int(offsets[i + 1] - offsets[i]), 2) + 64
                      for i in range(n))) + 4096 if n < 4096 else int(len(data) * 1.01) + 64 * n + (1 << 20)
        d_dst = torch.empty(cap, dtype=torch.uint8, device="cuda")
        times = {"plain": [], "index": []}
        if with_build:
            times["plain+build"] = []
        digests, isize = set(), None
        for r in range(a.runs + 1):  # run 0 warms up
            for v in (["plain", "index"] if r % 2 == 0 else ["index", "plain"]):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if v == "plain":
                    oo = ctx.compress_batch_device(d_src.data_ptr(), offsets, level, z.dfGzip, d_dst.data_ptr(), cap)
                else:
                    oo, idx = ctx.compress_batch_device(d_src.data_ptr(), offsets, level, z.dfGzip, d_dst.data_ptr(),
                                                        cap, index_span=1 << 20)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                digests.add(hashlib.sha256(d_dst[:int(oo[-1])].cpu().numpy().tobytes()).hexdigest())
                if v == "index":
                    if isize is None:
                        isize = sum(len(x.to_bytes()) for x in idx[:4]) if n > 1 else len(idx[0].to_bytes())
                    for x in idx:
                        x.close()
                if r:
                    times[v].append(dt)
                if v == "plain" and with_build:
                    member = d_dst[:int(oo[-1])].cpu().numpy()
                    t1 = time.perf_counter()
                    b = z.Index.build(member, z.dfGzip, 1 << 20, ctx=ctx)
                    tb = time.perf_counter() - t1
                    b.close()
                    if r:
                        times["plain+build"].append(dt + tb)
        assert len(digests) == 1, "the members with and without an index differ"
        # where the time of the call with an index goes: the C call alone (no Python Index objects), and its
        # kernels and copies from torch.profiler in a run of their own
        L = z._native.lib()
        offs = np.ascontiguousarray(offsets, dtype=np.uint64)
        oo = np.zeros(n + 1, dtype=np.uint64)
        hs = (ctypes.c_void_p * n)()
        c_times = []
        for r in range(a.runs + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rc = L.zb200_compress_batch_device_index(ctx._h, d_src.data_ptr(), offs.ctypes.data, n, level, z.dfGzip,
                                                     None, d_dst.data_ptr(), cap, oo.ctypes.data, None, 1 << 20, hs)
            dt = time.perf_counter() - t0
            assert rc == 0
            for i in range(n):
                L.zb200_index_free(hs[i])
            if r:
                c_times.append(dt)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            L.zb200_compress_batch_device_index(ctx._h, d_src.data_ptr(), offs.ctypes.data, n, level, z.dfGzip, None,
                                                d_dst.data_ptr(), cap, oo.ctypes.data, None, 1 << 20, hs)
            torch.cuda.synchronize()
        for i in range(n):
            L.zb200_index_free(hs[i])
        print(prof.key_averages().table(sort_by="device_time_total", row_limit=12), flush=True)
        dev = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                key = "k_index_rec" if "k_index_rec" in e.name else "k_gather" if "k_gather" in e.name else \
                    "memcpy" if "emcpy" in e.name else "memset" if "emset" in e.name else "other kernels"
                dev[key] = dev.get(key, 0.0) + e.device_time_total / 1e3
        med = {k: sorted(v)[len(v) // 2] * 1e3 for k, v in times.items()}
        med["index, C call only"] = sorted(c_times)[len(c_times) // 2] * 1e3
        res["results"][name] = {"median_ms": med, "index_bytes": isize,
                                "overhead_pct": 100.0 * (med["index"] / med["plain"] - 1.0),
                                "index_call_device_ms": dev}
        print(name, json.dumps(res["results"][name]), flush=True)

    device_case("1GiB-level1", big, [0, len(big)], 1, True)
    device_case("1GiB-default", big, [0, len(big)], -1, True)
    device_case("C2-65536x64KiB-level1", c2, [i * 65536 for i in range(65537)], 1, False)
    print("RESULT " + json.dumps(res), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
