#!/usr/bin/env python3
"""Where k_lz<1>'s cycles go: per-stage clock64() shares of the level-1 parse on C2.

    python tools/lz1_stages.py [--blocks N] [--lib PATH] [--keep DIR]

Builds the library with -DZB_LZ1_STAGE_CLOCKS=1 into a temporary directory (or loads --lib, a library
built that way), compresses bench.py's C2 batch (N x 64 KiB text blocks, level 1, gzip, device-resident)
once to warm up and once measured, and prints each stage's share of the cycles that lane 0 of every warp
spent, next to the card's name and power limit and the measured launch's lz_ms.  The instrumented kernel
is slower than the shipped one (each stage boundary reads the clock); the shares are what it is for.
Nothing is written into the repository tree.
"""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# the order of the LZS_* enum in zb_deflate.cu
LZ1_STAGE_NAMES = ["wait + table load", "checksum", "clear + pre-seed", "probe", "verify + extend", "select",
                   "batch pass", "phase barrier + epilogue"]


def build_variant(out_dir):
    import __graft_entry__ as g
    lib = os.path.join(out_dir, "libzippy_b200.so")
    cmd = [os.environ.get("NVCC", "nvcc")] + g.NVCC_FLAGS + ["-DZB_LZ1_STAGE_CLOCKS=1", "-o", lib] + \
        [os.path.join(g.CSRC, s) for s in g.SOURCES]
    subprocess.check_call(cmd, cwd=g.CSRC)
    return lib


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": pl}
    except Exception as ex:  # the shares are still worth printing
        return {"name": None, "power_limit": None, "error": repr(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=65536)
    ap.add_argument("--lib", default=None, help="a library already built with -DZB_LZ1_STAGE_CLOCKS=1")
    args = ap.parse_args()

    tmp = tempfile.mkdtemp(prefix="lz1_stages_")
    try:
        lib_path = args.lib or build_variant(tmp)
        import numpy as np
        import torch
        from zippy_b200 import _native
        _native.LIB_PATH = lib_path          # before the first load
        import zippy_b200 as z
        import bench
        L = _native.lib()
        L.zb200_lz1_stage_clocks.restype = ctypes.c_int
        L.zb200_lz1_stage_clocks.argtypes = [ctypes.c_void_p]

        dev = torch.device("cuda", 0)
        torch.cuda.set_device(dev)
        d_src, _ = bench.gen_c2(types.SimpleNamespace(torch=torch, dev=dev), args.blocks, 0)
        offs = np.arange(args.blocks + 1, dtype=np.uint64) * bench.BLOCK
        cap = args.blocks * (bench.BLOCK + 96) + 4096
        d_dst = torch.empty(cap, dtype=torch.uint8, device=dev)
        ctx = z.Context(0)
        clk = (ctypes.c_ulonglong * len(LZ1_STAGE_NAMES))()
        ctx.compress_batch_device(d_src.data_ptr(), offs, z.BestSpeed, z.dfGzip, d_dst.data_ptr(), cap)
        torch.cuda.synchronize()
        if L.zb200_lz1_stage_clocks(ctypes.byref(clk)) != 0:   # zeroes the counters
            raise RuntimeError("reading the stage clocks failed")
        oo = ctx.compress_batch_device(d_src.data_ptr(), offs, z.BestSpeed, z.dfGzip, d_dst.data_ptr(), cap)
        torch.cuda.synchronize()
        lz_ms = ctx.timing()["lz_ms"]
        if L.zb200_lz1_stage_clocks(ctypes.byref(clk)) != 0:
            raise RuntimeError("reading the stage clocks failed")
        total = float(sum(clk))
        shares = {n: clk[i] / total for i, n in enumerate(LZ1_STAGE_NAMES)}
        out = {"gpu": gpu_info(), "blocks": args.blocks, "lz_ms_instrumented": lz_ms,
               "comp_bytes": int(oo[-1]), "cycles": {n: int(clk[i]) for i, n in enumerate(LZ1_STAGE_NAMES)},
               "shares": shares}
        print("%s, power limit %s; instrumented k_lz<1>: %.2f ms" % (out["gpu"]["name"], out["gpu"]["power_limit"], lz_ms))
        for n in LZ1_STAGE_NAMES:
            print("  %-26s %6.1f %%" % (n, 100.0 * shares[n]))
        print(json.dumps(out))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
