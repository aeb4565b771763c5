#!/usr/bin/env python3
"""Where a compress kernel's cycles go: per-stage clock64() shares of the level-1 parse (k_lz<1>) or of the
codebook builder (k_huff).

    python tools/lz1_stages.py [--kernel lz1|huff] [--workload c2|c5] [--blocks N] [--lib PATH]

Builds the library with -DZB_LZ1_STAGE_CLOCKS=1 (--kernel lz1, the default) or -DZB_HUFF_STAGE_CLOCKS=1
(--kernel huff) into a temporary directory (or loads --lib, a library built that way), compresses bench.py's
C2 batch (N x 64 KiB text blocks) or C5 batch (N x 64 KiB mixed-entropy blocks), level 1, gzip,
device-resident, once to warm up and once measured, and prints each stage's share of the cycles that lane 0
of every warp spent, next to the card's name and power limit and the measured launch's lz_ms / huff_ms.  The
instrumented kernel is slower than the shipped one (each stage boundary reads the clock); the shares are what
it is for.  Nothing is written into the repository tree.
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

# the order of the LZS_* enum in zb_deflate.cu.  The window loop is a one-window pipeline: "probe" counts only the
# probes that start it (a piece's first window, one after skipped windows or a drain); the other windows' probes,
# 4-byte checks and first extension steps run inside the previous window's selection and count there
LZ1_STAGE_NAMES = ["wait + table load", "checksum", "clear + pre-seed", "probe (pipeline start)", "verify + extend",
                   "select + next window's probe", "batch pass", "phase barrier + epilogue"]
# the order of the HWS_* enum in zb_huff_warp.cuh
HUFF_STAGE_NAMES = ["sum", "sort", "Moffat-Katajainen", "limit", "assign + sums", "RLE", "code-length code",
                    "choice + header", "canonical codes", "bit ranges", "store"]
KERNELS = {"lz1": ("-DZB_LZ1_STAGE_CLOCKS=1", "zb200_lz1_stage_clocks", LZ1_STAGE_NAMES, "lz_ms"),
           "huff": ("-DZB_HUFF_STAGE_CLOCKS=1", "zb200_huff_stage_clocks", HUFF_STAGE_NAMES, "huff_ms")}


def build_variant(out_dir, define):
    import __graft_entry__ as g
    lib = os.path.join(out_dir, "libzippy_b200.so")
    cmd = [os.environ.get("NVCC", "nvcc")] + g.NVCC_FLAGS + [define, "-o", lib] + \
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
    ap.add_argument("--kernel", default="lz1", choices=sorted(KERNELS))
    ap.add_argument("--workload", default="c2", choices=["c2", "c5"])
    ap.add_argument("--blocks", type=int, default=65536)
    ap.add_argument("--lib", default=None, help="a library already built with the kernel's stage-clock define")
    args = ap.parse_args()
    define, reader, names, figure = KERNELS[args.kernel]

    tmp = tempfile.mkdtemp(prefix="lz1_stages_")
    try:
        lib_path = args.lib or build_variant(tmp, define)
        import numpy as np
        import torch
        from zippy_b200 import _native
        _native.LIB_PATH = lib_path          # before the first load
        import zippy_b200 as z
        import bench
        L = _native.lib()
        read_clocks = getattr(L, reader)
        read_clocks.restype = ctypes.c_int
        read_clocks.argtypes = [ctypes.c_void_p]

        dev = torch.device("cuda", 0)
        torch.cuda.set_device(dev)
        gen = bench.gen_c2 if args.workload == "c2" else bench.gen_c5
        d_src, _ = gen(types.SimpleNamespace(torch=torch, dev=dev), args.blocks, 0)
        offs = np.arange(args.blocks + 1, dtype=np.uint64) * bench.BLOCK
        cap = args.blocks * (bench.BLOCK + 96) + 4096
        d_dst = torch.empty(cap, dtype=torch.uint8, device=dev)
        ctx = z.Context(0)
        clk = (ctypes.c_ulonglong * len(names))()
        ctx.compress_batch_device(d_src.data_ptr(), offs, z.BestSpeed, z.dfGzip, d_dst.data_ptr(), cap)
        torch.cuda.synchronize()
        if read_clocks(ctypes.byref(clk)) != 0:   # zeroes the counters
            raise RuntimeError("reading the stage clocks failed")
        oo = ctx.compress_batch_device(d_src.data_ptr(), offs, z.BestSpeed, z.dfGzip, d_dst.data_ptr(), cap)
        torch.cuda.synchronize()
        ms = ctx.timing()[figure]
        if read_clocks(ctypes.byref(clk)) != 0:
            raise RuntimeError("reading the stage clocks failed")
        total = float(sum(clk))
        shares = {n: clk[i] / total for i, n in enumerate(names)}
        out = {"gpu": gpu_info(), "kernel": args.kernel, "workload": args.workload, "blocks": args.blocks,
               figure + "_instrumented": ms, "comp_bytes": int(oo[-1]),
               "cycles": {n: int(clk[i]) for i, n in enumerate(names)}, "shares": shares}
        print("%s, power limit %s; %s, instrumented %s: %.2f ms" % (out["gpu"]["name"], out["gpu"]["power_limit"],
                                                                    args.workload.upper(), args.kernel, ms))
        for n in names:
            print("  %-26s %6.1f %%" % (n, 100.0 * shares[n]))
        print(json.dumps(out))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
