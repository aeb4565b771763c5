"""Streaming compression against the one-shot call on one large input in host memory.  Prints one JSON line per
level with the card's name and power limit.

    python tools/bench_compress_stream.py [--mib 1024] [--repeats 3] [--levels 1,-1] [--thresholds 16,64,256]

The input is the seeded C2-style text corpus (BASELINE config 2: 64 KiB windows of the test corpus at seeded
offsets, tests/util.c2_block), --mib MiB of it.  For each level, alternating in one process, median of --repeats
after one warm-up round:
- one_shot: Context.compress_batch of the whole input (one member);
- stream_<piece>: a CompressStream fed writes of 64 KiB, 1 MiB, 64 MiB and 256 MiB, on a context with the
  built-in batching threshold;
- batch<T>MiB_1MiB: the 1 MiB feed on contexts whose threshold (ZB200_STREAM_BATCH_BYTES) is T MiB: what the
  choice of the built-in threshold costs or saves.
Each variant reports GiB/s of input (host clock around the calls; every call returns with its output in host
memory) and the kernel launches it made (zb200_last_timing, summed over its calls).  Every variant's output is
compared with the one-shot member."""
import argparse
import hashlib
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_ziparchive import card  # noqa: E402


def corpus_text(mib):
    from tests import util
    T = util.text_corpus(util.load_corpus())
    return b"".join(util.c2_block(T, i) for i in range(mib * 16))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--levels", default="1,-1")
    ap.add_argument("--thresholds", default="16,64,256", help="MiB; batching thresholds tried with 1 MiB writes")
    a = ap.parse_args()
    import zippy_b200 as z
    data = corpus_text(a.mib)
    base, offs = z._pack([data])
    ctx = z.Context()
    tctx = {}
    for t in (int(x) for x in a.thresholds.split(",") if x):
        os.environ["ZB200_STREAM_BATCH_BYTES"] = str(t << 20)
        tctx[t] = z.Context()
    os.environ.pop("ZB200_STREAM_BATCH_BYTES", None)
    name, limit = card()

    def one_shot(level):
        out, oo = ctx.compress_batch(base, offs, level, z.dfGzip, [0])
        return [out[:int(oo[1])].tobytes()], ctx.timing()["kernel_launches"]

    def stream(c, piece):
        def run(level):
            outs, launches = [], 0
            with z.CompressStream(level, z.dfGzip, 0, c) as s:
                for i in range(0, len(data), piece):
                    outs.append(s.write(data[i:i + piece]))
                    launches += c.timing()["kernel_launches"]
                outs.append(s.finish())
                launches += c.timing()["kernel_launches"]
            return outs, launches
        return run

    variants = {"one_shot": one_shot}
    for piece in (64 << 10, 1 << 20, 64 << 20, 256 << 20):
        label = "%dKiB" % (piece >> 10) if piece < (1 << 20) else "%dMiB" % (piece >> 20)
        variants["stream_" + label] = stream(ctx, piece)
    for t, c in tctx.items():
        variants["batch%dMiB_1MiB" % t] = stream(c, 1 << 20)

    for level in (int(x) for x in a.levels.split(",")):
        times = {k: [] for k in variants}
        launches, digest = {}, {}
        for r in range(a.repeats + 1):
            for k, f in variants.items():
                t0 = time.perf_counter()
                outs, nl = f(level)
                dt = time.perf_counter() - t0
                if r:
                    times[k].append(dt)
                launches[k] = nl
                h = hashlib.sha256()
                for o in outs:
                    h.update(o)
                digest[k] = h.hexdigest()
        res = {"level": level, "input_gib": len(data) / (1 << 30), "card": name, "power_limit": limit,
               "same_bytes_as_one_shot": all(d == digest["one_shot"] for d in digest.values())}
        for k in variants:
            res[k] = {"gib_s": round(len(data) / (1 << 30) / statistics.median(times[k]), 3),
                      "kernel_launches": launches[k]}
        print(json.dumps(res), flush=True)
    for c in [ctx] + list(tctx.values()):
        c.close()


if __name__ == "__main__":
    main()
