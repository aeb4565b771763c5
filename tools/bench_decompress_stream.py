"""Streaming decompression against the one-shot decode on large members in host memory.  Prints one JSON line per
input with the card's name and power limit.

    python tools/bench_decompress_stream.py [--mib 1024] [--side-mib 256] [--repeats 3] [--thresholds 16,64,256]

Inputs (the C2-style text corpus: 64 KiB windows of the test corpus at seeded offsets, tests/util.c2_block):
- text_l1 / text_default: --mib MiB of it as one gzip member at level 1 / Default, written by compress_batch
  (this library's joints: the k_find_sync path);
- zlib6: --side-mib MiB of it as one zlib level-6 member written by Python's zlib (the k_find_blocks path);
- random_l1: --side-mib MiB of random bytes at level 1, stored chunks without joints (the open serial segment).
For each input, alternating in one process, median of --repeats after one warm-up round:
- one_shot: zb200_decode_begin / _finish of the whole member (Context.decode_one), pageable host memory to host;
- stream_<piece>: a DecompressStream fed writes of 64 KiB, 1 MiB and 64 MiB, reading after every write, on a
  context with the built-in batching threshold;
- batch<T>MiB_1MiB: the 1 MiB feed on contexts whose threshold (ZB200_DSTREAM_BATCH_BYTES) is T MiB.
Each variant reports GiB/s of output (host clock around the calls) and the kernel launches it made
(zb200_last_timing, summed over its calls).  Every variant's output is compared with the input."""
import argparse
import hashlib
import json
import os
import statistics
import sys
import time
import zlib

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
    ap.add_argument("--side-mib", type=int, default=256)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--thresholds", default="16,64,256", help="MiB; batching thresholds tried with 1 MiB writes")
    ap.add_argument("--inputs", default="text_l1,text_default,zlib6,random_l1")
    a = ap.parse_args()
    import zippy_b200 as z
    ctx = z.Context()
    tctx = {}
    for t in (int(x) for x in a.thresholds.split(",") if x):
        os.environ["ZB200_DSTREAM_BATCH_BYTES"] = str(t << 20)
        tctx[t] = z.Context()
    os.environ.pop("ZB200_DSTREAM_BATCH_BYTES", None)
    name, limit = card()
    text = corpus_text(a.mib)
    side = text[:a.side_mib << 20]

    def lib_member(data, level):
        base, offs = z._pack([data])
        out, oo = ctx.compress_batch(base, offs, level, z.dfGzip, [0])
        return out[:int(oo[1])].tobytes()

    makers = {"text_l1": lambda: (lib_member(text, 1), text),
              "text_default": lambda: (lib_member(text, -1), text),
              "zlib6": lambda: (zlib.compress(side, 6), side),
              "random_l1": lambda: ((lambda r: (lib_member(r, 1), r))(os.urandom(a.side_mib << 20)))}

    def one_shot(comp):
        return [ctx.decode_one(comp, z.dfDetect)], ctx.timing()["kernel_launches"]

    def stream(c, piece):
        def run(comp):
            outs, launches = [], 0
            with z.DecompressStream(z.dfDetect, c) as s:
                for i in range(0, len(comp), piece):
                    outs.append(s.write(comp[i:i + piece]))
                    launches += c.timing()["kernel_launches"]
                outs.append(s.finish())
                launches += c.timing()["kernel_launches"]
            return outs, launches
        return run

    variants = {"one_shot": one_shot}
    for piece in (64 << 10, 1 << 20, 64 << 20):
        label = "%dKiB" % (piece >> 10) if piece < (1 << 20) else "%dMiB" % (piece >> 20)
        variants["stream_" + label] = stream(ctx, piece)
    for t, c in tctx.items():
        variants["batch%dMiB_1MiB" % t] = stream(c, 1 << 20)

    for iname in a.inputs.split(","):
        comp, data = makers[iname]()
        want = hashlib.sha256(data).hexdigest()
        times = {k: [] for k in variants}
        launches, same = {}, {}
        for r in range(a.repeats + 1):
            for k, f in variants.items():
                t0 = time.perf_counter()
                outs, nl = f(comp)
                dt = time.perf_counter() - t0
                if r:
                    times[k].append(dt)
                launches[k] = nl
                h = hashlib.sha256()
                for o in outs:
                    h.update(o)
                same[k] = h.hexdigest() == want
                print("%s round %d %s: %.2f s" % (iname, r, k, dt), file=sys.stderr, flush=True)
        res = {"input": iname, "output_gib": len(data) / (1 << 30), "compressed_mib": round(len(comp) / (1 << 20), 1),
               "card": name, "power_limit": limit, "all_outputs_equal_input": all(same.values())}
        for k in variants:
            res[k] = {"gib_s": round(len(data) / (1 << 30) / statistics.median(times[k]), 3),
                      "kernel_launches": launches[k]}
        print(json.dumps(res), flush=True)
    for c in [ctx] + list(tctx.values()):
        c.close()


if __name__ == "__main__":
    main()
