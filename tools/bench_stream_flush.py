"""Flushed compress streams and drained decompress streams.  Prints one JSON line per measurement with the card's
name and power limit.

    python tools/bench_stream_flush.py [--mib 1024] [--repeats 3] [--levels 1,-1] [--messages 2000]

- latency: per-call time of CompressStream.flush and DecompressStream.drain for messages of 1 KiB and 64 KiB,
  each written and then flushed (the receiver writes what the flush emitted, then drains); median and 90th
  percentile over --messages messages of the C2 text, after 50 warm-up messages.  flush_ms includes the write of
  the message (which only buffers it).
- throughput: --mib MiB of the C2 text (tests/util.c2_block) compressed as one gzip member with a sync flush every
  1 MiB, every 64 MiB and never, in 1 MiB writes; GiB/s of input, median of --repeats after one warm-up round,
  the variants alternating.  Every member is checked with zlib.
- size: the compressed size under each schedule, against zlib at the same level with the same Z_SYNC_FLUSH
  schedule."""
import argparse
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


def latency(z, ctx, data, level, msg, count):
    tx = z.CompressStream(level, z.dfGzip, 0, ctx)
    rx = z.DecompressStream(z.dfGzip, ctx)
    fl, dr, got, sent, member = [], [], 0, 0, 0
    for i in range(count + 50):
        m = data[(i * msg) % (len(data) - msg):][:msg]
        t0 = time.perf_counter()
        piece = tx.write(m) + tx.flush()
        t1 = time.perf_counter()
        out = rx.write(piece) + rx.drain()
        t2 = time.perf_counter()
        sent += len(m)
        got += len(out)
        member += len(piece)
        assert got == sent or member < 20   # the gzip header (11 bytes) is decided with 9 bytes more
        if i >= 50:
            fl.append((t1 - t0) * 1e3)
            dr.append((t2 - t1) * 1e3)
    tx.close()
    rx.close()

    def q(v, p):
        return round(sorted(v)[int(p * (len(v) - 1))], 4)
    return {"flush_ms_median": q(fl, 0.5), "flush_ms_p90": q(fl, 0.9), "drain_ms_median": q(dr, 0.5),
            "drain_ms_p90": q(dr, 0.9)}


def zlib_size(data, level, every):
    co = zlib.compressobj(6 if level == -1 else level, zlib.DEFLATED, 31)
    n = 0
    for i in range(0, len(data), every or len(data)):
        n += len(co.compress(data[i:i + (every or len(data))]))
        if every:
            n += len(co.flush(zlib.Z_SYNC_FLUSH))
    return n + len(co.flush())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--levels", default="1,-1")
    ap.add_argument("--messages", type=int, default=2000)
    ap.add_argument("--no-zlib", action="store_true", help="skip the zlib sizes (single-threaded, slow at 1 GiB)")
    a = ap.parse_args()
    import zippy_b200 as z
    data = corpus_text(a.mib)
    ctx = z.Context()
    name, limit = card()
    levels = [int(x) for x in a.levels.split(",")]

    for level in levels:
        for msg in (1 << 10, 64 << 10):
            res = {"what": "latency", "level": level, "message_bytes": msg, "messages": a.messages, "card": name,
                   "power_limit": limit}
            res.update(latency(z, ctx, data[:64 << 20], level, msg, a.messages))
            print(json.dumps(res), flush=True)

    piece = 1 << 20
    for level in levels:
        scheds = {"none": 0, "every_1MiB": 1 << 20, "every_64MiB": 64 << 20}
        times = {k: [] for k in scheds}
        sizes = {}
        for r in range(a.repeats + 1):
            for k, every in scheds.items():
                outs = []
                t0 = time.perf_counter()
                with z.CompressStream(level, z.dfGzip, 0, ctx) as s:
                    for i in range(0, len(data), piece):
                        outs.append(s.write(data[i:i + piece]))
                        if every and (i + piece) % every == 0:
                            outs.append(s.flush())
                    outs.append(s.finish())
                dt = time.perf_counter() - t0
                if r:
                    times[k].append(dt)
                else:
                    member = b"".join(outs)
                    assert zlib.decompress(member, 31) == data, k
                    sizes[k] = len(member)
        for k, every in scheds.items():
            res = {"what": "throughput", "level": level, "flush": k, "input_gib": len(data) / (1 << 30),
                   "gib_s": round(len(data) / (1 << 30) / statistics.median(times[k]), 3), "bytes": sizes[k],
                   "ratio": round(sizes[k] / len(data), 5), "card": name, "power_limit": limit}
            if not a.no_zlib:
                res["zlib_bytes"] = zlib_size(data, level, every)
                res["vs_zlib"] = round(sizes[k] / res["zlib_bytes"], 4)
            print(json.dumps(res), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
