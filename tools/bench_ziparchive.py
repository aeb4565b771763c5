"""Time the ZipArchive object API through the GPU on one large archive, and the decode call behind its reader.
Prints one JSON line with the card's name and power limit.

    python tools/bench_ziparchive.py [--mib 1024] [--repeats 3] [--seed 7]

The tree is seeded and held in memory (the files of tools/bench_tarball.py: text windows of the test corpus,
byte runs and random bytes in files of 0..8 MiB).  Reported, median of --repeats after one warm-up call:
- write_zip_archive: one compress_batch at DefaultCompression, one checksum_batch, the layout, the file write;
- ZipArchive.open: the header walk, one inflate_batch_crc32 for the deflated entries, the checks;
- for the same archive's entries, the two ways to get outputs and their CRC-32s, alternating in one run:
  inflate_batch_crc32 (the CRC comes from the decode call) against uncompress_batch + a host join of the outputs
  + checksum_batch (the v2 reader's way).
Every call returns after its device work has finished and its output is in host memory; the host clock times it."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=60).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in q.split(",")]
        return name, limit
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    import zippy_b200 as z
    import zippy_b200.ziparchives as za
    from tools.bench_tarball import seeded_contents
    ctx = z.default_context()
    archive = za.ZipArchive(ctx)
    for path, e in seeded_contents(a.mib << 20, a.seed).items():
        archive.contents[path + "/" if e.kind == "dir" else path] = za.ArchiveEntry(e.kind, e.contents,
                                                                                  e.last_modified, e.permissions)
    total = sum(len(e.contents) for e in archive.contents.values())
    med = lambda ts: statistics.median(ts[1:])  # noqa: E731  (the first call is a warm-up)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "big.zip")
        w_ms, o_ms = [], []
        for _ in range(a.repeats + 1):
            t0 = time.perf_counter()
            archive.write_zip_archive(path)
            w_ms.append((time.perf_counter() - t0) * 1e3)
        back = za.ZipArchive(ctx)
        for _ in range(a.repeats + 1):
            t0 = time.perf_counter()
            back.open(path)
            o_ms.append((time.perf_counter() - t0) * 1e3)
        assert [k for k in back.contents] == list(archive.contents)
        assert all(back.contents[k].contents == e.contents for k, e in archive.contents.items())
        data = open(path, "rb").read()
    # the deflated entries of the archive, as ZipArchive.open hands them to the decode
    members, sizes, want = [], [], []
    pos = 0
    while int.from_bytes(data[pos:pos + 4], "little") == 0x04034B50:
        method, crc, csize, usize, nlen = (int.from_bytes(data[pos + 8:pos + 10], "little"),
                                           *(int.from_bytes(data[pos + k:pos + k + 4], "little") for k in (14, 18, 22)),
                                           int.from_bytes(data[pos + 26:pos + 28], "little"))
        p = pos + 30 + nlen
        if method == 8:
            members.append(data[p:p + csize])
            sizes.append(usize)
            want.append(crc)
        pos = p + csize
    offs = np.zeros(len(members) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(m) for m in members])
    base = np.frombuffer(b"".join(members), dtype=np.uint8)
    sizes = np.array(sizes, dtype=np.uint64)

    def fused():
        out, do, lens, crcs, st = ctx.inflate_batch_crc32(base, offs, sizes)
        return crcs, st

    def separate():
        out, do, lens, st = ctx.uncompress_batch(base, offs, z.dfDeflate, sizes=sizes)
        blobs = [out[int(do[i]):int(do[i]) + int(lens[i])] for i in range(len(members))]
        o2 = np.zeros(len(blobs) + 1, dtype=np.uint64)
        o2[1:] = np.cumsum([len(b) for b in blobs])
        return ctx.checksum_batch(np.concatenate(blobs), o2, "crc32"), st

    f_ms, s_ms = [], []
    for _ in range(a.repeats + 1):
        for fn, ts in ((fused, f_ms), (separate, s_ms)):
            t0 = time.perf_counter()
            crcs, st = fn()
            ts.append((time.perf_counter() - t0) * 1e3)
            assert not st.any() and [int(c) for c in crcs] == want
    name, limit = card()
    gib = total / (1 << 30)
    print(json.dumps({
        "gpu": name, "power_limit": limit, "entries": len(archive.contents), "deflated_entries": len(members),
        "contents_gib": round(gib, 4), "archive_bytes": len(data),
        "write_zip_archive_ms": round(med(w_ms), 1), "open_ms": round(med(o_ms), 1),
        "inflate_batch_crc32_ms": round(med(f_ms), 1), "uncompress_join_checksum_ms": round(med(s_ms), 1),
        "all_ms": {"write_zip_archive": [round(x, 1) for x in w_ms], "open": [round(x, 1) for x in o_ms],
                   "inflate_batch_crc32": [round(x, 1) for x in f_ms],
                   "uncompress_join_checksum": [round(x, 1) for x in s_ms]},
    }))


if __name__ == "__main__":
    main()
