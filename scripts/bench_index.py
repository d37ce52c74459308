"""What an index of one large stream gains (DESIGN.md section 4.9): its build against decompress_large, full-stream
extracts at several spacings, and batches of random 64 KiB reads.

    python scripts/bench_index.py [--mib 1024] [--reps 3] [--out DIR]

--mib MiB of bench/synth.c class T as gzip L6, twice: from compress_large (split at sync points) and from Python
zlib (no sync points: the index's points are found block starts).  Per stream, device-resident, with the card's
name and power limit read in the same run:
  * decompress_large and index_build (default spacing) on the same buffer: host clock of the device-form call,
    its host waits and the final synchronisation included (best of --reps);
  * per spacing (256 KiB, 1 MiB, 4 MiB): access points, window bytes as a share of the output, and the output
    GB/s of one extract of the whole stream, checked against decompress_large's output (best of --reps);
  * random 64 KiB reads (seeded, uniform offsets) at batches of 1, 64 and 4096: reads per second of one
    extract call per batch (best of --reps).
"""
import argparse
import ctypes
import json
import os
import random
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import libdeflate_b200 as ldb  # noqa: E402
from bench_compress_large import card  # noqa: E402
from bench_decompress_large import Dev, synth  # noqa: E402

GZ = ldb.GZIP
SPACINGS = (256 << 10, 1 << 20, 4 << 20)
READ = 65536
BATCHES = (1, 64, 4096)


def best_of(reps, fn):
    best = None
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        dt = time.perf_counter() - t
        best = dt if best is None else min(best, dt)
    return best


def build(ctx, d_z, zn, d_out, n, spacing):
    ain, aout, res, ix = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int32(0), ctypes.c_void_p(None)
    ctx._check(ctx.l.libdeflate_b200_index_build(ctx.h, GZ, 0, d_z, zn, d_out, n, spacing, ctypes.byref(ain), ctypes.byref(aout),
                                                 ctypes.byref(res), ctypes.byref(ix)), "index_build")
    assert res.value == 0 and aout.value == n and ix.value, (res.value, aout.value)
    return ix.value


def extract(ctx, ix, d_z, zn, ranges, d_dst):
    k = len(ranges)
    offs = (ctypes.c_uint64 * k)(*[o for o, _ in ranges])
    lens = (ctypes.c_size_t * k)(*[ln for _, ln in ranges])
    dst = (ctypes.c_void_p * k)(*d_dst)
    res = (ctypes.c_int32 * k)()
    ctx._check(ctx.l.libdeflate_b200_index_extract(ctx.h, ix, d_z, zn, offs, lens, dst, res, k), "index_extract")
    assert all(r == 0 for r in res), list(res)[:8]


def stream_row(ctx, z, hb, reps):
    l, n, zn = ctx.l, len(hb), len(z)
    dz, dout, dres, dx = Dev(ctx, zn), Dev(ctx, n), Dev(ctx, 32), Dev(ctx, n)
    ctx._check(l.libdeflate_b200_memcpy_h2d(ctx.h, dz.p, z, zn), "h2d")
    ctx.sync()
    row = {"ratio": round(zn / n, 5)}
    large = lambda: (ctx._check(l.libdeflate_b200_decompress_large(ctx.h, GZ, 0, dz.p, zn, dout.p, n, dres.p, dres.p + 8, dres.p + 16),
                                "decompress_large"), ctx.sync())
    large()
    t_large = best_of(reps, large)
    row["decompress_large_ms"] = round(t_large * 1e3, 2)
    row["segments"] = l.libdeflate_b200_decompress_large_segments(ctx.h)
    l.libdeflate_b200_index_destroy(build(ctx, dz.p, zn, dout.p, n, 0))
    t_build = best_of(reps, lambda: l.libdeflate_b200_index_destroy(build(ctx, dz.p, zn, dout.p, n, 0)))
    row["index_build_ms"] = round(t_build * 1e3, 2)
    row["build_over_decompress_large"] = round(t_build / t_large, 3)
    row["spacings"] = {}
    rng = random.Random(1)
    for sp in SPACINGS:
        ix = build(ctx, dz.p, zn, dout.p, n, sp)
        pts = l.libdeflate_b200_index_points(ix)
        r = {"points": pts, "window_share": round((pts - 1) * 32768 / n, 4)}
        full = lambda: extract(ctx, ix, dz.p, zn, [(0, n)], [dx.p])
        full()
        ctx.sync()
        t = best_of(reps, full)
        same = np.empty(n, np.uint8)
        ctx._check(l.libdeflate_b200_memcpy_d2h(ctx.h, same.ctypes.data, dx.p, n), "d2h")
        ctx.sync()
        assert same.tobytes() == hb, "extract differs from the stream"
        r["full_extract_GB/s"] = round(n / t / 1e9, 2)
        r["full_extract_over_decompress_large"] = round(t_large / t, 2)
        for b in BATCHES:
            ranges = [(rng.randrange(n - READ), READ) for _ in range(b)]
            dsts = [dx.p + i * READ for i in range(b)]
            call = lambda: extract(ctx, ix, dz.p, zn, ranges, dsts)
            call()
            r["reads_per_s_batch_%d" % b] = round(b / best_of(reps, call), 1)
        row["spacings"]["%d_KiB" % (sp >> 10)] = r
        l.libdeflate_b200_index_destroy(ix)
        print("  spacing %d KiB: %s" % (sp >> 10, json.dumps(r)), flush=True)
    for d in (dz, dout, dres, dx):
        d.free()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()
    n = args.mib << 20
    name, power = card()
    res = {"card": name, "power_limit": power, "output_mib": args.mib, "class": "T", "format": "gzip", "level": 6, "streams": {}}
    print("card: %s, power limit %s; %d MiB of class T, gzip L6" % (name, power, args.mib), flush=True)
    ctx = ldb.Context(0)
    hb = synth(n, 0).tobytes()
    co = zlib.compressobj(6, zlib.DEFLATED, 31)
    for label, z in (("compress_large", lambda: ctx.compress_large(hb, 6, GZ)), ("zlib_no_sync", lambda: co.compress(hb) + co.flush())):
        print("%s:" % label, flush=True)
        row = stream_row(ctx, z(), hb, args.reps)
        res["streams"][label] = row
        print("%s: %s" % (label, json.dumps(row)), flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_index.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
