"""Throughput of a decompress stream (one stream read call by call) against decompress_large on the same bytes.

    python scripts/bench_decompress_stream.py [--mib 1024] [--reps 3] [--writes-mib 1 8 64 256] [--out DIR]

Input: --mib MiB of bench/synth.c class T (text-like) data as gzip, made two ways: by compress_large at L6 (sync
points every piece) and by Python zlib at L6 (no sync points: split at the block starts the finder lists).  The
stream is resident in HBM.  For every write size it is fed through the device form
(libdeflate_b200_decompress_stream_write) in writes of that many MiB, the last one with 'last' set, each write's
output placed behind the previous one's.  Reported, with the card's name and power limit read in the same run:
  * GB/s: output bytes over the CUDA-event time of the whole write sequence (stream create and destroy
    included), best of --reps after one warm-up;
  * segments per write: the chain segments of each write (decompress_large_segments after it), averaged;
  * decompress_large on the same device buffer in the same process, timed the same way.
"""
import argparse
import ctypes
import json
import os
import sys
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
import libdeflate_b200 as ldb  # noqa: E402
from bench_compress_large import card  # noqa: E402

GZ = ldb.GZIP


class Bench:
    def __init__(self, ctx, z, n_out):
        self.l = ctx.l
        self.ctx = ctx
        self.nz, self.n = len(z), n_out
        self.d_in = self.l.libdeflate_b200_device_malloc(ctx.h, self.nz)
        self.d_out = self.l.libdeflate_b200_device_malloc(ctx.h, self.n + (1 << 20))
        self.d_res = self.l.libdeflate_b200_device_malloc(ctx.h, 32)
        buf = ctypes.create_string_buffer(z, len(z))
        ctx._check(self.l.libdeflate_b200_memcpy_h2d(ctx.h, self.d_in, buf, self.nz), "h2d")
        ctx.sync()
        self.segs = []

    def large(self):
        r = self.d_res
        self.ctx._check(self.l.libdeflate_b200_decompress_large(self.ctx.h, GZ, 0, self.d_in, self.nz, self.d_out, self.n + (1 << 20),
                                                                r, r + 8, r + 16), "decompress_large")

    def stream(self, step):
        l, ctx = self.l, self.ctx
        s = l.libdeflate_b200_decompress_stream_create(ctx.h, GZ)
        w, need, unused, res = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int32()
        off, segs = 0, []
        for k in range(0, self.nz, step):
            m = min(step, self.nz - k)
            ctx._check(l.libdeflate_b200_decompress_stream_write(s, self.d_in + k, m, int(k + m >= self.nz), self.d_out + off,
                                                                 self.n + (1 << 20) - off, ctypes.byref(w), ctypes.byref(need),
                                                                 ctypes.byref(unused), ctypes.byref(res)), "decompress_stream_write")
            off += w.value
            segs.append(l.libdeflate_b200_decompress_large_segments(ctx.h))
        l.libdeflate_b200_decompress_stream_destroy(s)
        assert res.value == 0 and off == self.n, (res.value, off, self.n)
        self.segs = segs

    def timed(self, f, reps):
        f()
        self.ctx.sync()
        best = None
        for _ in range(reps):
            self.l.libdeflate_b200_timer_start(self.ctx.h)
            f()
            ms = self.l.libdeflate_b200_timer_stop_ms(self.ctx.h)
            best = ms if best is None else min(best, ms)
        return self.n / best / 1e6

    def free(self):
        for p in (self.d_in, self.d_out, self.d_res):
            self.l.libdeflate_b200_device_free(self.ctx.h, p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--writes-mib", type=int, nargs="*", default=[1, 8, 64, 256])
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()
    n = args.mib << 20
    host = np.empty(n, np.uint8)
    bench.load_synth().synth_fill(host.ctypes.data, 65536, 0, n // 65536, 0, os.cpu_count() or 8)
    name, power = card()
    res = {"card": name, "power_limit": power, "output_mib": args.mib, "data": "bench/synth.c class T", "format": "gzip",
           "streams": {}}
    print("card: %s, power limit %s; %d MiB class T, gzip" % (name, power, args.mib), flush=True)
    ctx = ldb.Context(0)
    data = host.tobytes()
    co = zlib.compressobj(6, zlib.DEFLATED, 31)
    makers = {"compress_large L6": lambda: ctx.compress_large(data, 6, GZ),
              "zlib L6": lambda: co.compress(data) + co.flush()}
    for key, make in makers.items():
        z = make()
        b = Bench(ctx, z, n)
        r = {"compressed_mib": round(len(z) / 2**20, 1)}
        gbs = b.timed(b.large, args.reps)
        r["decompress_large GB/s"] = round(gbs, 2)
        r["decompress_large segments"] = ctx.large_segments()
        print("%s: decompress_large %.2f GB/s, %d segments" % (key, gbs, ctx.large_segments()), flush=True)
        for w in args.writes_mib:
            gbs = b.timed(lambda: b.stream(w << 20), args.reps)
            spw = sum(b.segs) / len(b.segs)
            r["%d MiB writes" % w] = {"GB/s": round(gbs, 2), "writes": len(b.segs), "segments per write": round(spw, 1)}
            print("%s, %d MiB writes: %.2f GB/s, %d writes, %.1f segments per write" % (key, w, gbs, len(b.segs), spw), flush=True)
        res["streams"][key] = r
        b.free()
    ctx.close()
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_decompress_stream.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
