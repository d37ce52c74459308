"""Throughput of a compress stream (one stream written call by call) against compress_large on the same bytes.

    python scripts/bench_compress_stream.py [--mib 1024] [--reps 3] [--writes-mib 1 8 64 256] [--out DIR]

Input: --mib MiB of bench/synth.c class T (text-like) data, resident in HBM; gzip at L1 / L6 / L9.  For every
write size the stream is fed through the device form (libdeflate_b200_compress_stream_write) in writes of that
many MiB, the last one with FINISH, each write's output placed behind the previous one's bound.  Reported, with
the card's name and power limit read in the same run:
  * GB/s: input bytes over the CUDA-event time of the whole write sequence (stream create and destroy
    included), best of --reps after one warm-up;
  * ratio: stream bytes over input bytes (without a flush the stream is compress_large's, byte for byte);
  * compress_large on the same device buffer in the same process, timed the same way.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
import libdeflate_b200 as ldb  # noqa: E402
from bench_compress_large import card  # noqa: E402

GZ = ldb.GZIP


class Bench:
    def __init__(self, host_in):
        self.l = ldb.lib()
        self.ctx = ldb.Context(0, self.l)
        self.n = host_in.nbytes
        self.bound = self.l.libdeflate_b200_compress_large_bound(GZ, self.n)
        self.d_in = self.l.libdeflate_b200_device_malloc(self.ctx.h, self.n)
        # (room for the per-write bounds of the smallest writes: a little above compress_large's bound)
        self.out_avail = self.bound + (self.n >> 10) + (1 << 20)
        self.d_out = self.l.libdeflate_b200_device_malloc(self.ctx.h, self.out_avail)
        self.d_res = self.l.libdeflate_b200_device_malloc(self.ctx.h, 8)
        self.ctx._check(self.l.libdeflate_b200_memcpy_h2d(self.ctx.h, self.d_in, host_in.ctypes.data, self.n), "h2d")
        self.ctx.sync()

    def size(self):
        r = ctypes.c_size_t(0)
        self.ctx._check(self.l.libdeflate_b200_memcpy_d2h(self.ctx.h, ctypes.byref(r), self.d_res, 8), "d2h")
        self.ctx.sync()
        return r.value

    def large(self, level):
        self.ctx._check(self.l.libdeflate_b200_compress_large(self.ctx.h, GZ, level, self.d_in, self.n, self.d_out,
                                                              self.bound, self.d_res), "compress_large")

    def stream(self, level, step):
        """The whole input in writes of step bytes, queued without waiting (destroy waits at the end)."""
        l, ctx = self.l, self.ctx
        with ctx.compressobj(level, GZ) as cs:
            off = 0
            for k in range(0, self.n, step):
                m = min(step, self.n - k)
                fl = ldb.FINISH if k + m >= self.n else ldb.NO_FLUSH
                b = cs.bound(m, fl)
                assert off + b <= self.out_avail
                ctx._check(l.libdeflate_b200_compress_stream_write(cs.h, self.d_in + k, m, fl, self.d_out + off, b, self.d_res),
                           "compress_stream_write")
                off += b

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

    def stream_bytes(self, level, step):
        """Exact stream size: every write's size word read back in turn."""
        l, ctx = self.l, self.ctx
        total = 0
        with ctx.compressobj(level, GZ) as cs:
            for k in range(0, self.n, step):
                m = min(step, self.n - k)
                fl = ldb.FINISH if k + m >= self.n else ldb.NO_FLUSH
                ctx._check(l.libdeflate_b200_compress_stream_write(cs.h, self.d_in + k, m, fl, self.d_out, self.out_avail,
                                                                   self.d_res), "compress_stream_write")
                total += self.size()
        return total

    def free(self):
        for p in (self.d_in, self.d_out, self.d_res):
            self.l.libdeflate_b200_device_free(self.ctx.h, p)
        self.ctx.close()


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
    res = {"card": name, "power_limit": power, "input_mib": args.mib, "data": "bench/synth.c class T", "format": "gzip",
           "piece": ldb.LARGE_PIECE, "large": {}, "stream": {}}
    print("card: %s, power limit %s; %d MiB class T, gzip" % (name, power, args.mib), flush=True)
    b = Bench(host)
    for level in (1, 6, 9):
        key = "L%d" % level
        gbs = b.timed(lambda: b.large(level), args.reps)
        ratio = b.size() / n
        res["large"][key] = {"GB/s": round(gbs, 2), "ratio": round(ratio, 5)}
        print("compress_large %s: %.2f GB/s, ratio %.5f" % (key, gbs, ratio), flush=True)
        res["stream"][key] = {}
        for w in args.writes_mib:
            gbs = b.timed(lambda: b.stream(level, w << 20), args.reps)
            ratio = b.stream_bytes(level, w << 20) / n
            res["stream"][key]["%d MiB writes" % w] = {"GB/s": round(gbs, 2), "ratio": round(ratio, 5)}
            print("stream %s, %d MiB writes: %.2f GB/s, ratio %.5f" % (key, w, gbs, ratio), flush=True)
    b.free()
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_compress_stream.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
