"""Throughput and ratio of compress_large (one buffer -> one stream) against the other ways to compress
the same bytes on the GPU.

    python scripts/bench_compress_large.py [--mib 1024] [--reps 3] [--piece-libs P=LIB ...] [--out DIR]

Input: --mib MiB of bench/synth.c class T (text-like) data, resident in HBM; gzip throughout.
Reported, with the card's name and power limit read in the same run:
  * compress_large at L1 / L6 / L9: GB/s (input bytes over CUDA-event time of the whole call, setup,
    checksums, deflate and stitch included) and ratio;
  * the same bytes as a batch of 64 KiB chunks through compress_batch (GB/s, ratio), and through BGZF
    (ratio; a host call, so its time is not comparable);
  * the classic single call (libdeflate_gzip_compress) on a 64 MiB device buffer: the speed a caller
    who holds one buffer gets without compress_large;
  * with --piece-libs (libraries built with -DLDB_LARGE_PIECE=...): compress_large GB/s and ratio per
    piece size, the measurement the default piece size was chosen from.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import libdeflate_b200 as ldb  # noqa: E402

GZ = ldb.GZIP
CHUNK = 65536


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [x.strip() for x in q.splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # (reported, never guessed)
        return "unknown (%s)" % e, "unknown"


class Large:
    """One library's context with the input and a bound-sized output in device memory."""

    def __init__(self, lib, host_in):
        self.l = ldb.load_library(lib) if lib else ldb.lib()
        self.ctx = ldb.Context(0, self.l)
        self.n = host_in.nbytes
        self.bound = self.l.libdeflate_b200_compress_large_bound(GZ, self.n)
        self.d_in = self.l.libdeflate_b200_device_malloc(self.ctx.h, self.n)
        self.d_out = self.l.libdeflate_b200_device_malloc(self.ctx.h, self.bound)
        self.d_res = self.l.libdeflate_b200_device_malloc(self.ctx.h, 8)
        self.ctx._check(self.l.libdeflate_b200_memcpy_h2d(self.ctx.h, self.d_in, host_in.ctypes.data, self.n), "h2d")
        self.ctx.sync()

    def run(self, level, reps):
        """(GB/s of the best rep, ratio)"""
        call = lambda: self.ctx._check(self.l.libdeflate_b200_compress_large(
            self.ctx.h, GZ, level, self.d_in, self.n, self.d_out, self.bound, self.d_res), "compress_large")
        call()
        self.ctx.sync()
        best = None
        for _ in range(reps):
            self.l.libdeflate_b200_timer_start(self.ctx.h)
            call()
            ms = self.l.libdeflate_b200_timer_stop_ms(self.ctx.h)
            best = ms if best is None else min(best, ms)
        r = ctypes.c_size_t(0)
        self.ctx._check(self.l.libdeflate_b200_memcpy_d2h(self.ctx.h, ctypes.byref(r), self.d_res, 8), "d2h")
        self.ctx.sync()
        assert r.value, "compress_large did not fit its bound"
        return self.n / best / 1e6, r.value / self.n

    def free(self):
        for p in (self.d_in, self.d_out, self.d_res):
            self.l.libdeflate_b200_device_free(self.ctx.h, p)
        self.ctx.close()


def batch_64k(ctx, l, d_in, n, level, reps):
    """The same bytes as n / 64 KiB independent chunks: (GB/s, ratio)."""
    k = n // CHUNK
    stride = (l.libdeflate_gzip_compress_bound(None, CHUNK) + 15) & ~15
    din = bench.DeviceBatch(ctx, k, CHUNK, slab=d_in)
    din.set_sizes(np.full(k, CHUNK, np.uint64))
    dout = bench.DeviceBatch(ctx, k, stride)
    dout.set_sizes(np.full(k, stride, np.uint64))
    d_sz = l.libdeflate_b200_device_malloc(ctx.h, 8 * k)
    call = lambda: ctx._check(l.libdeflate_b200_compress_batch(ctx.h, GZ, level, din.d_ptrs, din.d_sizes, dout.d_ptrs,
                                                                dout.d_sizes, d_sz, k), "compress_batch")
    call()
    ctx.sync()
    best = None
    for _ in range(reps):
        l.libdeflate_b200_timer_start(ctx.h)
        call()
        ms = l.libdeflate_b200_timer_stop_ms(ctx.h)
        best = ms if best is None else min(best, ms)
    sz = np.empty(k, np.uint64)
    ctx._check(l.libdeflate_b200_memcpy_d2h(ctx.h, sz.ctypes.data, d_sz, 8 * k), "d2h")
    ctx.sync()
    din.free()
    dout.free()
    l.libdeflate_b200_device_free(ctx.h, d_sz)
    return k * CHUNK / best / 1e6, float(sz.sum()) / (k * CHUNK)


def classic_single(l, ctx, d_in, n):
    """libdeflate_gzip_compress(L6) on one device buffer of n bytes: GB/s (host clock around a synchronous call)."""
    c = l.libdeflate_alloc_compressor(6)
    bound = l.libdeflate_gzip_compress_bound(c, n)
    d_out = l.libdeflate_b200_device_malloc(ctx.h, bound)
    l.libdeflate_gzip_compress(c, d_in, n, d_out, bound)         # (creates the compressor's context)
    t = time.perf_counter()
    r = l.libdeflate_gzip_compress(c, d_in, n, d_out, bound)
    dt = time.perf_counter() - t
    l.libdeflate_free_compressor(c)
    l.libdeflate_b200_device_free(ctx.h, d_out)
    return n / dt / 1e9, r / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--piece-libs", nargs="*", default=[], help="PIECE=LIB: compress_large of each library at L1 / L6")
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()
    n = args.mib << 20
    host = np.empty(n, np.uint8)
    bench.load_synth().synth_fill(host.ctypes.data, CHUNK, 0, n // CHUNK, 0, os.cpu_count() or 8)
    name, power = card()
    res = {"card": name, "power_limit": power, "input_mib": args.mib, "data": "bench/synth.c class T", "format": "gzip",
           "piece": ldb.LARGE_PIECE}
    print("card: %s, power limit %s; %d MiB class T, gzip" % (name, power, args.mib), flush=True)

    lg = Large(None, host)
    res["large"] = {}
    for level in (1, 6, 9):
        gbs, ratio = lg.run(level, args.reps)
        res["large"]["L%d" % level] = {"GB/s": round(gbs, 2), "ratio": round(ratio, 5)}
        print("compress_large L%d: %.2f GB/s, ratio %.5f" % (level, gbs, ratio), flush=True)
    res["batch_64KiB"] = {}
    for level in (1, 6, 9):
        gbs, ratio = batch_64k(lg.ctx, lg.l, lg.d_in, n, level, args.reps)
        res["batch_64KiB"]["L%d" % level] = {"GB/s": round(gbs, 2), "ratio": round(ratio, 5)}
        print("compress_batch 64 KiB chunks L%d: %.2f GB/s, ratio %.5f" % (level, gbs, ratio), flush=True)
    res["bgzf"] = {}
    host_bytes = host.tobytes()
    for level in (1, 6, 9):
        z = lg.ctx.bgzf_compress(host_bytes, level)
        res["bgzf"]["L%d" % level] = {"ratio": round(len(z) / n, 5)}
        print("bgzf L%d: ratio %.5f" % (level, len(z) / n), flush=True)
    m = min(n, 64 << 20)
    gbs, ratio = classic_single(lg.l, lg.ctx, lg.d_in, m)
    res["classic_single_64MiB_L6"] = {"GB/s": round(gbs, 4), "ratio": round(ratio, 5)}
    print("classic libdeflate_gzip_compress, one 64 MiB device buffer, L6: %.4f GB/s, ratio %.5f" % (gbs, ratio), flush=True)
    lg.free()

    res["piece_sizes"] = {}
    for spec in args.piece_libs:
        piece, lib = spec.split("=", 1)
        side = Large(lib, host)
        row = {}
        for level in (1, 6, 9):
            gbs, ratio = side.run(level, args.reps)
            row["L%d" % level] = {"GB/s": round(gbs, 2), "ratio": round(ratio, 5)}
        res["piece_sizes"][piece] = row
        print("piece %s: %s" % (piece, json.dumps(row)), flush=True)
        side.free()
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_compress_large.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
