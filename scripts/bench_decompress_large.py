"""Throughput of decompress_large (one stream -> its bytes, split at its sync points) against the other ways
to decompress the same bytes on the GPU.

    python scripts/bench_decompress_large.py [--mib 1024] [--reps 3] [--classes T,M,R] [--zlib-mib 256] [--out DIR]

Per bench/synth.c class: --mib MiB compressed by compress_large (gzip, L6), the stream resident in HBM.
Reported, with the card's name and power limit read in the same run:
  * decompress_large: output GB/s over the host clock of the whole device-form call, its host waits and the
    final stream synchronisation included (best of --reps), the segment count, and the stage split from
    the kernel-time kinds (2 decode, 5 resolve, 6 scan / windows / substitution / results, 0+1 checksums);
  * the same bytes as BGZF through bgzf_decompress (a host call: staging over PCIe included) and as a batch of
    64 KiB gzip chunks through decompress_batch (CUDA-event time);
  * the classic one-lane call (libdeflate_gzip_decompress) on the compress_large stream of a 16 MiB PREFIX;
  * Python-zlib streams sync-flushed every 128 KiB and every 1 MiB (--zlib-mib MiB of class T);
  * Python-zlib streams WITHOUT sync points (split at the block starts the finder lists): class T at L1, L6 and
    L9 and classes M and R at L6, --zlib-mib MiB each, with the finder's own kernel time (torch.profiler, one
    more call) and the one-lane call on the first 16 MiB of class T at L6.
"""
import argparse
import ctypes
import json
import os
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench  # noqa: E402
import libdeflate_b200 as ldb  # noqa: E402
from bench_compress_large import card  # noqa: E402

GZ = ldb.GZIP
CHUNK = 65536
CLASSES = {"T": 0, "PAT": 1, "S": 2, "R": 3, "Z": 4, "M": 5}


def synth(n, cls):
    host = np.empty(n, np.uint8)
    bench.load_synth().synth_fill(host.ctypes.data, CHUNK, 0, n // CHUNK, cls, os.cpu_count() or 8)
    return host


class Dev:
    def __init__(self, ctx, nbytes):
        self.ctx, self.l = ctx, ctx.l
        self.p = self.l.libdeflate_b200_device_malloc(ctx.h, max(nbytes, 1))

    def free(self):
        self.l.libdeflate_b200_device_free(self.ctx.h, self.p)


def large(ctx, d_z, zn, n, reps):
    """(GB/s of output, segments, {stage: ms}) of decompress_large on a device-resident stream."""
    l = ctx.l
    out, res = Dev(ctx, n), Dev(ctx, 32)
    call = lambda: ctx._check(l.libdeflate_b200_decompress_large(ctx.h, GZ, 0, d_z, zn, out.p, n, res.p, res.p + 8, res.p + 16),
                              "decompress_large")
    call()
    ctx.sync()
    best = None
    for _ in range(reps):
        t = time.perf_counter()
        call()
        ctx.sync()
        dt = time.perf_counter() - t
        best = dt if best is None else min(best, dt)
    r = (ctypes.c_uint64 * 3)()
    ctx._check(l.libdeflate_b200_memcpy_d2h(ctx.h, r, res.p, 24), "d2h")
    ctx.sync()
    assert r[2] & 0xffffffff == 0 and r[1] == n, "decompress_large failed: %r" % list(r)
    segs = l.libdeflate_b200_decompress_large_segments(ctx.h)
    l.libdeflate_b200_kernel_time_reset(ctx.h)
    l.libdeflate_b200_ctx_set_profiling(ctx.h, 1)
    call()
    ctx.sync()
    l.libdeflate_b200_ctx_set_profiling(ctx.h, 0)
    stages = {}
    for kind, name in ((2, "decode"), (5, "resolve"), (6, "scan+windows+substitute+results"), (0, "crc32")):
        stages[name] = round(l.libdeflate_b200_kernel_time_ms(ctx.h, kind, None), 3)
    out.free()
    res.free()
    return n / best / 1e9, segs, stages


def batch_64k(ctx, host, reps):
    """The same bytes as 64 KiB gzip chunks through decompress_batch: output GB/s (CUDA events)."""
    l = ctx.l
    n = host.nbytes
    k = n // CHUNK
    packed, offs, sizes = ctx.compress_batch_host_packed([host[i * CHUNK:(i + 1) * CHUNK] for i in range(k)], 6, GZ)
    din = Dev(ctx, len(packed))
    ctx._check(l.libdeflate_b200_memcpy_h2d(ctx.h, din.p, packed, len(packed)), "h2d")
    ptrs = np.array([din.p + o for o in offs[:k]], np.uint64)
    dout = bench.DeviceBatch(ctx, k, CHUNK)
    dout.set_sizes(np.full(k, CHUNK, np.uint64))
    d_ptrs, d_sz, d_res = Dev(ctx, 8 * k), Dev(ctx, 8 * k), Dev(ctx, 4 * k)
    ctx._check(l.libdeflate_b200_memcpy_h2d(ctx.h, d_ptrs.p, ptrs.ctypes.data, 8 * k), "h2d")
    sz = np.array(sizes, np.uint64)
    ctx._check(l.libdeflate_b200_memcpy_h2d(ctx.h, d_sz.p, sz.ctypes.data, 8 * k), "h2d")
    call = lambda: ctx._check(l.libdeflate_b200_decompress_batch(ctx.h, GZ, 0, d_ptrs.p, d_sz.p, dout.d_ptrs, dout.d_sizes,
                                                                 None, None, d_res.p, k), "decompress_batch")
    call()
    ctx.sync()
    best = None
    for _ in range(reps):
        l.libdeflate_b200_timer_start(ctx.h)
        call()
        ms = l.libdeflate_b200_timer_stop_ms(ctx.h)
        best = ms if best is None else min(best, ms)
    for b in (din, d_ptrs, d_sz, d_res):
        b.free()
    dout.free()
    return k * CHUNK / best / 1e6


def classic_prefix(ctx, host):
    """libdeflate_gzip_decompress (one lane) on the compress_large stream of a 16 MiB prefix: output GB/s."""
    l = ctx.l
    m = min(host.nbytes, 16 << 20)
    z = ctx.compress_large(host[:m].tobytes(), 6, GZ)
    dz, dout = Dev(ctx, len(z)), Dev(ctx, m)
    ctx._check(l.libdeflate_b200_memcpy_h2d(ctx.h, dz.p, z, len(z)), "h2d")
    ctx.sync()
    d = l.libdeflate_alloc_decompressor()
    aout = ctypes.c_size_t(0)
    t = time.perf_counter()
    r = l.libdeflate_gzip_decompress(d, dz.p, len(z), dout.p, m, ctypes.byref(aout))
    dt = time.perf_counter() - t
    l.libdeflate_free_decompressor(d)
    dz.free()
    dout.free()
    assert r == 0 and aout.value == m
    return m / dt / 1e9


def kernel_ms(fn):
    """{kernel name: ms} of one call, from torch.profiler's CUDA activities (None where unavailable)."""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
        out = {}
        for e in prof.events():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = getattr(e, "cuda_time_total", 0)
            if t:
                out[e.name] = out.get(e.name, 0.0) + t / 1000.0
        return out
    except Exception as ex:  # noqa: BLE001
        print("torch.profiler unavailable: %s" % ex, flush=True)
        return None


def nosync(ctx, hb, level, reps):
    """decompress_large of a Python-zlib gzip stream without sync points."""
    z = zlib.compressobj(level, zlib.DEFLATED, 31)
    z = z.compress(hb) + z.flush()
    assert b"\x00\x00\xff\xff" not in z
    dz = Dev(ctx, len(z))
    ctx._check(ctx.l.libdeflate_b200_memcpy_h2d(ctx.h, dz.p, z, len(z)), "h2d")
    ctx.sync()
    gbs, segs, stages = large(ctx, dz.p, len(z), len(hb), reps)
    out, res = Dev(ctx, len(hb)), Dev(ctx, 32)
    km = kernel_ms(lambda: (ctx.l.libdeflate_b200_decompress_large(ctx.h, GZ, 0, dz.p, len(z), out.p, len(hb), res.p, res.p + 8,
                                                                    res.p + 16), ctx.sync()))
    out.free()
    res.free()
    dz.free()
    row = {"ratio": round(len(z) / len(hb), 5), "decompress_large_GB/s": round(gbs, 2), "segments": segs, "stage_ms": stages}
    if km is not None:
        row["finder_ms"] = round(sum(v for k, v in km.items() if "block_scan" in k), 3)
        row["window_chain_ms"] = round(sum(v for k, v in km.items() if "window_chain" in k), 3)
    return row


def one_lane(ctx, hb, level):
    """libdeflate_gzip_decompress (one lane) on a Python-zlib stream without sync points: output GB/s."""
    l = ctx.l
    z = zlib.compressobj(level, zlib.DEFLATED, 31)
    z = z.compress(hb) + z.flush()
    dz, dout = Dev(ctx, len(z)), Dev(ctx, len(hb))
    ctx._check(l.libdeflate_b200_memcpy_h2d(ctx.h, dz.p, z, len(z)), "h2d")
    ctx.sync()
    d = l.libdeflate_alloc_decompressor()
    aout = ctypes.c_size_t(0)
    t = time.perf_counter()
    r = l.libdeflate_gzip_decompress(d, dz.p, len(z), dout.p, len(hb), ctypes.byref(aout))
    dt = time.perf_counter() - t
    l.libdeflate_free_decompressor(d)
    dz.free()
    dout.free()
    assert r == 0 and aout.value == len(hb)
    return len(hb) / dt / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--classes", default="T,M,R")
    ap.add_argument("--zlib-mib", type=int, default=256)
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    ap.add_argument("--nosync-only", action="store_true", help="only the streams without sync points")
    args = ap.parse_args()
    n = args.mib << 20
    name, power = card()
    res = {"card": name, "power_limit": power, "input_mib": args.mib, "format": "gzip", "level": 6, "classes": {}}
    print("card: %s, power limit %s; %d MiB per class, gzip L6" % (name, power, args.mib), flush=True)
    ctx = ldb.Context(0)
    res["zlib_no_sync"] = {}
    m = args.zlib_mib << 20
    for cname, level in (("T", 1), ("T", 6), ("T", 9), ("M", 6), ("R", 6)):
        hb = synth(m, CLASSES[cname]).tobytes()
        row = nosync(ctx, hb, level, args.reps)
        if (cname, level) == ("T", 6):
            row["one_lane_16MiB_GB/s"] = round(one_lane(ctx, hb[:16 << 20], level), 4)
        res["zlib_no_sync"]["%s_L%d" % (cname, level)] = row
        print("zlib without sync points, class %s L%d, %d MiB: %s" % (cname, level, args.zlib_mib, json.dumps(row)), flush=True)
    for cname in ([] if args.nosync_only else args.classes.split(",")):
        host = synth(n, CLASSES[cname])
        hb = host.tobytes()
        z = ctx.compress_large(hb, 6, GZ)
        dz = Dev(ctx, len(z))
        ctx._check(ctx.l.libdeflate_b200_memcpy_h2d(ctx.h, dz.p, z, len(z)), "h2d")
        ctx.sync()
        gbs, segs, stages = large(ctx, dz.p, len(z), n, args.reps)
        dz.free()
        row = {"ratio": round(len(z) / n, 5), "decompress_large_GB/s": round(gbs, 2), "segments": segs, "stage_ms": stages}
        bg = ctx.bgzf_compress(hb, 6)
        t = time.perf_counter()
        r, _ = ctx.bgzf_decompress(bg, n)
        row["bgzf_decompress_host_GB/s"] = round(n / (time.perf_counter() - t) / 1e9, 2)
        assert r == 0
        row["batch_64KiB_GB/s"] = round(batch_64k(ctx, host, args.reps), 2)
        row["classic_one_lane_16MiB_prefix_GB/s"] = round(classic_prefix(ctx, host), 4)
        res["classes"][cname] = row
        print("class %s: %s" % (cname, json.dumps(row)), flush=True)
    hb = synth(m, 0).tobytes()
    res["zlib_sync_flush"] = {}
    for every in (() if args.nosync_only else (128 << 10, 1 << 20)):
        co = zlib.compressobj(6, zlib.DEFLATED, 31)
        z = b"".join(co.compress(hb[i:i + every]) + co.flush(zlib.Z_SYNC_FLUSH) for i in range(0, m, every)) + co.flush()
        dz = Dev(ctx, len(z))
        ctx._check(ctx.l.libdeflate_b200_memcpy_h2d(ctx.h, dz.p, z, len(z)), "h2d")
        ctx.sync()
        gbs, segs, stages = large(ctx, dz.p, len(z), m, args.reps)
        dz.free()
        row = {"decompress_large_GB/s": round(gbs, 2), "segments": segs, "stage_ms": stages}
        res["zlib_sync_flush"]["%d_KiB" % (every >> 10)] = row
        print("zlib Z_SYNC_FLUSH every %d KiB, %d MiB class T: %s" % (every >> 10, args.zlib_mib, json.dumps(row)), flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_decompress_large.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
