"""A/B timing of the deflate kernel of two library builds, alternated in one process on one GPU.

    python scripts/ab_deflate.py LIB_A LIB_B [--rounds 3] [--data-class 0] [--legs ...] [--out DIR]

Both libraries compress the same device-resident synthetic batches (bench/synth.c class 0, the
bench corpus, unless --data-class picks another of its six classes); every round times each library
once per leg, A then B, so that drift of the card shows up in both.  Legs: the bench shape (65 536 x 64 KiB, gzip level 6), levels 1 and 9 on a
quarter of it, and 528 x 1 MiB at level 12 (four waves of the 132 CTAs).  Reported: deflate kernel
ms per launch (library event pairs), and whether the two libraries' compressed sizes and a sample of
their streams agree byte for byte.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import libdeflate_b200 as ldb  # noqa: E402

LEGS = [("L6_65536x64KiB", 6, 65536, 65536), ("L1_16384x64KiB", 1, 16384, 65536),
        ("L9_16384x64KiB", 9, 16384, 65536), ("L12_528x1MiB", 12, 528, 1 << 20)]


class Side:
    def __init__(self, path, pin_in, n, chunk):
        self.l = ldb.load_library(path)
        self.ctx = ldb.Context(0, self.l)
        self.n, self.chunk = n, chunk
        self.cstride = (self.l.libdeflate_gzip_compress_bound(None, chunk) + 15) & ~15
        self.d_in = bench.DeviceBatch(self.ctx, n, chunk)
        self.ctx._check(self.l.libdeflate_b200_memcpy_h2d(self.ctx.h, self.d_in.slab, pin_in, n * chunk), "h2d")
        self.d_in.set_sizes(np.full(n, chunk, dtype=np.uint64))
        self.d_comp = bench.DeviceBatch(self.ctx, n, self.cstride)
        self.d_comp.set_sizes(np.full(n, self.cstride, dtype=np.uint64))
        self.d_csz = self.l.libdeflate_b200_device_malloc(self.ctx.h, 8 * n)

    def launch(self, level):
        self.ctx._check(self.l.libdeflate_b200_compress_batch(self.ctx.h, ldb.GZIP, level, self.d_in.d_ptrs, self.d_in.d_sizes,
                                                               self.d_comp.d_ptrs, self.d_comp.d_sizes, self.d_csz, self.n), "compress_batch")

    def time(self, level, launches):
        self.launch(level)
        self.ctx.sync()
        self.l.libdeflate_b200_ctx_set_profiling(self.ctx.h, 1)
        self.l.libdeflate_b200_kernel_time_reset(self.ctx.h)
        for _ in range(launches):
            self.launch(level)
        self.ctx.sync()
        cnt = ctypes.c_uint64(0)
        t = self.l.libdeflate_b200_kernel_time_ms(self.ctx.h, bench.KIND["deflate"], ctypes.byref(cnt))
        self.l.libdeflate_b200_ctx_set_profiling(self.ctx.h, 0)
        return t / max(cnt.value, 1)

    def outputs(self, sample):
        csz = np.empty(self.n, dtype=np.uint64)
        self.ctx._check(self.l.libdeflate_b200_memcpy_d2h(self.ctx.h, csz.ctypes.data, self.d_csz, 8 * self.n), "d2h")
        self.ctx.sync()
        crcs = []
        for i in sample:
            buf = np.empty(int(csz[i]), dtype=np.uint8)
            self.ctx._check(self.l.libdeflate_b200_memcpy_d2h(self.ctx.h, buf.ctypes.data, self.d_comp.slab + int(i) * self.cstride, buf.size), "d2h")
            self.ctx.sync()
            crcs.append(zlib.crc32(buf.tobytes()))
        return csz, crcs

    def free(self):
        self.d_in.free()
        self.d_comp.free()
        self.l.libdeflate_b200_device_free(self.ctx.h, self.d_csz)
        self.ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("lib_a")
    ap.add_argument("lib_b")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=3, help="timed launches per library, leg and round")
    ap.add_argument("--legs", default=",".join(name for name, *_ in LEGS))
    ap.add_argument("--data-class", type=int, default=0, choices=range(6), help="bench/synth.c class of the inputs")
    ap.add_argument("--out", default=None, help="directory for ab_deflate.json")
    args = ap.parse_args()
    try:
        gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        gpu = "unknown"
    synth = bench.load_synth()
    report = {"gpu": gpu, "lib_a": args.lib_a, "lib_b": args.lib_b, "data_class": args.data_class, "legs": {}}
    for name, level, n, chunk in LEGS:
        if name not in args.legs.split(","):
            continue
        pin = ctypes.create_string_buffer(n * chunk)
        synth.synth_fill(pin, chunk, 0, n, args.data_class, os.cpu_count() or 1)
        sides = [Side(args.lib_a, pin, n, chunk), Side(args.lib_b, pin, n, chunk)]
        del pin
        ms = [[], []]
        for _ in range(args.rounds):
            for k, s in enumerate(sides):
                ms[k].append(s.time(level, args.launches))
        sample = np.random.default_rng(7).choice(n, size=min(n, 64), replace=False)
        (csz_a, crc_a), (csz_b, crc_b) = (s.outputs(sample) for s in sides)
        for s in sides:
            s.free()
        leg = {"ms_a": [round(x, 2) for x in ms[0]], "ms_b": [round(x, 2) for x in ms[1]],
               "median_a": round(float(np.median(ms[0])), 2), "median_b": round(float(np.median(ms[1])), 2),
               "b_over_a": round(float(np.median(ms[1]) / np.median(ms[0])), 4),
               "sizes_identical": bool((csz_a == csz_b).all()), "sample_streams_identical": crc_a == crc_b,
               "ratio": round(float(csz_b.sum()) / (n * chunk), 4)}
        report["legs"][name] = leg
        print(name, json.dumps(leg), flush=True)
    print(json.dumps(report))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        name = "ab_deflate.json" if args.data_class == 0 else "ab_deflate_class%d.json" % args.data_class
        with open(os.path.join(args.out, name), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
