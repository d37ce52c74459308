"""What collecting an index costs a decompress stream (DESIGN.md section 4.10), and how fast its host-window index
reads.

    python scripts/bench_index_stream.py [--mib 1024] [--reps 3] [--out DIR]
    python scripts/bench_index_stream.py --gib N [--out DIR]

--mib MiB of bench/synth.c class T as gzip L6, twice: from compress_large (points at sync points) and from Python
zlib (points at found block starts and at write boundaries).  Per stream, device-resident and fed in 64 MiB
device-form writes, with the card's name and power limit read in the same run:
  * output GB/s of a plain decompress stream and of indexed ones at spacings of 256 KiB, 1 MiB and 4 MiB: host
    clock around all the writes of one stream, each write waited for (best of --reps);
  * the index's points and host window bytes;
  * random 64 KiB reads (seeded, uniform offsets) in batches of 64: reads per second of one device-form extract
    call per batch, from the stream's host-window index and from the same blob loaded with device windows
    (best of --reps).

--gib N streams N GiB of class T (one 64 MiB piece, repeated) through a device-form gzip compress stream at L6,
64 MiB per write, and every compressed write straight into a plain and three indexed decompress streams, so that
neither the output nor the stream is ever stored: the output GB/s of each (decompress writes only) and the host
window bytes.  Reads need the compressed stream, which this mode does not keep, so it measures none.
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
WRITE = 64 << 20
READ = 65536
BATCH = 64


def best_of(reps, fn):
    best = None
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        dt = time.perf_counter() - t
        best = dt if best is None else min(best, dt)
    return best


class Stream:
    """One device-form decompress stream (spacing None: plain)."""

    def __init__(self, ctx, spacing):
        self.ctx, self.l = ctx, ctx.l
        self.h = (self.l.libdeflate_b200_decompress_stream_create(ctx.h, GZ) if spacing is None
                  else self.l.libdeflate_b200_decompress_stream_create_indexed(ctx.h, GZ, spacing))
        assert self.h
        self.total, self.res, self.seconds = 0, ldb.MORE_INPUT, 0.0

    def write(self, d_in, n, last, d_out, room):
        """Writes n bytes at d_in, the output at d_out (room bytes); the output bytes."""
        w, need, unused, res = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int32(0)
        t = time.perf_counter()
        self.ctx._check(self.l.libdeflate_b200_decompress_stream_write(self.h, d_in, n, 1 if last else 0, d_out, room, ctypes.byref(w),
                                                                       ctypes.byref(need), ctypes.byref(unused), ctypes.byref(res)),
                        "decompress_stream_write")
        self.ctx.sync()
        self.seconds += time.perf_counter() - t
        assert res.value in (ldb.SUCCESS, ldb.MORE_INPUT), res.value
        self.res = res.value
        self.total += w.value
        return w.value

    def take(self):
        ix = self.l.libdeflate_b200_decompress_stream_take_index(self.h)
        assert ix, self.l.libdeflate_b200_last_error()
        return ix

    def close(self):
        self.l.libdeflate_b200_decompress_stream_destroy(self.h)


def feed(ctx, dz, zn, dout, n, spacing):
    """The whole device-resident stream in WRITE-byte writes: (seconds, index handle or None)."""
    s = Stream(ctx, spacing)
    for off in range(0, zn, WRITE):
        c = min(WRITE, zn - off)
        s.write(dz + off, c, off + c == zn, dout + s.total, n - s.total)
    assert s.res == ldb.SUCCESS and s.total == n
    ix = s.take() if spacing is not None else None
    s.close()
    return s.seconds, ix


def reads_per_s(ctx, ix, dz, zn, dx, n, reps, rng):
    ranges = [(rng.randrange(n - READ), READ) for _ in range(BATCH)]
    offs = (ctypes.c_uint64 * BATCH)(*[o for o, _ in ranges])
    lens = (ctypes.c_size_t * BATCH)(*[ln for _, ln in ranges])
    dst = (ctypes.c_void_p * BATCH)(*[dx + i * READ for i in range(BATCH)])
    res = (ctypes.c_int32 * BATCH)()

    def call():
        ctx._check(ctx.l.libdeflate_b200_index_extract(ctx.h, ix, dz, zn, offs, lens, dst, res, BATCH), "index_extract")
        assert all(r == 0 for r in res), list(res)[:8]
    call()
    return round(BATCH / best_of(reps, call), 1)


def blob_of(ctx, ix):
    nb = ctx.l.libdeflate_b200_index_serialized_size(ix)
    buf = ctypes.create_string_buffer(nb)
    ctx._check(ctx.l.libdeflate_b200_index_serialize(ix, buf, nb), "index_serialize")
    return buf


def stream_row(ctx, z, hb, reps):
    l, n, zn = ctx.l, len(hb), len(z)
    dz, dout, dx = Dev(ctx, zn), Dev(ctx, n), Dev(ctx, BATCH * READ)
    ctx._check(l.libdeflate_b200_memcpy_h2d(ctx.h, dz.p, z, zn), "h2d")
    ctx.sync()
    row = {"ratio": round(zn / n, 5), "writes": (zn + WRITE - 1) // WRITE}
    feed(ctx, dz.p, zn, dout.p, n, None)
    t_plain = best_of(reps, lambda: feed(ctx, dz.p, zn, dout.p, n, None))
    row["plain_GB/s"] = round(n / t_plain / 1e9, 2)
    row["spacings"] = {}
    rng = random.Random(1)
    for sp in SPACINGS:
        t, ix = None, None
        for _ in range(reps):
            dt, k = feed(ctx, dz.p, zn, dout.p, n, sp)
            if t is None or dt < t:
                t = dt
            if ix is None:
                ix = k
            else:
                l.libdeflate_b200_index_destroy(k)
        same = np.empty(n, np.uint8)
        ctx._check(l.libdeflate_b200_memcpy_d2h(ctx.h, same.ctypes.data, dout.p, n), "d2h")
        ctx.sync()
        assert same.tobytes() == hb, "the indexed stream's output differs"
        pts = l.libdeflate_b200_index_points(ix)
        r = {"points": pts, "host_window_bytes": (pts - 1) * 32768, "indexed_GB/s": round(n / t / 1e9, 2),
             "indexed_over_plain": round(t_plain / t, 3)}
        blob = blob_of(ctx, ix)
        dev = l.libdeflate_b200_index_load(ctx.h, blob, len(blob))
        assert dev
        r["reads_per_s_host_windows"] = reads_per_s(ctx, ix, dz.p, zn, dx.p, n, reps, rng)
        r["reads_per_s_device_windows"] = reads_per_s(ctx, dev, dz.p, zn, dx.p, n, reps, rng)
        l.libdeflate_b200_index_destroy(dev)
        l.libdeflate_b200_index_destroy(ix)
        row["spacings"]["%d_KiB" % (sp >> 10)] = r
        print("  spacing %d KiB: %s" % (sp >> 10, json.dumps(r)), flush=True)
    for d in (dz, dout, dx):
        d.free()
    return row


def gib_row(ctx, gib):
    """N GiB through a compress stream into four decompress streams, nothing stored."""
    l = ctx.l
    piece = synth(WRITE, 0)
    cs = l.libdeflate_b200_compress_stream_create(ctx.h, GZ, 6)
    assert cs
    bound = l.libdeflate_b200_compress_stream_bound(cs, 2 * WRITE, ldb.FINISH)    # (a write also flushes what earlier ones held)
    din, dc, dout, dn = Dev(ctx, WRITE), Dev(ctx, bound), Dev(ctx, 2 * WRITE + (1 << 20)), Dev(ctx, 8)
    ctx._check(l.libdeflate_b200_memcpy_h2d(ctx.h, din.p, piece.ctypes.data, WRITE), "h2d")
    ctx.sync()
    streams = {"plain": Stream(ctx, None)}
    for sp in SPACINGS:
        streams["%d_KiB" % (sp >> 10)] = Stream(ctx, sp)
    pieces = gib * ((1 << 30) // WRITE)
    zn_total = 0
    for i in range(pieces):
        last = i + 1 == pieces
        cn = ctypes.c_size_t(0)
        # (the output size is written on the device: d_out_nbytes is a device pointer)
        ctx._check(l.libdeflate_b200_compress_stream_write(cs, din.p, WRITE, ldb.FINISH if last else ldb.NO_FLUSH, dc.p, bound, dn.p),
                   "compress_stream_write")
        ctx._check(l.libdeflate_b200_memcpy_d2h(ctx.h, ctypes.byref(cn), dn.p, 8), "d2h")
        ctx.sync()
        zn_total += cn.value
        for s in streams.values():
            # (all the output a write delivers fits: the held input is at most one write's, which decodes to
            # less than 2 x 64 MiB of class T)
            s.write(dc.p, cn.value, last, dout.p, 2 * WRITE + (1 << 20))
    l.libdeflate_b200_compress_stream_destroy(cs)
    n = pieces * WRITE
    row = {"output_bytes": n, "compressed_bytes": zn_total}
    for name, s in streams.items():
        assert s.res == ldb.SUCCESS and s.total == n, (name, s.res, s.total)
        r = {"GB/s": round(n / s.seconds / 1e9, 2)}
        if name != "plain":
            ix = s.take()
            pts = l.libdeflate_b200_index_points(ix)
            r.update(points=pts, host_window_bytes=(pts - 1) * 32768, indexed_over_plain=round(streams["plain"].seconds / s.seconds, 3))
            l.libdeflate_b200_index_destroy(ix)
        s.close()
        row[name] = r
        print("  %s: %s" % (name, json.dumps(r)), flush=True)
    for d in (din, dc, dout, dn):
        d.free()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--gib", type=int, default=0, help="stream this many GiB through a compress stream instead")
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()
    name, power = card()
    ctx = ldb.Context(0)
    res = {"card": name, "power_limit": power, "class": "T", "format": "gzip", "level": 6, "write_mib": WRITE >> 20}
    print("card: %s, power limit %s" % (name, power), flush=True)
    if args.gib:
        res["gib"] = args.gib
        res["streams"] = gib_row(ctx, args.gib)
    else:
        n = args.mib << 20
        res["output_mib"] = args.mib
        res["streams"] = {}
        hb = synth(n, 0).tobytes()
        co = zlib.compressobj(6, zlib.DEFLATED, 31)
        for label, z in (("compress_large", lambda: ctx.compress_large(hb, 6, GZ)), ("zlib_no_sync", lambda: co.compress(hb) + co.flush())):
            print("%s:" % label, flush=True)
            res["streams"][label] = stream_row(ctx, z(), hb, args.reps)
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_index_stream%s.json" % ("_gib" if args.gib else "")), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
