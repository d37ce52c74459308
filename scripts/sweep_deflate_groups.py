"""Sweeps the parse/flush group sizes of the deflate kernel (LIBDEFLATE_B200_DEFLATE_GROUPS=Q,F,H) in one process.

    python scripts/sweep_deflate_groups.py LIB [--level 6] [--chunks 65536] [--q 4,6,8,10,12] [--f 12,14,16,18,20,24]
                                               [--h 12,16] [--rounds 2] [--launches 3] [--out DIR]

The library reads the variable at every launch, so one set of device buffers serves every setting.  Each round
times every (Q, F, H) once, in a fresh shuffled order, on bench/synth.c class 0 at 64 KiB chunks (gzip);
reported: deflate kernel ms per launch (library event pairs), median over rounds, and whether every setting's
compressed sizes and sample streams equal the first one's (they must: streams do not depend on the sizes).
"""
import argparse
import ctypes
import itertools
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ab_deflate as ab  # noqa: E402

ENV = "LIBDEFLATE_B200_DEFLATE_GROUPS"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("lib")
    ap.add_argument("--level", type=int, default=6)
    ap.add_argument("--chunks", type=int, default=65536)
    ap.add_argument("--q", default="4,6,8,10,12")
    ap.add_argument("--f", default="12,14,16,18,20,24")
    ap.add_argument("--h", default="12,16")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--launches", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    chunk = 65536
    synth = ab.bench.load_synth()
    pin = ctypes.create_string_buffer(args.chunks * chunk)
    synth.synth_fill(pin, chunk, 0, args.chunks, 0, os.cpu_count() or 1)
    side = ab.Side(args.lib, pin, args.chunks, chunk)
    del pin
    combos = list(itertools.product(*(map(int, s.split(",")) for s in (args.q, args.f, args.h))))
    sample = np.random.default_rng(7).choice(args.chunks, size=min(args.chunks, 64), replace=False)
    ms = {c: [] for c in combos}
    first, identical = None, True
    rng = np.random.default_rng(1)
    for r in range(args.rounds):
        for i in rng.permutation(len(combos)):
            c = combos[i]
            os.environ[ENV] = "%d,%d,%d" % c
            ms[c].append(side.time(args.level, args.launches))
            if r == 0:
                csz, crc = side.outputs(sample)
                if first is None:
                    first = (csz, crc)
                elif not ((csz == first[0]).all() and crc == first[1]):
                    identical = False
                    print("streams differ at", c, flush=True)
    os.environ.pop(ENV, None)
    side.free()
    rows = sorted(((float(np.median(v)), c, v) for c, v in ms.items()))
    for med, c, v in rows:
        print("Q=%2d F=%2d H=%2d  median %8.2f ms  rounds %s" % (c + (med, [round(x, 2) for x in v])))
    report = {"level": args.level, "chunks": args.chunks, "streams_identical": identical,
              "ms": {"%d,%d,%d" % c: [round(x, 3) for x in v] for c, v in ms.items()}}
    print(json.dumps({"best": "%d,%d,%d" % rows[0][1], "median_ms": round(rows[0][0], 2), "streams_identical": identical}))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sweep_groups_L%d.json" % args.level), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
