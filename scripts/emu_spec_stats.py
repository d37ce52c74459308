"""Speculation rounds of the deflate parse per pass, on the CPU emulator build with -DLZ_SPEC_STATS (dev tooling).

    python scripts/emu_spec_stats.py [--chunks 2] [--size 65536] [--levels 1,6,9,12] [--classes 0,1,2,3,4,5] [-DLZ_...]

For every bench/synth.c class and level: how many parsed passes settled in round r (round 1: every
window's guessed entry of round 0 was right; a window whose entry changes walks again) and how many
needed the in-order tail after LZ_SPEC_ROUNDS rounds.  Classes 'a'.. name the inputs of
tests/golden/make_parse_digests.py, built to keep speculative walks apart.
"""
import argparse
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=2)
    ap.add_argument("--size", type=int, default=65536)
    ap.add_argument("--levels", default="1,6,9,12")
    ap.add_argument("--classes", default="0,1,2,3,4,5")
    ap.add_argument("--rounds", type=int, default=8, help="LZ_SPEC_ROUNDS of the build (set it with -DLZ_SPEC_ROUNDS=)")
    args, defs = ap.parse_known_args()
    os.environ["LDB_EMU_DEFS"] = " ".join(["-DLZ_SPEC_STATS"] + [d for d in defs if d.startswith("-D")])
    import libdeflate_b200 as ldb
    from libdeflate_b200 import build
    import bench
    import make_parse_digests as mpd
    lib = ldb.load_library(build.build_emu(force=True))
    ctx = ldb.Context(0, lib)
    synth = bench.load_synth()
    st = (ctypes.c_ulonglong * 16)()
    print("class level  passes  by round 1..R, then tail")
    for cls in args.classes.split(","):
        if cls.isdigit():
            buf = ctypes.create_string_buffer(args.size * args.chunks)
            synth.synth_fill(buf, args.size, 0, args.chunks, int(cls), 1)
            chunks = [buf.raw[i * args.size:(i + 1) * args.size] for i in range(args.chunks)]
        else:
            chunks = [mpd.INPUTS[cls](args.size, i) for i in range(args.chunks)]
        for level in [int(x) for x in args.levels.split(",")]:
            lib.ldb_lz_spec_stats(st, 1)
            ctx.compress_batch_host(chunks, level, ldb.RAW)
            lib.ldb_lz_spec_stats(st, 1)
            v = list(st)
            print("%5s %5d %7d  %s | %d" % (cls, level, sum(v), " ".join("%d" % x for x in v[1:args.rounds + 1]), v[args.rounds + 1]),
                  flush=True)
    os.environ.pop("LDB_EMU_DEFS")
    build.build_emu(force=True)	# leave the plain emulator build behind for the tests


if __name__ == "__main__":
    main()
