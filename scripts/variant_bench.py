"""Runs bench.py's decompress workload against a variant library (tuning only)."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import libdeflate_b200 as ldb  # noqa: E402

name = sys.argv[1]
ldb._lib = ldb.load_library(os.path.join(ROOT, "build", "variants", "libdeflate_b200_%s.so" % name))
import bench  # noqa: E402
if len(sys.argv) > 4:
    bench.LEVEL = int(sys.argv[4])

a = argparse.Namespace(gpus=1, steps=3, warmup=3, impl="b200", workload=sys.argv[2] if len(sys.argv) > 2 else "decompress",
                       chunks=int(sys.argv[3]) if len(sys.argv) > 3 else 32768, chunk_size=int(sys.argv[5]) if len(sys.argv) > 5 else 65536, no_e2e=True, no_cpu=True, no_extra=True, no_l12=True, no_origin=True, data_class=0,
                       dump_outputs=None)
bench.run_b200(a)
try:
    ldb._lib.ldb_lz_timing_dump()
except AttributeError:
    pass
