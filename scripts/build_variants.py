"""Builds instrumented variant libraries (extra -D switches) under build/variants/; scripts/variant_bench.py runs them.
Dev tooling only; the product library is always libdeflate_b200/libdeflate_b200.so."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from libdeflate_b200 import build as b  # noqa: E402

VARIANTS = {
    "timing": ["-DLZ_TIMING"],
}


def main():
    outdir = os.path.join(ROOT, "build", "variants")
    os.makedirs(outdir, exist_ok=True)
    nvcc = "/usr/local/cuda/bin/nvcc"
    for name, defs in VARIANTS.items():
        objs = []
        for src in b.SOURCES:
            obj = os.path.join(outdir, "%s_%s.o" % (name, src.replace(".cu", "")))
            subprocess.check_call([nvcc] + [f for f in b.NVCC_FLAGS if f not in ("-Xptxas", "-v")] + defs + ["-c", os.path.join(b.CSRC, src), "-o", obj])
            objs.append(obj)
        so = os.path.join(outdir, "libdeflate_b200_%s.so" % name)
        subprocess.check_call([nvcc, "-shared", "-o", so] + objs + b.ARCH + ["-lcudart_static"])
        print(so)


if __name__ == "__main__":
    main()
