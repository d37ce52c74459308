"""Tuning sweeps: builds variant libraries (different -D geometry) under build/variants/.
Dev tooling only; the product library is always libdeflate_b200/libdeflate_b200.so."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from libdeflate_b200 import build as b  # noqa: E402

GEO_A = ["-DINF_LB=8", "-DINF_LSUB_SM=64", "-DINF_OB=6", "-DINF_OSUB_SM=64"]      # 896 B/lane, 7 warps/SM (default)
GEO_G = ["-DINF_LB=7", "-DINF_LSUB_SM=96", "-DINF_OB=6", "-DINF_OSUB_SM=64"]      # 704 B, 9 warps
GEO_C = ["-DINF_LB=7", "-DINF_LSUB_SM=64", "-DINF_OB=5", "-DINF_OSUB_SM=32"]      # 512 B, 13 warps
GEO_D = ["-DINF_LB=7", "-DINF_LSUB_SM=32", "-DINF_OB=5", "-DINF_OSUB_SM=32"]      # 448 B, 15 warps
VARIANTS = {
    "timing": ["-DLZ_TIMING"],
    "nofuse": ["-DINF_FUSE_OFF=0"],     # offset decoded in its own step
    "fuse_lit3": ["-DINF_LIT2=2"],
    "lit6": ["-DINF_LIT2=6"],           # up to six follow-on literals (default four)
    "g6": ["-DINF_LSUB_SM=16", "-DINF_OB=6", "-DINF_OSUB_SM=16"],      # 6-bit main offset table: more matches take the fused path
    "g6lit6": ["-DINF_LSUB_SM=16", "-DINF_OB=6", "-DINF_OSUB_SM=16", "-DINF_LIT2=6"],
}
# other knobs a sweep can set: -DRES_PER_SM (resolve warps per SM), -DINF_QUANTUM (decode steps between service phases),
# -DLZ_QUANTUM (resumable chain walk of the deflate search), -DINF_WQ2=1 (two-slot asynchronous lookahead)


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
