"""Build driver for libdeflate_b200.so (the C-ABI library with the sm_90a kernels).

    python -m libdeflate_b200.build          # nvcc build, in-tree
    python -m libdeflate_b200.build --emu    # g++ build against tests/emu (CPU logic tests only)

The product library is ALWAYS the nvcc build; the --emu artefact lives under
tests/emu/_build/ and is never imported by the package.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["shim.cu", "checksum_kernels.cu", "inflate_kernel.cu", "inflate_resolve.cu", "deflate_kernel.cu", "pack_kernels.cu", "large_kernels.cu", "large_inflate.cu"]
HEADERS = ["ldb_common.cuh", "deflate_lz_kernel.cuh", "deflate_block.cuh", "deflate_parse.cuh"]
LIB = os.path.join(HERE, "libdeflate_b200.so")
EMU_DIR = os.path.join(ROOT, "tests", "emu")
EMU_LIB = os.path.join(EMU_DIR, "_build", "libdeflate_b200_emu.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]     # H100 (Hopper)
NVCC_FLAGS = ARCH + [
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden", "--use_fast_math", "-Xptxas", "-v",
]


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _deps():
    d = [os.path.join(CSRC, f) for f in SOURCES + HEADERS]
    d += [os.path.join(ROOT, "include", "libdeflate.h"), os.path.join(ROOT, "include", "libdeflate_b200.h")]
    return d


def build(verbose=False, force=False):
    """Compile every .cu for sm_90a and link libdeflate_b200.so in-tree."""
    if not force and not _newer(LIB, _deps() + [os.path.abspath(__file__)]):
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    logs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        logs.append("== %s ==\n%s" % (src, out))
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError("nvcc failed on %s" % src)
    with open(os.path.join(HERE, "build", "ptxas.log"), "w") as f:
        f.write("\n".join(logs))
    if verbose:
        print("\n".join(logs))
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ARCH + ["-lcudart_static", "-Xlinker", "--exclude-libs,ALL"]
    subprocess.check_call(cmd)
    return LIB


def build_emu(force=False):
    """g++ build of the same sources against the SIMT emulator (tests only)."""
    deps = _deps() + [os.path.join(EMU_DIR, f) for f in ("cuda_emu.h", "cuda_emu.cpp", "alloc_probe.cpp")]
    if not force and not _newer(EMU_LIB, deps):
        return EMU_LIB
    os.makedirs(os.path.dirname(EMU_LIB), exist_ok=True)
    objs = []
    procs = []
    common = ["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-DLDB_EMU", "-I", EMU_DIR, "-include", "cuda_emu.h",
              "-Wno-unused-function", "-fno-strict-aliasing"] + os.environ.get("LDB_EMU_DEFS", "").split()	# (-D switches of an instrumented build, e.g. -DINF_STATS)
    for src in SOURCES:
        obj = os.path.join(os.path.dirname(EMU_LIB), src.replace(".cu", ".emu.o"))
        procs.append(subprocess.Popen(common + ["-x", "c++", "-c", os.path.join(CSRC, src), "-o", obj]))
        objs.append(obj)
    for src in ("cuda_emu.cpp", "alloc_probe.cpp"):
        obj = os.path.join(os.path.dirname(EMU_LIB), src.replace(".cpp", ".o"))
        procs.append(subprocess.Popen(common + ["-c", os.path.join(EMU_DIR, src), "-o", obj]))
        objs.append(obj)
    for p in procs:
        if p.wait() != 0:
            raise RuntimeError("emu build failed")
    subprocess.check_call(["g++", "-shared", "-o", EMU_LIB] + objs + ["-lpthread"])
    return EMU_LIB


if __name__ == "__main__":
    if "--emu" in sys.argv:
        print(build_emu(force="--force" in sys.argv))
    else:
        print(build(verbose="-v" in sys.argv, force="--force" in sys.argv))
