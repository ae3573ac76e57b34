"""Build libsessd_b200.so (hand-written CUDA for sm_90a + the C ABI of include/sessd_b200.h) IN-TREE.

    python se-ssd_b200/build.py [--force]

nvcc cross-compiles without a GPU; the resulting .so and the objects under build/ are git-ignored.
Files that implement the rotated-box geometry are compiled with -fmad=false so that their fp32 arithmetic rounds
like the CPU twin of the reference (see csrc/rotbox.cuh).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libsessd_b200.so")
LAB_OUT = os.path.join(HERE, "libsessd_b200_lab.so")
# non-default operand formats (include/sessd_b200_lab.h): built into their own library, never loaded by the product path
LAB = {"bevconv_split.cu"}
OBJ = os.path.join(HERE, "build")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"] + os.environ.get("SESSD_DEFINES", "").split()
NO_FMA = {"iou3d.cu", "postproc.cu", "assign.cu", "odiou.cu", "kitti_eval.cu", "augment.cu", "gtaug.cu", "sada.cu", "kitti_prep.cu"}
# files whose host code evaluates the collision predicate of csrc/augment.cuh: the host compiler must not contract it into fmas either
HOST_NO_CONTRACT = {"augment.cu", "gtaug.cu"}


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def newest_dep():
    inc = os.path.join(os.path.dirname(HERE), "include")
    t = max(os.path.getmtime(os.path.join(inc, "sessd_b200.h")), os.path.getmtime(os.path.join(inc, "sessd_b200_lab.h")))
    for f in os.listdir(CSRC):
        t = max(t, os.path.getmtime(os.path.join(CSRC, f)))
    return t


def build(force=False, verbose=False):
    if (not force) and os.path.exists(OUT) and os.path.exists(LAB_OUT) and min(os.path.getmtime(OUT), os.path.getmtime(LAB_OUT)) >= newest_dep():
        return OUT
    os.makedirs(OBJ, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

    def compile_one(src):
        obj = os.path.join(OBJ, src[:-3] + ".o")
        cmd = [nvcc] + ARCH + COMMON + (["-fmad=false"] if src in NO_FMA else []) + \
            (["-Xcompiler", "-ffp-contract=off"] if src in HOST_NO_CONTRACT else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
        return obj

    srcs = sources()
    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(compile_one, srcs))
    prod = [o for o, f in zip(objs, srcs) if f not in LAB]
    lab = [o for o, f in zip(objs, srcs) if f in LAB]
    for out, group, extra in ((OUT, prod, []), (LAB_OUT, lab, ["-L" + HERE, "-l:libsessd_b200.so", "-Xlinker", "-rpath=$ORIGIN"])):
        cmd = [nvcc] + ARCH + ["-shared", "-o", out] + group + extra + ["-lcudart"]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
