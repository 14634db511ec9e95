"""Builds libytk_b200.so (the sm_90a CUDA kernels + C ABI) in-tree with nvcc.

nvcc cross-compiles without a GPU; the resulting .so and objects are git-ignored build products.
Run as `python -m yomitoku_b200.build` or through `__graft_entry__.build()`.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "csrc", "build")
LIB = os.path.join(HERE, "libytk_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


# OpenCV's float / double expressions are not contracted into FMAs: the bit-exact restatement in crop_math.h needs the
# same (csrc/crop_ops.cu header).  Pillow's resample coefficients are double arithmetic computed on the host
# (csrc/resample_ops.cu header): neither the device nor the host compiler may contract them.  The table parser's overlap
# ratios are fp64 restatements of Python arithmetic (csrc/table_ops.cu header).
EXTRA_FLAGS = {"crop_ops.cu": ["--fmad=false"],
               "resample_ops.cu": ["--fmad=false", "-Xcompiler", "-ffp-contract=off"],
               "table_ops.cu": ["--fmad=false"]}


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stamp():
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)):
        p = os.path.join(CSRC, f)
        if os.path.isfile(p) and f.split(".")[-1] in ("cu", "cuh", "h"):
            h.update(f.encode())
            h.update(open(p, "rb").read())
    h.update(open(os.path.join(HERE, "..", "include", "yomitoku_b200.h"), "rb").read())
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(repr(sorted(EXTRA_FLAGS.items())).encode())
    return h.hexdigest()


def _compile(src):
    obj = os.path.join(BUILD, src[:-3] + ".o")
    cmd = ["nvcc"] + NVCC_FLAGS + EXTRA_FLAGS.get(src, []) + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    return obj


def build(force=False, verbose=True):
    os.makedirs(BUILD, exist_ok=True)
    stamp_file = os.path.join(BUILD, "stamp")
    stamp = _stamp()
    if not force and os.path.exists(LIB) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return LIB
    srcs = _sources()
    if verbose:
        print("[yomitoku_b200.build] nvcc sm_90a: %s" % " ".join(srcs), flush=True)
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(_compile, srcs))
    cmd = ["nvcc", "-shared", "-o", LIB] + objs + ["-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    open(stamp_file, "w").write(stamp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
