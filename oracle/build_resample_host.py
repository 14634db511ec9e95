"""Builds oracle/_build/libresample_host.so: the product's RT-DETRv2 input resize arithmetic
(yomitoku_b200/csrc/resample_math.h) compiled for the host with g++, for the CPU parity tests against Pillow.  TEST
INFRASTRUCTURE ONLY (see oracle/resample_host.cpp)."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build", "libresample_host.so")
SRC = os.path.join(HERE, "resample_host.cpp")
HDR = os.path.join(HERE, "..", "yomitoku_b200", "csrc", "resample_math.h")


def build(force=False):
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        return OUT
    cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", SRC, "-o", OUT]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ failed:\n%s\n%s" % (r.stdout, r.stderr))
    return OUT


if __name__ == "__main__":
    print(build(force=True))
