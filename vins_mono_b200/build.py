"""Builds libvinsb200.so (CUDA kernels + C ABI + host glue) in-tree for sm_90a (H100) with nvcc."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "libvinsb200.so")

# The front end must reproduce OpenCV's float arithmetic bit for bit: no FMA contraction there.  The back end is
# double precision checked to a tolerance, so its kernels (ba_*.cu, and the pose graph's pg_*.cu) keep nvcc's default
# contraction (DFMA).
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [*ARCH, "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC,-ffp-contract=off,-O2", "-I", os.path.join(ROOT, "include"), "-I", CSRC]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
           [os.path.join(ROOT, "include", "vinsb200", f) for f in os.listdir(os.path.join(ROOT, "include", "vinsb200"))]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    objs = []
    objdir = os.path.join(HERE, "lib", "obj")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        objs.append(obj)
        fmad = "--fmad=true" if os.path.basename(src).startswith(("ba_", "pg_")) else "--fmad=false"
        cmd = ["nvcc", *NVCC_FLAGS, fmad, "-x", "cu", "-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{out}")
        if verbose and out.strip():
            print(out)
    subprocess.check_call(["nvcc", *ARCH, "-shared", "-o", LIB, *objs])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
