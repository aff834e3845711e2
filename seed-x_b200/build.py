"""Build libseedx.so (all CUDA sources under csrc/) for sm_90a with nvcc, in-tree.

Object files are cached per source under seed-x_b200/lib/obj and rebuilt when the source (or a header) is newer.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(LIBDIR, "obj")
LIB = os.path.join(LIBDIR, "libseedx.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "--use_fast_math" if False else "-DSEEDX_NO_FAST_MATH"]


def _newest_header():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(os.path.dirname(HERE), "include", "seedx.h"))
    return max(os.path.getmtime(h) for h in hs)


def build(verbose=False, force=False):
    os.makedirs(OBJDIR, exist_ok=True)
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdr_t = _newest_header()
    jobs = []
    objs = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJDIR, s[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_t):
            jobs.append([NVCC, *FLAGS, "-c", src, "-o", obj])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose and (r.stdout or r.stderr):
            print(r.stdout, r.stderr)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(run, jobs))
    if jobs or not os.path.exists(LIB):
        run([NVCC, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a"])
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
