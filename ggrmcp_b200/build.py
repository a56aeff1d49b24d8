"""Builds libggrmcp_b200.so (sm_90a only, for the H100) in-tree with nvcc.  No JIT, no other architectures.

One object per translation unit, compiled in parallel, then linked:
  ggr_engine.cu       host side of the C ABI + the block-sum scan kernel
  ggr_kernels_enc.cu  request-side kernels (JSON -> wire)
  ggr_kernels_dec.cu  reply-side kernels (wire -> JSON)
  ggr_kernels_coop.cu warp-cooperative reply-side kernels
  ggr_kernels_coop_enc.cu lock-step request-side parser (one warp per item)
  ggr_kernels_walk.cu token index + token-parallel walker of the request side (one warp per item)
  ggr_kernels_wrap.cu MCP result bodies around the protojson texts
  ggr_schema.cc       descriptor-table compiler (host)
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libggrmcp_b200.so")
UNITS = ["ggr_engine.cu", "ggr_kernels_enc.cu", "ggr_kernels_dec.cu", "ggr_kernels_coop.cu", "ggr_kernels_coop_enc.cu", "ggr_kernels_walk.cu", "ggr_kernels_wrap.cu", "ggr_schema.cc"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "-I" + os.path.join(os.path.dirname(HERE), "include")]


def units():
    return [u for u in UNITS if os.path.exists(os.path.join(CSRC, u))]


def deps():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(os.path.dirname(HERE), "include", "ggrmcp_b200.h")]


def stale(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in sources)


def build(force=False, verbose=False, only=None):
    os.makedirs(OBJ, exist_ok=True)
    headers = [d for d in deps() if d.endswith((".h", ".cuh"))]
    jobs = []
    objs = []
    for u in units():
        src = os.path.join(CSRC, u)
        obj = os.path.join(OBJ, u.rsplit(".", 1)[0] + ".o")
        objs.append(obj)
        if only and u not in only and os.path.exists(obj):
            continue
        if force or stale(obj, [src] + headers):
            cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj, src]
            print(" ".join(cmd), flush=True)
            jobs.append((u, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for u, p in jobs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            print("==== %s ====\n%s" % (u, out), flush=True)
        failed |= p.returncode != 0
    if failed:
        raise SystemExit("nvcc failed")
    if jobs or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB] + objs
        print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
