"""Builds libsimilari_b200.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc.

nvcc cross-compiles without a GPU; the built .so travels to the GPU box with the repo snapshot."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsimilari_b200.so")
SOURCES = ["engine.cu", "ops.cu", "kernels_cost.cu", "kernels_feat_tc.cu", "kernels_feat_dense.cu", "kernels_assign.cu", "kernels_state.cu", "kernels_nms.cu", "kernels_own.cu", "kernels_geom.cu", "kernels_xfer.cu", "comm.cu", "kernels_fstore.cu", "fstore.cu", "wasted_store.cu", "live_store.cu"]
HEADERS = ["sb_engine.cuh", "sb_math.cuh", "sb_own_area.cuh", "sb_tc.cuh", "sb_sincos.cuh", "sb_sincos_table.inc", "sb_fstore.cuh", "sb_host.cuh", "sb_blob.cuh", "sb_wstore.cuh", os.path.join("..", "..", "include", "similari_b200.h")]

# --fmad=false: the reference (Rust) never contracts a*b+c; parity of the i64 weights depends on it.
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--fmad=false",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fno-fast-math", "-Xptxas", "-v",
]


def nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found")
    return exe


def is_stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + [os.path.normpath(os.path.join(CSRC, h)) for h in HEADERS]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return LIB
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for s in SOURCES:
        o = os.path.join(objdir, s.replace(".cu", ".o"))
        cmd = [nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    logs = []
    for s, p in procs:
        out, _ = p.communicate()
        logs.append(f"==== {s}\n{out}")
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {s}:\n{out}")
    with open(os.path.join(objdir, "ptxas.log"), "w") as f:
        f.write("\n".join(logs))
    if verbose:
        print("\n".join(logs))
    cmd = [nvcc(), "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static", "-ldl"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    import sys

    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
