"""Builds pinot_b200/libpinot_b200.so in-tree with nvcc for sm_90a (no torch, no JIT cache: the .so travels with the repo).

    python -m pinot_b200.build            # incremental
    python -m pinot_b200.build --force
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_obj")
LIB = os.path.join(HERE, "libpinot_b200.so")
SCAN_KERNELS = ["w6_agg", "w8_agg", "w8_agg_nodefer", "w6_gb1", "w8_gb1", "w6_gb2", "w8_gb2"]  # one instantiation per TU
SOURCES = [f"pb200_scan_k_{k}.cu" for k in SCAN_KERNELS] + ["pb200_api.cu", "pb200_plan.cpp", "pb200_domain.cu", "pb200_extract.cu", "pb200_comm.cu", "pb200_roaring.cu", "pb200_synth.cu",
                                                             "host/plan_maker.cpp", "host/star_tree.cpp", "host/datatable.cpp", "host/segment_cache.cpp", "host/raw_forward.cpp", "host/filtered_agg.cpp"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "-Xptxas", "-v", "--expt-relaxed-constexpr"]


def _deps():
    out = []
    for root in (CSRC, os.path.join(CSRC, "host"), os.path.join(os.path.dirname(HERE), "include")):
        for f in os.listdir(root):
            if f.endswith((".cu", ".cuh", ".h", ".cpp", ".inc")):
                out.append(os.path.join(root, f))
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    newest = max(os.path.getmtime(p) for p in _deps())
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= newest:
        return LIB
    os.makedirs(OBJ, exist_ok=True)

    def compile_one(src):
        obj = os.path.join(OBJ, os.path.basename(src).replace(".cu", ".o").replace(".cpp", ".o"))
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(OBJ, os.path.basename(src).replace(".cu", ".ptxas.log").replace(".cpp", ".log"))
        with open(log, "w") as f:
            f.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 4)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    tmp = LIB + ".tmp"  # link beside the target, then rename: a reader (or a repo snapshot) never sees a half-written .so
    cmd = [NVCC, "-shared", "-o", tmp, *objs, "-cudart", "static", "-gencode", "arch=compute_90a,code=sm_90a", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
