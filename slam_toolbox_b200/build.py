"""In-tree build of libb200slam.so (sm_90a only).

nvcc cross-compiles without a GPU, so the library builds on machines without one.
The .so stays in-tree (slam_toolbox_b200/lib/, git-ignored): the package runs from the repository tree.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libb200slam.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-ffp-contract=off,-Wall"]
# translation units and their extra flags. The scan matcher's FP64 must round exactly like the
# reference's x86-64 build: no FMA contraction on device (-fmad=false) or host (-ffp-contract=off).
UNITS = {
    "scan_matcher.cu": ["-fmad=false"],
    "sm_sweep.cu": ["-fmad=false"],
    "sm_tile.cu": ["-fmad=false"],
    "pose_graph.cu": [],
    "pg_pcg.cu": [],
    "pg_cholesky.cu": [],
    "occupancy.cu": ["-fmad=false"],
}


def _newer(src: str, dst: str) -> bool:
    if not os.path.exists(dst):
        return True
    t = os.path.getmtime(dst)
    deps = [src] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    deps.append(os.path.join(HERE, "..", "include", "b200slam.h"))
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    nvcc = os.environ.get("NVCC", "nvcc")
    objs = []
    rebuilt = False
    for unit, extra in UNITS.items():
        src = os.path.join(CSRC, unit)
        obj = os.path.join(LIBDIR, unit.replace(".cu", ".o"))
        objs.append(obj)
        if force or _newer(src, obj):
            cmd = [nvcc] + ARCH + COMMON + extra + ["-c", src, "-o", obj]
            if verbose:
                print(" ".join(cmd), file=sys.stderr)
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed for {unit}:\n{r.stdout}\n{r.stderr}")
            rebuilt = True
    if rebuilt or not os.path.exists(LIB) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        cmd = [nvcc] + ARCH + ["-shared", "--cudart", "shared", "-Xlinker", "-rpath,/usr/local/cuda/lib64", "-o", LIB] + objs + ["-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
