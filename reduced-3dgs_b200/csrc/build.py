"""Build libgs_b200.so (the C-ABI library of include/gs_b200.h) for sm_90a (H100), in-tree.

    python reduced-3dgs_b200/csrc/build.py [--force] [--verbose]

nvcc cross-compiles without a GPU.  The .so lands in reduced-3dgs_b200/gs_b200/ (git-ignored).  -lineinfo keeps profiler
source views usable; no --use_fast_math (parity needs IEEE div/sqrt).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(os.path.dirname(HERE), "gs_b200")
SO = os.path.join(OUT_DIR, "libgs_b200.so")
SOURCES = ["gsb_api.cu", "gsb_preprocess.cu", "gsb_binning.cu", "gsb_render.cu", "gsb_backward.cu", "gsb_tools.cu", "gsb_kmeans.cu", "gsb_knn.cu", "gsb_loss.cu", "gsb_adam.cu", "gsb_densify.cu", "gsb_deterministic.cu", "gsb_mercy.cu", "gsb_features.cu", "gsb_mcmc.cu"]
HEADERS = ["gsb_common.cuh", os.path.join("..", "..", "include", "gs_b200.h")]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]


def nvcc() -> str:
    """nvcc from PATH, else from $CUDA_HOME / $CUDA_PATH / /usr/local/cuda (a plain user shell often lacks the CUDA bin dir)."""
    found = shutil.which("nvcc")
    if found:
        return found
    for root in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if root and os.path.isfile(os.path.join(root, "bin", "nvcc")):
            return os.path.join(root, "bin", "nvcc")
    raise FileNotFoundError("nvcc not found: put the CUDA toolkit's bin directory on PATH or set CUDA_HOME")


def build(force: bool = False, verbose: bool = False, extra_flags=()) -> str:
    srcs = [os.path.join(HERE, s) for s in SOURCES]
    deps = srcs + [os.path.join(HERE, h) for h in HEADERS] + [os.path.abspath(__file__)]
    if not force and os.path.isfile(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return SO
    obj_dir = os.path.join(HERE, "build")
    os.makedirs(obj_dir, exist_ok=True)
    objs = [os.path.join(obj_dir, os.path.basename(s) + ".o") for s in srcs]

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode != 0:
            sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))

    with ThreadPoolExecutor(max_workers=len(srcs)) as ex:
        list(ex.map(run, [[nvcc(), "-c", s, "-o", o] + NVCC_FLAGS + list(extra_flags) for s, o in zip(srcs, objs)]))
    run([nvcc(), "-shared", "-o", SO] + objs + ARCH + ["-Xcompiler", "-fPIC", "-lcudart"])
    return SO


if __name__ == "__main__":
    flags = ["-Xptxas", "-v"] if "--verbose" in sys.argv else []
    print(build(force="--force" in sys.argv or "--verbose" in sys.argv, verbose="--verbose" in sys.argv, extra_flags=flags))
