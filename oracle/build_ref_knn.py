"""Build the UNMODIFIED reference kNN extension (submodules/simple-knn, the module `simple_knn._C`) into oracle/_ref/_refKnn.so
(test infrastructure only; next to _refC.so, which oracle/build_ref.py makes).

The translation units spatial.cu, simple_knn.cu and ext.cpp are compiled where they lie (no sources are copied) with the flags
torch's BuildExtension passes for the reference's setup.py (setup.py:21-31: no extra nvcc flags; arch = the GPU's: sm_90 on H100),
plus one forced include: simple_knn.cu uses FLT_MAX without including <cfloat>, which CUDA 12.9's headers no longer pull in
transitively (nvcc stops with `identifier "FLT_MAX" is undefined`), so `-include cfloat` supplies it — the same kind of fix as the
`-include cstdint` of the rasterizer's build.

Output (git-ignored):
    oracle/_ref/_refKnn.so    pybind module with the reference's three entry points (ext.cpp:16-18): distCUDA2, distIndex2, distIndexQ

Uses: tests/golden/make_golden_knn.py and tools/bench_knn.py.  Never used by the product.
"""
from __future__ import annotations

import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_ref  # noqa: E402

SKNN = os.path.join(build_ref.REF, "submodules", "simple-knn")
OUT = os.path.join(HERE, "_ref")
SO = os.path.join(OUT, "_refKnn.so")


def reference_available() -> bool:
    return os.path.isfile(os.path.join(SKNN, "simple_knn.cu"))


def build(force: bool = False, verbose: bool = False) -> str | None:
    """Returns the path of the built module, or None when the reference sources are absent."""
    if not reference_available():
        return SO if os.path.isfile(SO) else None
    srcs = [os.path.join(SKNN, f) for f in ("spatial.cu", "simple_knn.cu", "ext.cpp")]
    deps = srcs + [os.path.join(SKNN, h) for h in ("spatial.h", "simple_knn.h")] + [__file__]
    if not force and os.path.isfile(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return SO
    obj_dir = os.path.join(OUT, "obj_knn")
    os.makedirs(obj_dir, exist_ok=True)
    from torch.utils import cpp_extension as ce
    import torch
    inc = []
    for p in ce.include_paths("cuda") if "device_type" in ce.include_paths.__code__.co_varnames else ce.include_paths(True):
        inc += ["-I", p]
    inc += ["-I", sysconfig.get_paths()["include"], "-I", SKNN]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    common = ["-std=c++17", "-DTORCH_EXTENSION_NAME=_refKnn", "-DTORCH_API_INCLUDE_EXTENSION_H", f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
              "-include", "cstdint",
              "-include", "cfloat"]       # simple_knn.cu uses FLT_MAX without <cfloat>; CUDA 12.9 no longer provides it indirectly
    nvcc_flags = ["-gencode", "arch=compute_90,code=sm_90", "--expt-relaxed-constexpr",
                  "-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__",
                  "-D__CUDA_NO_BFLOAT16_CONVERSIONS__", "-D__CUDA_NO_HALF2_OPERATORS__",
                  "--compiler-options", "-fPIC"]
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    objs, cmds = [], []
    for s in srcs:
        o = os.path.join(obj_dir, os.path.basename(s) + ".o")
        objs.append(o)
        if s.endswith(".cu"):
            cmds.append([nvcc, "-c", s, "-o", o] + common + nvcc_flags + inc)
        else:
            cmds.append(["g++", "-c", s, "-o", o, "-O2", "-fPIC"] + common + inc)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("reference kNN build failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose:
            print(" ".join(cmd[:4]), "... ok", flush=True)

    with ThreadPoolExecutor(max_workers=len(cmds)) as ex:
        list(ex.map(run, cmds))
    libdir = os.path.join(os.path.dirname(torch.__file__), "lib")
    run(["g++", "-shared", "-o", SO] + objs + ["-L", libdir, "-L", "/usr/local/cuda/lib64", "-lc10", "-ltorch_cpu", "-ltorch",
                                              "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart", f"-Wl,-rpath,{libdir}"])
    return SO


def load():
    """Import oracle/_ref/_refKnn.so (build first if the reference tree is present). None if unavailable."""
    path = build()
    if path is None or not os.path.isfile(path):
        return None
    import importlib.util
    import torch  # noqa: F401  (libtorch must be loaded before the extension)
    spec = importlib.util.spec_from_file_location("_refKnn", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print("reference kNN module:", build(force="--force" in sys.argv, verbose=True))
