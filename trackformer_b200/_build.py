"""In-tree build of the native pieces (explicit nvcc / g++ -- no JIT cache, no setuptools).

Artefacts (git-ignored, shipped to the GPU box by gpurun):
  trackformer_b200/libmsda_b200.so                    C-ABI library (include/msda_b200.h), cudart linked statically
  trackformer_b200/MultiScaleDeformableAttention.so   pybind11/torch glue importing under the reference's module name

The reference builds its extension with a CUDAExtension and *no* -gencode flags
(src/trackformer/models/ops/setup.py:34-39) and refuses to build without a visible GPU
(:40-41); here nvcc cross-compiles for sm_90a (H100) explicitly, GPU or not.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB_SO = os.path.join(HERE, "libmsda_b200.so")
EXT_SO = os.path.join(HERE, "MultiScaleDeformableAttention.so")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc() -> str:
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    return cand if os.path.exists(cand) else (shutil.which("nvcc") or "nvcc")


def _newer(target: str, sources) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _public_headers():
    inc = os.path.join(ROOT, "include")
    return [os.path.join(inc, f) for f in sorted(os.listdir(inc)) if f.endswith(".h")]


def _run(cmd, verbose):
    if verbose:
        print("+", " ".join(cmd), flush=True)
    subprocess.check_call(cmd)


def build_library(force: bool = False, verbose: bool = False) -> str:
    srcs = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".h"))]
    srcs += _public_headers()
    if not force and _newer(LIB_SO, [*srcs, __file__]):              # a change of the flags here rebuilds too
        return LIB_SO
    cu = [s for s in srcs if s.endswith(".cu")]
    _run([_nvcc(), "-O3", "-std=c++17", *GENCODE, "-lineinfo", "-Xcompiler", "-fPIC", "-shared",
          "-I", os.path.join(ROOT, "include"), "-o", LIB_SO, *cu], verbose)
    return LIB_SO


def build_extension(force: bool = False, verbose: bool = False) -> str:
    build_library(False, verbose)
    src = os.path.join(CSRC, "msda_torch.cpp")
    hdrs = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".h")]
    if not force and _newer(EXT_SO, [src, LIB_SO, __file__, *hdrs, *_public_headers()]):
        return EXT_SO
    import torch
    from torch.utils import cpp_extension as ce

    tlib = os.path.join(os.path.dirname(torch.__file__), "lib")
    cuda_home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    inc = [f"-I{p}" for p in ce.include_paths()] + [f"-I{sysconfig.get_paths()['include']}",
                                                    f"-I{os.path.join(cuda_home, 'include')}",
                                                    f"-I{os.path.join(ROOT, 'include')}"]
    abi = int(getattr(torch._C, "_GLIBCXX_USE_CXX11_ABI", True))
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", *inc,
           "-DTORCH_EXTENSION_NAME=MultiScaleDeformableAttention", "-DTORCH_API_INCLUDE_EXTENSION_H",
           f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-o", EXT_SO, src,
           f"-L{HERE}", "-lmsda_b200", f"-L{tlib}", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda",
           "-ltorch", "-ltorch_python", "-Wl,-rpath,$ORIGIN", f"-Wl,-rpath,{tlib}"]
    _run(cmd, verbose)
    return EXT_SO


def build_all(force: bool = False, verbose: bool = False):
    lib = build_library(force, verbose)
    return lib, build_extension(force, verbose)


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv, verbose=True))
