"""In-tree build of the sm_90a (H100) extension (``mlx_sharding_b200/ops/_b200_C.so``).

Kernel sources are plain CUDA (no torch headers) compiled by nvcc with
``-gencode arch=compute_90a,code=sm_90a -lineinfo``; only ``bindings.cpp`` sees torch.  nvcc
cross-compiles without a GPU, so the extension can be built on a machine without one; the ``.so`` and
the object directory are git-ignored build products.

``python -m mlx_sharding_b200.ops.build [--force] [--verbose]``
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_build")
MODULE = "_b200_C"
SO_PATH = os.path.join(HERE, MODULE + ".so")

CU_SOURCES = ["gemm_host.cu", "gemm_splitk.cu", "gemm_persistent.cu", "gemm_q_splitk.cu", "gemm_q_persistent.cu", "gemm_fp8.cu", "elementwise.cu", "attention.cu", "attention_prefill.cu", "mla_decode.cu", "moe.cu", "sampler.cu", "p2p.cu", "ep.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--use_fast_math",
                     "-Xptxas", "-v"]


def _nvcc() -> str:
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    return cand if os.path.exists(cand) else "nvcc"


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(p.encode())
            h.update(f.read())
    return h.hexdigest()


def _run(cmd, verbose):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"command failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    if verbose:
        sys.stderr.write(r.stdout + r.stderr)
    return r.stdout + r.stderr


def build(force: bool = False, verbose: bool = False) -> str:
    import torch
    from torch.utils import cpp_extension

    os.makedirs(OBJ, exist_ok=True)
    all_src = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    stamp = os.path.join(OBJ, "stamp.txt")
    dig = _digest(all_src) + torch.__version__
    if not force and os.path.exists(SO_PATH) and os.path.exists(stamp) and open(stamp).read() == dig:
        return SO_PATH

    logs = {}

    def compile_cu(name):
        out = os.path.join(OBJ, name.replace(".cu", ".o"))
        logs[name] = _run([_nvcc(), *NVCC_FLAGS, "-I", CSRC, "-c", os.path.join(CSRC, name), "-o", out], verbose)
        return out

    def compile_cpp():
        out = os.path.join(OBJ, "bindings.o")
        inc = []
        for p in cpp_extension.include_paths("cuda"):
            inc += ["-isystem", p]
        inc += ["-isystem", sysconfig.get_paths()["include"]]
        abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
        _run(["g++", "-O2", "-std=c++17", "-fPIC", f"-DTORCH_EXTENSION_NAME={MODULE}", f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
              "-DTORCH_API_INCLUDE_EXTENSION_H", "-I", CSRC, *inc, "-c", os.path.join(CSRC, "bindings.cpp"), "-o", out],
             verbose)
        return out

    with ThreadPoolExecutor(max_workers=8) as ex:
        futs = [ex.submit(compile_cu, n) for n in CU_SOURCES] + [ex.submit(compile_cpp)]
        objs = [f.result() for f in futs]
    libdirs = cpp_extension.library_paths("cuda")
    link = ["g++", "-shared", "-o", SO_PATH, *objs]
    for d in libdirs:
        link += ["-L", d, f"-Wl,-rpath,{d}"]
    link += ["-lc10", "-ltorch_cpu", "-ltorch", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart"]
    _run(link, verbose)
    with open(stamp, "w") as f:
        f.write(dig)
    with open(os.path.join(OBJ, "ptxas.log"), "w") as f:
        for k, v in logs.items():
            f.write(f"==== {k}\n{v}\n")
    return SO_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(p)
