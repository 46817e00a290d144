"""Builds libsgp.so (CUDA kernels + C-ABI) in-tree for sm_90a (H100) with nvcc.  No JIT cache: the package loads the
.so from its own directory."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsgp.so")
SOURCES = ["api.cu", "bcm_nll.cu", "gram_f64.cu", "gram_i8.cu", "gram_i8_wgmma.cu", "greedy.cu", "kernel_eval.cu", "kmeans.cu", "kmn_sweep.cu", "laplace.cu", "laplace_global.cu", "misc_kernels.cu", "predict.cu", "scale.cu", "tail.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-Xptxas", "-v"]
LINK = ["-lcusolver", "-lcublas", "-ldl", "-Xlinker", "-rpath=/usr/local/cuda/lib64"]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "sgp.h"),
                                                                 os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build_native(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    log = []
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log.append(r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        objs.append(obj)
    cmd = [nvcc, "-shared", "-o", LIB, *objs, *LINK]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    with open(os.path.join(HERE, "build.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        sys.stderr.write("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build_native(force="--force" in sys.argv, verbose=True))
