"""In-tree native builds: libetl_decode.so (nvcc, sm_90a — H100) and libwalgen.so (gcc).

Built artefacts live next to the sources (git-ignored).  nvcc cross-compiles sm_90a without a GPU, so the
library can be built, and the build checked, on a machine that has none.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from typing import List

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
INCLUDE = os.path.join(ROOT, "include")

# ETL_LIB_SUFFIX / ETL_NVCC_DEFS: build and load an experimental variant (kernel geometry sweeps)
DECODE_LIB = os.path.join(PKG, "libetl_decode%s.so" % os.environ.get("ETL_LIB_SUFFIX", ""))
WALGEN_LIB = os.path.join(PKG, "libwalgen.so")

NVCC_ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-O3",
              "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _stale(target: str, sources: List[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources if os.path.exists(s))


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA decode library cannot be built")


def decode_sources() -> List[str]:
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h", ".cpp")))


def build_decode(force: bool = False, verbose: bool = False) -> str:
    srcs = decode_sources() + [os.path.join(INCLUDE, "etl_decode.h")]
    if force or _stale(DECODE_LIB, srcs):
        cu = [s for s in srcs if s.endswith((".cu", ".cpp"))]
        cmd = [_nvcc()] + NVCC_ARCH + NVCC_FLAGS + os.environ.get("ETL_NVCC_DEFS", "").split() + ["-I", INCLUDE, "-I", CSRC, "-shared", "-o", DECODE_LIB] + cu + ["-lcudart"]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        log = os.path.join(PKG, "build_decode.log")
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + res.stdout)
        if verbose or res.returncode != 0:
            sys.stderr.write(res.stdout)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed (see {log})")
    return DECODE_LIB


def build_walgen(force: bool = False) -> str:
    src = os.path.join(CSRC, "walgen.c")
    if force or _stale(WALGEN_LIB, [src]):
        subprocess.check_call(["gcc", "-O3", "-march=x86-64-v3", "-std=c11", "-fPIC", "-shared", "-o", WALGEN_LIB, src, "-lm"])
    return WALGEN_LIB


def build_all(force: bool = False, verbose: bool = False):
    build_walgen(force)
    build_decode(force, verbose)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose=True)
    print("built", DECODE_LIB, WALGEN_LIB)
