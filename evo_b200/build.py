"""Builds evo_b200/libevo_b200.so (sm_90a, H100) in-tree with nvcc.  No JIT cache: build() leaves the
library next to the sources, and the package loads it from there."""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libevo_b200.so")
SOURCES = ["api.cu", "elementwise.cu", "hyena.cu", "gemm_wgmma.cu", "gemm_smallm.cu", "attention.cu", "decode.cu", "sampler.cu", "ingest.cu", "pool.cu"]
# comparators for the GPU tests (cuBLASLt GEMM, CUDA-core attention): a separate library, never loaded by the product
TEST_SRC = os.path.join(HERE, "..", "tests", "support", "test_support.cu")
TEST_LIB = os.path.join(HERE, "..", "tests", "support", "libevo_b200_test.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--use_fast_math", "-Xptxas", "-v"]
# --use_fast_math would change erff/div rounding of the reference-faithful epilogues: keep IEEE there
FLAGS.remove("--use_fast_math")
FLAGS += os.environ.get("NVCC_EXTRA", "").split()      # experiment builds only (e.g. -DEVO_SMALLM_TRACE)


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    hdrs = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(HERE, "..", "include", "evo_b200.h"))
    stamp = os.path.join(OBJ, "stamp")
    dig = _digest(srcs + hdrs)
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB

    def cc(src):
        obj = os.path.join(OBJ, os.path.basename(src).replace(".cu", ".o"))
        r = subprocess.run([NVCC, *FLAGS, "-c", src, "-o", obj], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        with open(obj + ".ptxas.log", "w") as f:
            f.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(cc, srcs))
    r = subprocess.run([NVCC, "-shared", "-o", LIB, *objs, "-lcudart",
                        "-Xlinker", "-rpath", "-Xlinker", "/usr/local/cuda/lib64"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


def build_test_support(force: bool = False) -> str:
    """tests/support/libevo_b200_test.so: the comparators the GPU tests use (links cuBLASLt; the product does not)."""
    src = os.path.abspath(TEST_SRC)
    lib = os.path.abspath(TEST_LIB)
    stamp = lib + ".stamp"
    dig = _digest([src, os.path.join(HERE, "..", "include", "evo_b200.h")])
    if not force and os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read() == dig:
        return lib
    r = subprocess.run([NVCC, *[f for f in FLAGS if f not in ("-Xptxas", "-v")], "-shared", src, "-o", lib, "-lcudart", "-lcublasLt",
                        "-Xlinker", "-rpath", "-Xlinker", "/usr/local/cuda/lib64"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
    print(build_test_support(force="--force" in sys.argv))
