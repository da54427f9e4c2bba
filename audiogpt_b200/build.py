"""Build libagpt_b200.so in-tree with nvcc for sm_90a (no torch types in the ABI).

    python -m audiogpt_b200.build          # incremental
    python -m audiogpt_b200.build --force

The .so lands next to this file (git-ignored), so the package imports from the source tree.
"""
from __future__ import annotations

import glob
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libagpt_b200.so")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-O3",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _sig(path: str, deps: list) -> str:
    h = hashlib.sha1()
    h.update(" ".join(NVCC_FLAGS).encode())
    for p in [path] + deps:
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    hdrs = sorted(glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) +
                  glob.glob(os.path.join(HERE, "..", "include", "*.h")))
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()
    todo, objs = [], []
    for s in srcs:
        o = os.path.join(OBJ, os.path.basename(s)[:-3] + ".o")
        sigf = o + ".sig"
        sig = _sig(s, hdrs)
        objs.append(o)
        if force or not os.path.exists(o) or not os.path.exists(sigf) or open(sigf).read() != sig:
            todo.append((s, o, sigf, sig))

    def compile_one(job):
        s, o, sigf, sig = job
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        with open(sigf, "w") as f:
            f.write(sig)

    if todo:
        with ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            list(ex.map(compile_one, todo))
    if todo or not os.path.exists(LIB):
        cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
