"""Build libovg.so for sm_90a (H100) with nvcc (cross-compiles without a GPU).  In-tree output so the .so travels with the
repo snapshot to the GPU box."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "ovg.cu")
OUT = os.path.join(HERE, "libovg.so")
DEPS = sorted(os.path.join(HERE, "csrc", f) for f in os.listdir(os.path.join(HERE, "csrc"))
              if f.endswith((".cu", ".cuh", ".inc", ".h"))) + [os.path.join(os.path.dirname(HERE), "include", "ovg.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-shared",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in DEPS):
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, *NVCC_FLAGS, "-o", OUT, SRC]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed building libovg.so")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
