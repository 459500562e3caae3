"""Build libcsnet_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache: the library sits next to its sources)."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libcsnet_b200.so")
SOURCES = ["plan.cu", "train_ops.cu", "train_csf.cu", "train_bf16.cu", "train_csf_bf16.cu", "bn_sync.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC,-O3,-Wall", "-shared", "-cudart", "shared"]


def nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; the CUDA toolkit is required to build libcsnet_b200.so")
    return exe


STAMP = LIB + ".srchash"


def source_hash() -> str:
    """sha256 over every source the library is built from (csrc/*, the C-ABI header) and the compiler flags: the rebuild
    decision is keyed on CONTENT, not on mtimes — a pushed .so that is newer than the sources but built from other sources
    (the snapshot that travels to the GPU box) is rebuilt, never silently reused."""
    import hashlib

    h = hashlib.sha256(" ".join(NVCC_FLAGS + SOURCES).encode())
    deps = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC)) + [os.path.join(HERE, "..", "include", "csnet_b200.h")]
    for d in deps:
        h.update(os.path.basename(d).encode())
        with open(d, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def needs_build() -> bool:
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    return open(STAMP).read().strip() != source_hash()


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    cmd = [nvcc(), *NVCC_FLAGS, *(["-Xptxas", "-v"] if verbose else []), "-o", LIB,
           *[os.path.join(CSRC, s) for s in SOURCES]]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    with open(STAMP, "w") as f:
        f.write(source_hash() + "\n")
    if verbose:
        print(res.stdout + res.stderr)
    return LIB


if __name__ == "__main__":
    import sys
    print(build(force=True, verbose="-v" in sys.argv))
