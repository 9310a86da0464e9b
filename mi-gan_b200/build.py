"""Build the C-ABI shared library in-tree with nvcc for sm_90a (no torch dependency).

    python -m migan_b200.build          # or __graft_entry__.build()

Output: mi-gan_b200/lib/libmigan_b200.so (git-ignored build product).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIBPATH = os.path.join(LIBDIR, "libmigan_b200.so")
STAMP = os.path.join(LIBDIR, "libmigan_b200.stamp")

SOURCES = ["elementwise.cu", "gemm_simt.cu", "ops.cu", "sepconv_tc.cu", "abi_error.cu", "migan_abi.cu", "comodgan_abi.cu", "prepost.cu", "pipeline.cu", "demo_resize.cu", "fullres.cu", "holewin.cu", "masks.cu", "reparam.cu", "inception.cu", "inception_abi.cu", "lpips_abi.cu", "metrics.cu", "frechet.cu", "ids.cu", "kid.cu", "prdc.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def _source_hash() -> str:
    h = hashlib.sha256()
    files = sorted(os.listdir(CSRC)) + [os.path.join("..", "..", "include", "migan_b200.h"),
                                        os.path.join("..", "..", "include", "comodgan_b200.h"),
                                        os.path.join("..", "..", "include", "inception_b200.h"),
                                        os.path.join("..", "..", "include", "lpips_b200.h"),
                                        os.path.join("..", "..", "include", "metrics_b200.h")]
    for name in files:
        path = os.path.join(CSRC, name)
        if os.path.isfile(path):
            h.update(name.encode())
            with open(path, "rb") as f:
                h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_current() -> bool:
    if not (os.path.exists(LIBPATH) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as f:
        return f.read().strip() == _source_hash()


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA source into the shared library; returns its path."""
    if not force and is_current():
        return LIBPATH
    os.makedirs(LIBDIR, exist_ok=True)
    tmp = LIBPATH + ".tmp.%d" % os.getpid()
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + SOURCES
    proc = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n%s\n%s" % (" ".join(cmd), proc.stderr[-8000:]))
    if verbose:
        sys.stderr.write(proc.stderr)
    os.replace(tmp, LIBPATH)
    with open(STAMP, "w") as f:
        f.write(_source_hash())
    return LIBPATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
