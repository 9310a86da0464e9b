"""Host-emulation builds of the CUDA sources (TEST INFRASTRUCTURE ONLY).

The sources compile as plain C++ with ``-DMIGAN_EMULATE``: every launch becomes a host loop over the very same kernel
functors (``comod_kernels.cuh``), block functions run with the threads of a block in turn, and the GEMMs are reference
loops.  The index math, the resampler and mask arithmetic, the batching, the host planners and the C ABI's argument
checks are then checked against the oracles on a machine without a GPU.  ``csrc/portable.cuh`` holds what differs
between the two builds; ``-ffp-contract=off`` keeps every product and sum of its ``*_rn`` functions rounded on its own,
as their ``__f*_rn`` / ``__d*_rn`` intrinsics do on the device.  The package never loads these libraries, and the
product library contains no host loop (it is compiled without the macro).

- ``build()``: the Co-Mod-GAN host runtime and every request path with their ``extern "C"`` entry points and the error
  unit behind ``migan_last_error`` (``tests/test_*_emul.py``).
- ``build_harness(name)``: a test harness of ``tests/emul`` over the shared-memory stages of the fused SeparableConv2d
  kernel (``sepconv_stages.cuh``).
"""
import hashlib
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "mi-gan_b200", "csrc")
OUT = os.path.join(HERE, "_build")
SOURCES = ["comodgan_abi.cu", "abi_error.cu", "prepost.cu", "pipeline.cu", "reparam.cu", "demo_resize.cu", "fullres.cu",
           "holewin.cu", "masks.cu"]


def _stamp(cmd, sources) -> str:
    """Every file under csrc/ and include/, the sources and the command line: an edit to any header rebuilds."""
    h = hashlib.sha256(" ".join(cmd).encode())
    for d in (CSRC, os.path.join(ROOT, "include")):
        for name in sorted(os.listdir(d)):
            with open(os.path.join(d, name), "rb") as f:
                h.update(name.encode() + b"\0" + f.read())
    for s in sources:
        with open(s, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _compile(name, sources, openmp=True) -> str:
    os.makedirs(OUT, exist_ok=True)
    lib = os.path.join(OUT, "lib%s.so" % name)
    stamp_path = os.path.join(OUT, name + ".stamp")
    cmd = ["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17", "-DMIGAN_EMULATE", "-I", CSRC,
           "-x", "c++"] + (["-fopenmp"] if openmp else []) + sources
    stamp = _stamp(cmd, sources)
    if os.path.exists(lib) and os.path.exists(stamp_path):
        with open(stamp_path) as f:
            if f.read() == stamp:
                return lib
    tmp = lib + ".tmp.%d" % os.getpid()
    proc = subprocess.run(cmd + ["-o", tmp], capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("%s emulation build failed:\n%s" % (name, proc.stderr[-4000:]))
    os.replace(tmp, lib)
    with open(stamp_path, "w") as f:
        f.write(stamp)
    return lib


def build() -> str:
    return _compile("migan_emul", [os.path.join(CSRC, s) for s in SOURCES])


def build_harness(cpp: str) -> str:
    return _compile(os.path.splitext(cpp)[0], [os.path.join(HERE, cpp)], openmp=False)


if __name__ == "__main__":
    print(build())
