"""Host-emulation build of the free-form mask generator, ``mi-gan_b200/csrc/masks.cu`` (TEST INFRASTRUCTURE ONLY).

The file compiles as plain C++ with ``-DMIGAN_EMULATE``: the numpy stream and the attempt planner are the product's host
code, the rasterizer's block functions run with the threads of a block in turn (16-byte stores become 16-byte copies,
shared-memory atomics plain ORs) and the compaction is a host loop, so the masks are checked against the fixture and
``oracle/masks_oracle.py`` on a machine without a GPU (``tests/test_masks_emul.py``).  ``-ffp-contract=off`` keeps every
product and sum rounded on its own, as the device code's explicit ``__fmul_rn`` / ``__fadd_rn`` do.  The package never
loads this library.
"""
import hashlib
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "mi-gan_b200", "csrc")
OUT = os.path.join(HERE, "_build")
LIB = os.path.join(OUT, "libmasks_emul.so")
SRCS = [os.path.join(CSRC, "masks.cu"), os.path.join(CSRC, "prepost.cuh"), os.path.join(CSRC, "comod_kernels.cuh"),
        os.path.join(ROOT, "include", "migan_b200.h")]


def _hash() -> str:
    h = hashlib.sha256()
    for s in SRCS:
        with open(s, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def build() -> str:
    os.makedirs(OUT, exist_ok=True)
    stamp = os.path.join(OUT, "masks_stamp")
    if os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == _hash():
        return LIB
    tmp = LIB + ".tmp.%d" % os.getpid()
    cmd = ["g++", "-O2", "-fopenmp", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17", "-DMIGAN_EMULATE", "-x", "c++",
           "masks.cu", "-o", tmp]
    proc = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("mask emulation build failed:\n" + proc.stderr[-4000:])
    os.replace(tmp, LIB)
    with open(stamp, "w") as f:
        f.write(_hash())
    return LIB


if __name__ == "__main__":
    print(build())
