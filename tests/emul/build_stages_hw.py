"""Host-emulation build of the UP / STEM pre-stages on an H x W image (TEST INFRASTRUCTURE ONLY).

``mi-gan_b200/csrc/sepconv_stages.cuh`` compiles as plain C++ with ``-DMIGAN_EMULATE``; ``stages_hw_emul.cpp`` loops the
128 workers of one prologue group over host buffers laid out like the kernel's TMA-filled pipeline stage, for tiles at the
right / bottom edge of a rectangular image (``tests/test_fullconv_emul.py``).  The package never loads this library.
"""
import hashlib
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "mi-gan_b200", "csrc")
OUT = os.path.join(HERE, "_build")
LIB = os.path.join(OUT, "libstages_hw_emul.so")
SRCS = [os.path.join(CSRC, "sepconv_stages.cuh"), os.path.join(HERE, "stages_hw_emul.cpp")]


def _hash() -> str:
    h = hashlib.sha256()
    for s in SRCS:
        with open(s, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def build() -> str:
    os.makedirs(OUT, exist_ok=True)
    stamp = os.path.join(OUT, "stages_hw_stamp")
    if os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == _hash():
        return LIB
    cmd = ["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-DMIGAN_EMULATE", "-I", CSRC,
           os.path.join(HERE, "stages_hw_emul.cpp"), "-o", LIB]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("stage emulation build failed:\n" + proc.stderr[-4000:])
    with open(stamp, "w") as f:
        f.write(_hash())
    return LIB


if __name__ == "__main__":
    print(build())
