"""The C ABI's argument checks on the CPU: the entry points of include/migan_b200.h are compiled once, with their
checks and messages, into the product library and into the emulation build alike, so a malformed call is refused here
exactly as on the GPU: the product's return code and, where it records one, a migan_last_error() message that names the
entry point."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

from migan_b200 import _abi  # noqa: E402
import build_emul  # noqa: E402

INVALID = _abi.ERR_INVALID


@pytest.fixture(scope="module")
def emul():
    return _abi.bind(ctypes.CDLL(build_emul.build()), [s for s in _abi.SYMBOLS if s[0] in NAMES])


# Buffers large enough for every call below; the checks refuse the call before anything is read.
U8 = np.zeros(1 << 16, np.uint8)
F32 = np.zeros(1 << 14, np.float32)
I32 = np.zeros(64, np.int32)
u8, f32, i32 = U8.ctypes.data, F32.ctypes.data, I32.ctypes.data
BOX = np.array([0, 2, 0, 8], np.int32)          # 2 columns wide: too narrow for a crop window
K25 = np.ones(25, np.float32).ctypes.data

# (entry point, arguments, expected return, prefix of migan_last_error() or None when the call records no message)
CASES = [
    ("b200_mask_raster", (None, 1, 64, u8, i32, None), INVALID, "mask_raster:"),
    ("b200_mask_raster", (u8, 1, 64, u8 + 1, i32, None), INVALID, "mask_raster:"),          # attempts not 16-byte aligned
    ("b200_mask_compact", (u8, i32, 1, 64, 65536, u8, None), INVALID, "mask_compact:"),
    ("b200_mask_compact", (u8, i32, 1, 64, -1, u8, None), INVALID, "mask_compact:"),
    ("b200_mask_compact", (u8, None, 1, 64, 1, u8, None), INVALID, "mask_compact:"),
    ("b200_feather_composite", (f32, u8, u8, u8, 1, 2, 8, K25, None), INVALID, "feather_composite:"),
    ("b200_feather_composite", (f32, u8, None, u8, 1, 8, 8, K25, None), INVALID, "feather_composite:"),
    ("b200_eval_composite", (f32, f32, 1, 8193, f32, f32, None), INVALID, "eval_composite:"),
    ("migan_demo_resized_size", (0, 5, 512, ctypes.byref(ctypes.c_int()), ctypes.byref(ctypes.c_int())), INVALID,
     "demo_resized_size:"),
    ("b200_pipeline_scratch_bytes", (0, 8, 16), 0, None),
    ("b200_hole_flags", (None, 8, 8, u8, None), INVALID, "hole_flags:"),
    ("b200_hole_flags", (u8, 0, 8, u8, None), INVALID, "hole_flags:"),
    ("migan_crop_box", (u8, 8, 8, 16, -1, i32), INVALID, "crop_box:"),
    ("migan_crop_box", (u8, 8, 8, 16, 0, None), INVALID, "crop_box:"),
    ("b200_pipeline_preprocess", (u8, u8, 8, 8, BOX.ctypes.data, 16, f32, u8, U8.nbytes, None), INVALID,
     "pipeline_preprocess:"),
    ("b200_pipeline_postprocess", (f32, u8, u8, 8, 8, None, 16, K25, u8, U8.nbytes, None), INVALID, "pipeline_postprocess:"),
]
NAMES = {c[0] for c in CASES} | {"migan_last_error", "b200_hole_cells_bytes"}


@pytest.mark.parametrize("name,args,rc,prefix", CASES, ids=["%s-%d" % (c[0], i) for i, c in enumerate(CASES)])
def test_product_argument_checks(emul, name, args, rc, prefix):
    assert emul.b200_hole_cells_bytes(None, 1, 64) == 0          # leaves a message no case below records
    assert emul.migan_last_error().startswith(b"hole_cells_bytes:")
    assert getattr(emul, name)(*args) == rc
    if prefix is not None:
        msg = emul.migan_last_error().decode()
        assert msg.startswith(prefix), msg
