"""Staging memory of the host-memory calls: the sizes callers allocate by, and the two slot rings (fp32 and uint8) used
side by side on one context."""
import ctypes

import numpy as np
import pytest
import torch

import migan_b200
from migan_b200 import _abi
from oracle import migan_oracle as O

# (R, n): (migan_workspace_bytes, migan_graph_staging_bytes, migan_host_staging_bytes, migan_u8_staging_bytes).
# One slot holds x fp32 [n,4,R,R], y fp32 [n,3,R,R] and, for uint8 requests, img [n,R,R,3], out [n,R,R,3] and
# mask [n,R,R], each rounded up to 1024 bytes; the host calls have two slots.  At R = 8 the uint8 parts are smaller
# than the rounding.
SIZES = {
    (8, 1): (559104, 2048, 4096, 10240),
    (8, 3): (1677312, 6144, 12288, 18432),
    (8, 32): (17874944, 57344, 114688, 143360),
    (64, 1): (36438016, 114688, 229376, 286720),
    (64, 3): (109314048, 344064, 688128, 860160),
    (64, 32): (1166016512, 3670016, 7340032, 9175040),
    (256, 1): (163741696, 1835008, 3670016, 4587520),
    (256, 3): (491225088, 5505024, 11010048, 13762560),
    (256, 32): (5239734272, 58720256, 117440512, 146800640),
    (512, 1): (336232448, 7340032, 14680064, 18350080),
    (512, 3): (1008697344, 22020096, 44040192, 55050240),
    (512, 32): (10759438336, 234881024, 469762048, 587202560),
}
FUNCS = ("migan_workspace_bytes", "migan_graph_staging_bytes", "migan_host_staging_bytes", "migan_u8_staging_bytes")


@pytest.mark.parametrize("R", [8, 64, 256, 512])
def test_workspace_and_staging_bytes(lib, R):
    h = ctypes.c_void_p()
    _abi.check(lib.migan_create(R, -1, ctypes.byref(h)))   # description-only context
    try:
        for n in (1, 3, 32):
            assert tuple(getattr(lib, f)(h, n) for f in FUNCS) == SIZES[(R, n)], n
        assert all(getattr(lib, f)(h, 0) == 0 for f in FUNCS)
    finally:
        lib.migan_destroy(h)


@pytest.mark.gpu
def test_interleaved_host_and_u8_serving(cuda_device):
    """fp32 and uint8 requests enqueued alternately on one Generator, with one change of batch size, then host_wait():
    every output equals the synchronous call on the same input."""
    R = 64
    g = migan_b200.Generator(R)
    g.load_state_dict(O.make_state_dict(R, seed=3))
    g = g.to(cuda_device).eval()
    rng = np.random.RandomState(21)
    calls = []
    for i, n in enumerate((4, 4, 4, 6, 6, 6)):
        x = O.make_input(R, n, seed=80 + i).pin_memory()
        y = torch.empty(n, 3, R, R).pin_memory()
        g.forward_host(x, out=y, wait=False)
        img = torch.from_numpy(rng.randint(0, 256, size=(n, R, R, 3), dtype=np.uint8)).pin_memory()
        mask = torch.from_numpy(((rng.rand(n, R, R) > 0.5) * 255).astype(np.uint8)).pin_memory()
        out = torch.empty(n, R, R, 3, dtype=torch.uint8).pin_memory()
        g.forward_u8(img, mask, out=out, wait=False)
        calls.append((x, y, img, mask, out))
    g.host_wait()
    for x, y, img, mask, out in calls:
        assert torch.equal(y, g.forward_host(x))
        assert torch.equal(out, g.forward_u8(img, mask))
