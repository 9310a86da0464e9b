"""The context life cycle both tensor-core networks share (InceptionV3 `inception_*`, LPIPS `lpips_*`), in each
runtime's emulation build: call order, refusals, the workspace size of a refused shape and the launch plan's
truncation."""
import ctypes
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

import build_emul  # noqa: E402
import migan_b200  # noqa: E402,F401
from migan_b200 import _abi, fid, lpips  # noqa: E402

# prefix, emulation build, wrapper module, a shape its input check refuses, a shape it takes
NETS = {
    "inception": ("inception_abi.cu", fid, (1, 0, 5), (2, 97, 131)),
    "lpips": ("lpips_abi.cu", lpips, (1, 30, 31), (3, 31, 40)),
}


@pytest.fixture(scope="module", params=sorted(NETS))
def net(request):
    prefix = request.param
    source, module, refused, taken = NETS[prefix]
    path = build_emul._compile(prefix + "_emul", [os.path.join(build_emul.CSRC, s) for s in (source, "abi_error.cu")])
    L = module.lib(ctypes.CDLL(path))
    L.migan_last_error.restype = ctypes.c_char_p
    return prefix, L, module, refused, taken


def _call(net, name, *args):
    prefix, L = net[0], net[1]
    return getattr(L, prefix + "_" + name)(*args)


def _error(net):
    return net[1].migan_last_error().decode()


def _create(net, device):
    h = ctypes.c_void_p()
    assert _call(net, "create", device, ctypes.byref(h)) == 0
    return h


def _load_all(net, h):
    """Sets every key of the network's spec to zeros."""
    for key, shape in net[2].weight_spec(net[1]):
        t = torch.zeros(shape, dtype=torch.float32)
        assert _call(net, "set_weight", h, key.encode(), t.data_ptr(), t.numel()) == 0, _error(net)


def _forward(net, h, n, H, W):
    """The network's forward on placeholder buffers: only reached for the refusals before the walk."""
    buf = (ctypes.c_float * 16)()
    p = ctypes.addressof(buf)
    if net[0] == "inception":
        return _call(net, "features", h, p, n, H, W, p, p, 64, None)
    return _call(net, "forward", h, p, p, n, H, W, 0, p, p, p, 64, None)


@pytest.fixture
def finalized(net):
    h = _create(net, 0)
    _load_all(net, h)
    assert _call(net, "finalize_weights", h) == 0, _error(net)
    yield h
    _call(net, "destroy", h)


def test_finalize_twice_is_a_state_error(net, finalized):
    assert _call(net, "finalize_weights", finalized) == _abi.ERR_STATE
    assert "already finalized" in _error(net)


def test_set_weight_after_finalize_is_a_state_error(net, finalized):
    key, shape = net[2].weight_spec(net[1])[0]
    t = torch.zeros(shape, dtype=torch.float32)
    assert _call(net, "set_weight", finalized, key.encode(), t.data_ptr(), t.numel()) == _abi.ERR_STATE
    assert "already finalized" in _error(net)


def test_forward_before_finalize_is_a_state_error(net):
    h = _create(net, 0)
    try:
        _load_all(net, h)
        assert _forward(net, h, *net[4]) == _abi.ERR_STATE
        assert "%s_finalize_weights" % net[0] in _error(net)
        assert _call(net, "last_launch_count", h) == 0
    finally:
        _call(net, "destroy", h)


def test_description_only_context_cannot_finalize(net):
    h = _create(net, -1)
    try:
        _load_all(net, h)
        assert _call(net, "finalize_weights", h) == _abi.ERR_CUDA
        assert "description only" in _error(net)
        assert _forward(net, h, *net[4]) == _abi.ERR_STATE
    finally:
        _call(net, "destroy", h)


def test_null_context(net):
    t = torch.zeros(1)
    name, nd, shape = ctypes.c_char_p(), ctypes.c_int(), (ctypes.c_int64 * 4)()
    assert _call(net, "weight_info", None, 0, ctypes.byref(name), ctypes.byref(nd), shape) == _abi.ERR_INVALID
    assert _call(net, "set_weight", None, b"x", t.data_ptr(), 1) == _abi.ERR_INVALID
    assert _call(net, "finalize_weights", None) == _abi.ERR_INVALID
    assert _forward(net, None, *net[4]) == _abi.ERR_INVALID
    assert "null context" in _error(net)
    assert _call(net, "launch_plan", None, *net[4], None, 0) == -_abi.ERR_INVALID
    assert _call(net, "workspace_bytes", None, *net[4]) == 0
    assert _call(net, "num_weights", None) == 0
    assert _call(net, "last_launch_count", None) == 0
    assert _call(net, "destroy", None) == 0


def test_refused_shape(net):
    h = _create(net, -1)
    try:
        assert _call(net, "workspace_bytes", h, *net[3]) == 0
        assert _call(net, "workspace_bytes", h, 0, *net[4][1:]) == 0
        assert _call(net, "workspace_bytes", h, *net[4]) > 0
        assert _call(net, "launch_plan", h, *net[3], None, 0) == -_abi.ERR_INVALID
        assert "bad batch" in _error(net)
    finally:
        _call(net, "destroy", h)


def test_launch_plan_truncates_to_cap(net):
    h = _create(net, -1)
    try:
        full = "\n".join(net[2].launch_plan(*net[4], handle=net[1])) + "\n"
        assert _call(net, "launch_plan", h, *net[4], None, 0) == len(full)
        for cap in (1, 2, 40, len(full), len(full) + 1):
            buf = ctypes.create_string_buffer(b"#" * (cap + 4))
            assert _call(net, "launch_plan", h, *net[4], buf, cap) == len(full)
            assert buf.raw[:cap] == full[:cap - 1].encode() + b"\0"
            assert buf.raw[cap:] == b"#" * 4 + b"\0"
        buf = ctypes.create_string_buffer(b"#" * 4)
        assert _call(net, "launch_plan", h, *net[4], buf, 0) == len(full)
        assert buf.raw == b"#" * 4 + b"\0"
    finally:
        _call(net, "destroy", h)
