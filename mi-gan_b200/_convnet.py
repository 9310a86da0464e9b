"""The library side of the networks on the tensor-core implicit-GEMM convolution: fid.InceptionV3
(`include/inception_b200.h`) and lpips.LPIPS (`include/lpips_b200.h`).  Both C APIs have the same context calls under
their own prefix ("inception" or "lpips"): create, destroy, the weight registry, finalize, the workspace size, the
launch plan and the launch count."""
from __future__ import annotations

import contextlib
import ctypes
from typing import Dict, List, Tuple

import torch

from . import _abi


def _fn(lib, prefix: str, name: str):
    return getattr(lib, prefix + "_" + name)


@contextlib.contextmanager
def _description(lib, prefix: str):
    """A context without a device (weight spec and launch plan only), destroyed on exit."""
    h = ctypes.c_void_p()
    _abi.check(_fn(lib, prefix, "create")(-1, ctypes.byref(h)), lib)
    try:
        yield h
    finally:
        _fn(lib, prefix, "destroy")(h)


def _spec(lib, prefix: str, h) -> List[Tuple[str, Tuple[int, ...]]]:
    out = []
    name, nd, shape = ctypes.c_char_p(), ctypes.c_int(), (ctypes.c_int64 * 4)()
    for i in range(_fn(lib, prefix, "num_weights")(h)):
        _abi.check(_fn(lib, prefix, "weight_info")(h, i, ctypes.byref(name), ctypes.byref(nd), shape), lib)
        out.append((name.value.decode(), tuple(int(v) for v in shape[:nd.value])))
    return out


def weight_spec(lib, prefix: str) -> List[Tuple[str, Tuple[int, ...]]]:
    """(key, shape) of every state_dict entry the network takes, in state_dict order."""
    with _description(lib, prefix) as h:
        return _spec(lib, prefix, h)


def launch_plan(lib, prefix: str, n: int, H: int, W: int) -> List[str]:
    """The forward's launches for a batch of n at H x W, one line each ("<kind> <name> key=value ...")."""
    plan = _fn(lib, prefix, "launch_plan")
    with _description(lib, prefix) as h:
        size = plan(h, n, H, W, None, 0)
        if size < 0:
            _abi.check(-size, lib)
        buf = ctypes.create_string_buffer(size + 1)
        plan(h, n, H, W, buf, size + 1)
        return buf.value.decode().splitlines()


class Engine:
    """One library context: device None = description only (weights parsed, nothing uploaded)."""

    def __init__(self, lib, prefix: str, device, state: Dict[str, torch.Tensor]):
        self.lib, self.prefix, self.device = lib, prefix, device
        self.handle = ctypes.c_void_p()
        index = -1 if device is None else (device.index if device.index is not None else torch.cuda.current_device())
        _abi.check(_fn(lib, prefix, "create")(index, ctypes.byref(self.handle)), lib)
        self._workspace = _abi.Workspace()
        set_weight = _fn(lib, prefix, "set_weight")
        for k, t in state.items():
            t = t.detach().to("cpu", torch.float32).contiguous()
            _abi.check(set_weight(self.handle, k.encode(), t.data_ptr(), t.numel()), lib)
        if device is not None:
            _abi.check(_fn(lib, prefix, "finalize_weights")(self.handle), lib)
        else:
            missing = next((k for k, _ in _spec(lib, prefix, self.handle) if k not in state), None)
            if missing:
                raise _abi.MiganError(_abi.ERR_INVALID, "missing key '%s' in the state_dict" % missing)

    def workspace(self, n, H, W) -> torch.Tensor:
        nbytes = _fn(self.lib, self.prefix, "workspace_bytes")
        return self._workspace.get((n, H, W), lambda: nbytes(self.handle, n, H, W), self.device)

    def __del__(self):
        try:
            if self.handle:
                _fn(self.lib, self.prefix, "destroy")(self.handle)
        except Exception:
            pass


class Network(torch.nn.Module):
    """What fid.InceptionV3 and lpips.LPIPS share: the state_dict, its keys checked on the host when it is set, and one
    Engine per device, made on first use."""

    def _set_state(self, lib, prefix: str, state: Dict[str, torch.Tensor]) -> None:
        self._lib, self._prefix, self._state = lib, prefix, state
        Engine(lib, prefix, None, state)   # checks the keys on the host now: missing, unknown or mis-shaped fail by name
        self._engines: Dict[torch.device, Engine] = {}

    def _engine(self, device) -> Engine:
        eng = self._engines.get(device)
        if eng is None:
            eng = self._engines[device] = Engine(self._lib, self._prefix, device, self._state)
        return eng

    def last_launch_count(self) -> int:
        """The launches of the last forward."""
        eng = next(iter(self._engines.values()))
        return int(_fn(eng.lib, eng.prefix, "last_launch_count")(eng.handle))
