"""Co-Mod-GAN generator on H100: drop-in for `lib.model_zoo.comodgan.{Mapping, Encoder, Synthesis, Generator}`.

Reference construction (scripts/demo.py:95-100):

    model = Generator(Mapping(num_ws=14), Encoder(resolution=256), Synthesis(resolution=256))
    model.load_state_dict(torch.load(path)); model.to("cuda").eval(); img = model(x, z=z, noise_mode="const")

Same `state_dict` keys / shapes / order (180 entries @256: `mapping.*`, `synthesis.*`, `encoder.*`,
lib/model_zoo/stylegan.py:572-579 + comodgan.py:431-435), same forward signature (comodgan.py:438-455).  The modules hold
parameters only; all arithmetic happens in the C-ABI library (`include/comodgan_b200.h`).  PyTorch is used for device
memory, the current stream and -- as in the reference -- for drawing `z` / the random noise planes when the caller does
not pass them.  There is no CPU path.
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import _abi

NOISE_MODES = {"none": 0, "const": 1, "random": 2}
_BUFFER_LEAVES = ("w_avg", "resample_filter", "noise_const")   # register_buffer in the reference, the rest are Parameters


def _spec(resolution: int) -> List[Tuple[str, Tuple[int, ...]]]:
    """(key, shape) of every state_dict entry, from the library's own registry (description-only context)."""
    lib = _abi.load()
    h = ctypes.c_void_p()
    rc = lib.comodgan_create(resolution, -1, ctypes.byref(h))
    if rc != 0:
        msg = lib.comodgan_last_error().decode()
        if rc == _abi.ERR_INVALID:
            raise ValueError(msg)                    # non power-of-two resolution: ValueError like comodgan.py:132-134
        raise _abi.MiganError(rc, msg)
    out = []
    name, nd, shape = ctypes.c_char_p(), ctypes.c_int(), (ctypes.c_int64 * 4)()
    for i in range(lib.comodgan_num_weights(h)):
        _abi.check(lib.comodgan_weight_info(h, i, ctypes.byref(name), ctypes.byref(nd), shape))
        out.append((name.value.decode(), tuple(int(v) for v in shape[:nd.value])))
    lib.comodgan_destroy(h)
    return out


def _initial_value(key: str, shape) -> torch.Tensor:
    """Constructor-time values of the reference (stylegan.py:75-76, 223-225, 270-275, 391-392)."""
    if key.endswith("resample_filter"):
        f = torch.tensor([1.0, 3.0, 3.0, 1.0])
        f = torch.outer(f, f)
        return f / f.sum()
    if key.endswith("noise_const"):
        return torch.randn(shape)
    if key.endswith("noise_strength") or key.endswith("w_avg"):
        return torch.zeros(shape)
    if key.endswith("affine.bias"):
        return torch.ones(shape)
    if key.endswith(".bias"):
        return torch.zeros(shape)
    if key.startswith("mapping.fc") and key.endswith(".weight"):
        return torch.randn(shape) / 0.01
    return torch.randn(shape)


def _guard(device: torch.device):
    return torch.cuda.device(device)


def _stream(device: torch.device):
    return torch.cuda.current_stream(device).cuda_stream


def _device_index(device: torch.device) -> int:
    return device.index if device.index is not None else torch.cuda.current_device()


class _Node(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("migan_b200.comodgan sub-modules are parameter containers; call Generator.forward")


def _populate(root: nn.Module, resolution: int, prefix: str) -> None:
    for key, shape in _spec(resolution):
        if not key.startswith(prefix + "."):
            continue
        *mods, leaf = key[len(prefix) + 1:].split(".")
        node = root
        for m in mods:
            if not hasattr(node, m):
                node.add_module(m, _Node())
            node = getattr(node, m)
        value = _initial_value(key, shape)
        if leaf in _BUFFER_LEAVES:
            node.register_buffer(leaf, value)
        else:
            node.register_parameter(leaf, nn.Parameter(value))


class Mapping(_Node):
    """lib/model_zoo/stylegan.py:355-438 with c_dim = 0 (comodgan.py:27-29)."""

    def __init__(self, z_dim: int = 512, c_dim: int = 0, w_dim: int = 512, num_ws: int = 14, num_layers: int = 8):
        super().__init__()
        if (z_dim, c_dim, w_dim, num_layers) != (512, 0, 512, 8):
            raise NotImplementedError("only the demo configuration (z_dim=512, c_dim=0, w_dim=512, 8 layers) is built")
        self.z_dim, self.c_dim, self.w_dim, self.num_ws, self.num_layers = z_dim, c_dim, w_dim, num_ws, num_layers
        _populate(self, 8, "mapping")


class Encoder(_Node):
    """lib/model_zoo/comodgan.py:113-204 (defaults: ic_n=4, oc_n=1024, ch_base=32768, ch_max=512, no mbstd)."""

    def __init__(self, resolution: int = 256, ic_n: int = 4, oc_n: int = 1024):
        super().__init__()
        if (ic_n, oc_n) != (4, 1024):
            raise NotImplementedError("only ic_n=4, oc_n=1024 is built")
        self.resolution, self.ic_n = resolution, ic_n
        _populate(self, resolution, "encoder")


class Synthesis(_Node):
    """lib/model_zoo/comodgan.py:346-421 (defaults: w_dim=512, w0_dim=1024, rgb_n=3)."""

    def __init__(self, w_dim: int = 512, w0_dim: int = 1024, resolution: int = 256, rgb_n: int = 3):
        super().__init__()
        if (w_dim, w0_dim, rgb_n) != (512, 1024, 3):
            raise NotImplementedError("only w_dim=512, w0_dim=1024, rgb_n=3 is built")
        self.w_dim, self.resolution, self.rgb_n = w_dim, resolution, rgb_n
        self.num_ws = 2 * int(math.log2(resolution)) - 2          # 14 @256, 16 @512 (comodgan.py:371-374)
        _populate(self, resolution, "synthesis")


class _Engine:
    def __init__(self, resolution: int, device: torch.device):
        self.lib = _abi.load()
        self.device = device
        self.handle = ctypes.c_void_p()
        _abi.check(self.lib.comodgan_create(resolution, _device_index(device), ctypes.byref(self.handle)))
        self.weights_version = None
        self.workspaces: Dict[int, torch.Tensor] = {}
        self.noise_res = [self.lib.comodgan_noise_plane_res(self.handle, i)
                          for i in range(self.lib.comodgan_num_noise_planes(self.handle))]

    def close(self):
        if self.handle:
            self.lib.comodgan_destroy(self.handle)
            self.handle = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def upload(self, resolution: int, state: Dict[str, torch.Tensor], version) -> None:
        if self.weights_version is not None:       # weights changed: the C context is immutable once finalized
            dev = self.device
            self.close()
            self.__init__(resolution, dev)
        for key, t in state.items():
            h = t.detach().to(device="cpu", dtype=torch.float32).contiguous()
            _abi.check(self.lib.comodgan_set_weight(self.handle, key.encode(), h.data_ptr(), h.numel()))
        _abi.check(self.lib.comodgan_finalize_weights(self.handle))
        self.weights_version = version

    def workspace(self, n: int, seeded: bool = False) -> torch.Tensor:
        ws = self.workspaces.get((n, seeded))
        if ws is None:
            size = self.lib.comodgan_workspace_bytes_seeded if seeded else self.lib.comodgan_workspace_bytes
            nbytes = size(self.handle, n)
            raw = torch.empty(nbytes + 1024, dtype=torch.uint8, device=self.device)
            off = (-raw.data_ptr()) % 1024
            ws = raw[off:off + nbytes]
            self.workspaces = {(n, seeded): ws}
        return ws


class Generator(nn.Module):
    """lib/model_zoo/comodgan.py:424-455."""

    def __init__(self, mapping: Mapping, encoder: Encoder, synthesis: Synthesis):
        super().__init__()
        if not (isinstance(mapping, Mapping) and isinstance(encoder, Encoder) and isinstance(synthesis, Synthesis)):
            raise TypeError("Generator(mapping, encoder, synthesis) takes migan_b200.comodgan modules")
        self.mapping = mapping          # registration order = state_dict order of the reference
        self.synthesis = synthesis
        if synthesis.num_ws != mapping.num_ws:
            raise ValueError                                         # stylegan.py:580-581
        if encoder.resolution != synthesis.resolution:
            raise ValueError("encoder and synthesis resolutions differ")
        self.encoder = encoder
        self.num_ws, self.z_dim, self.c_dim, self.w_dim = mapping.num_ws, mapping.z_dim, mapping.c_dim, mapping.w_dim
        self.img_resolution, self.img_channels, self.ic_n = synthesis.resolution, synthesis.rgb_n, encoder.ic_n
        self._engines: Dict[torch.device, _Engine] = {}

    def __getstate__(self):
        state = self.__dict__.copy()
        state["_engines"] = {}
        return state

    def _state_version(self):
        return tuple((t._version, t.data_ptr()) for t in self.state_dict(keep_vars=True).values())

    def _engine(self, device: torch.device) -> _Engine:
        eng = self._engines.get(device)
        if eng is None:
            eng = _Engine(self.img_resolution, device)
            self._engines[device] = eng
        version = self._state_version()
        if eng.weights_version != version:
            eng.upload(self.img_resolution, self.state_dict(keep_vars=True), version)
        return eng

    def _validate(self, x, z, draw_z: bool = True):
        r = self.img_resolution
        if not isinstance(x, torch.Tensor) or x.dim() != 4 or tuple(x.shape[1:]) != (4, r, r):
            raise RuntimeError("expected x of shape [N, 4, %d, %d] (mask-0.5, img*mask)" % (r, r))
        if not x.is_cuda:
            raise RuntimeError("migan_b200.comodgan.Generator runs on H100 (sm_90a) only; got a %s tensor. "
                               "There is no CPU fallback (the CPU oracle lives in oracle/ for tests)." % x.device)
        if x.dtype != torch.float32:
            raise RuntimeError("expected float32 input, got %s" % x.dtype)
        if x.shape[0] == 0:
            raise RuntimeError("empty batch")
        if next(self.parameters()).device != x.device:
            raise RuntimeError("input is on %s but the module parameters are on %s" % (x.device, next(self.parameters()).device))
        if z is None:
            if not draw_z:
                return x.contiguous(), None
            z = torch.randn([x.shape[0], 512]).to(x.device)          # comodgan.py:444-445
        if tuple(z.shape) != (x.shape[0], self.z_dim):
            raise RuntimeError("expected z of shape [%d, %d], got %s" % (x.shape[0], self.z_dim, tuple(z.shape)))
        return x.contiguous(), z.to(device=x.device, dtype=torch.float32).contiguous()

    @torch.no_grad()
    def forward(self, x, z=None, c=None, truncation_psi=1, truncation_cutoff=None, noise_mode="random",
                return_intermediate_outs=False, *, noise: Optional[torch.Tensor] = None, seeds=None, _tap=None,
                _out: Optional[torch.Tensor] = None):
        """x: 4-channel mask+rgb input.  `noise` (optional, noise_mode='random'): the N(0,1) planes to use instead of
        fresh torch.randn draws, concatenated in forward order (see `noise_plane_shapes`).  `seeds` (optional,
        noise_mode='random'): one 64-bit seed per image, a sequence or an int64 / uint64 tensor; the planes, and z when it
        is None, are then drawn on the device from the seeded streams of `seeded_noise`, so image i's draws depend on
        seeds[i] alone."""
        if c is not None:
            raise NotImplementedError("conditional mapping (c_dim > 0) is not part of the Co-Mod-GAN demo configuration")
        if return_intermediate_outs:
            raise NotImplementedError("return_intermediate_outs is a training-loss hook (lib/experiments/loss.py); not built")
        if noise_mode not in NOISE_MODES:
            raise AssertionError("noise_mode must be one of %s" % sorted(NOISE_MODES))      # stylegan.py:282
        if seeds is not None:
            if noise_mode != "random":
                raise ValueError("seeds draw the random noise planes: they need noise_mode='random', got %r" % noise_mode)
            if noise is not None:
                raise ValueError("pass seeds or noise, not both")
            seeds = seed_array(seeds)
        x, z = self._validate(x, z) if seeds is None else self._validate(x, z, draw_z=False)
        n, r = x.shape[0], self.img_resolution
        if seeds is not None and len(seeds) != n:
            raise ValueError("%d seeds for %d images" % (len(seeds), n))
        with _guard(x.device):
            eng = self._engine(x.device)
            planes = None
            if noise_mode == "random" and seeds is None:
                total = n * sum(v * v for v in eng.noise_res)
                planes = torch.randn(total, device=x.device) if noise is None else noise.to(x.device, torch.float32).contiguous().reshape(-1)
                if planes.numel() != total:
                    raise RuntimeError("noise must hold %d values" % total)
            y = torch.empty((n, 3, r, r), dtype=torch.float32, device=x.device) if _out is None else _out
            ws = eng.workspace(n, seeded=seeds is not None)
            stream = _stream(x.device)
            tap_buf = None
            if _tap is not None:
                tap_buf = torch.zeros((n,) + tuple(_tap[1]), dtype=torch.float32, device=x.device)
                _abi.check(eng.lib.comodgan_set_tap(eng.handle, _tap[0].encode(), tap_buf.data_ptr()))
            psi, cutoff = float(truncation_psi), -1 if truncation_cutoff is None else int(truncation_cutoff)
            try:
                if seeds is not None:
                    _abi.check(eng.lib.comodgan_forward_seeded(
                        eng.handle, x.data_ptr(), seeds.ctypes.data, z.data_ptr() if z is not None else None, y.data_ptr(),
                        n, psi, cutoff, ws.data_ptr(), ws.numel(), stream))
                else:
                    _abi.check(eng.lib.comodgan_forward(
                        eng.handle, x.data_ptr(), z.data_ptr(), y.data_ptr(), n, psi, cutoff, NOISE_MODES[noise_mode],
                        planes.data_ptr() if planes is not None else None, ws.data_ptr(), ws.numel(), stream))
            finally:
                if _tap is not None:
                    eng.lib.comodgan_set_tap(eng.handle, None, None)
        return (y, tap_buf) if _tap is not None else y

    @torch.no_grad()
    def seeded_noise(self, seeds) -> Tuple[torch.Tensor, torch.Tensor]:
        """(z [n, 512], planes) that `forward(..., seeds=seeds)` draws, as CUDA tensors on the module's device.  planes is
        flat, in `forward(noise=...)`'s layout.  Request i's stream p (0: z, 1 + j: noise plane j) is numpy's
        Philox4x64-10 with key [seeds[i], p], turned into normals by float64 Box-Muller (include/comodgan_b200.h)."""
        seeds = seed_array(seeds)
        n = len(seeds)
        if n == 0:
            raise ValueError("no seeds")
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("migan_b200.comodgan.Generator runs on a CUDA device; the module is on %s" % dev)
        with _guard(dev):
            eng = self._engine(dev)
            z = torch.empty((n, self.z_dim), dtype=torch.float32, device=dev)
            planes = torch.empty(n * sum(v * v for v in eng.noise_res), dtype=torch.float32, device=dev)
            _abi.check(eng.lib.comodgan_seeded_noise(eng.handle, seeds.ctypes.data, n, z.data_ptr(), planes.data_ptr(),
                                                     _stream(dev)))
        return z, planes

    def noise_plane_shapes(self, n: int):
        """[(n, r, r)] of the planes `forward(..., noise_mode='random', noise=...)` consumes, in order."""
        res = [4] + [r for i in range(3, int(math.log2(self.img_resolution)) + 1) for r in (2 ** i, 2 ** i)]
        return [(n, r, r) for r in res]

    def last_launch_count(self) -> int:
        eng = next(iter(self._engines.values()))
        return int(eng.lib.comodgan_last_launch_count(eng.handle))


def seed_array(seeds) -> np.ndarray:
    """`seeds` (a sequence of ints in [0, 2**64) or an int64 / uint64 tensor, whose bits are taken as they are) as a
    contiguous uint64 numpy array."""
    if isinstance(seeds, torch.Tensor):
        if seeds.dtype not in (torch.int64, torch.uint64) or seeds.dim() != 1:
            raise ValueError("seeds must be a 1-D int64 or uint64 tensor, got %s %s" % (seeds.dtype, tuple(seeds.shape)))
        return np.ascontiguousarray(seeds.detach().cpu().view(torch.int64).numpy().view(np.uint64))
    seeds = [int(s) for s in seeds]
    if any(s < 0 or s >= 1 << 64 for s in seeds):
        raise ValueError("seeds must lie in [0, 2**64)")
    return np.array(seeds, dtype=np.uint64)


def load(model_or_state_dict_or_path, resolution: int) -> Generator:
    """The Co-Mod-GAN generator of scripts/demo.py (:95-106) in eval mode: `Generator(Mapping(num_ws), Encoder(R),
    Synthesis(R))` with num_ws = 14 at 256 and 16 at 512, loaded from a state_dict or a file `torch.load` reads one from.
    A `Generator` of that resolution is returned as it is, in eval mode."""
    resolution = int(resolution)
    if isinstance(model_or_state_dict_or_path, Generator):
        if model_or_state_dict_or_path.img_resolution != resolution:
            raise ValueError("generator resolution %d != %d" % (model_or_state_dict_or_path.img_resolution, resolution))
        return model_or_state_dict_or_path.eval()
    synthesis = Synthesis(resolution=resolution)
    g = Generator(Mapping(num_ws=synthesis.num_ws), Encoder(resolution=resolution), synthesis)
    sd = model_or_state_dict_or_path
    if not isinstance(sd, dict):
        sd = torch.load(sd, map_location="cpu")
    g.load_state_dict(sd)
    return g.eval()
