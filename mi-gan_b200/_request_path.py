"""What the request-path pipelines share: the generator they run, the upload of their inputs, their queued calls and
`wait()`, and the photo pipelines' request checks, workspace and result copy-back."""
from __future__ import annotations

import ctypes
from typing import List, Optional, Tuple

import numpy as np
import torch

from . import comodgan
from .generator import Generator


def load_generator(pipeline: torch.nn.Module, model_or_state_dict, resolution: int, device, accept_comodgan: bool = False):
    """The generator of `pipeline`, on the CUDA `device` in eval mode.  `model_or_state_dict`: a `migan_b200.Generator` of
    that resolution, a state_dict, or a file `torch.load` reads one from.  With `accept_comodgan`, also a
    `migan_b200.comodgan.Generator` of that resolution (Co-Mod-GAN checkpoints come in through `comodgan.load`)."""
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("migan_b200.%s runs on a CUDA device (there is no CPU path); got %s" % (type(pipeline).__name__, device))
    if accept_comodgan and isinstance(model_or_state_dict, comodgan.Generator):
        if model_or_state_dict.img_resolution != resolution:
            raise RuntimeError("generator resolution %d != pipeline resolution %d" % (model_or_state_dict.img_resolution, resolution))
        model = model_or_state_dict
    elif isinstance(model_or_state_dict, Generator):
        if model_or_state_dict.resolution != resolution:
            raise RuntimeError("generator resolution %d != pipeline resolution %d" % (model_or_state_dict.resolution, resolution))
        model = model_or_state_dict
    else:
        model = Generator(resolution=resolution)
        sd = model_or_state_dict if isinstance(model_or_state_dict, dict) else torch.load(model_or_state_dict, map_location="cpu")
        model.load_state_dict(sd)
    return model.to(device).eval()


class NoiseSeeds:
    """The noise seeds of a pipeline that accepts a Co-Mod-GAN generator, and its generator chunking.

    The k-th image the pipeline processes without explicit seeds, counted across calls, gets the seed
    noise_seed * 2**32 + k (k = `noise_index`, readable and settable).  A Co-Mod-GAN pass runs its generator in chunks of
    at most `generator_batch` images.  MI-GAN generators draw no noise: they take no seeds and run the pass whole."""

    def __init__(self, model, noise_seed: int, generator_batch: int):
        if not 0 <= int(noise_seed) < 1 << 32:
            raise ValueError("noise_seed must lie in [0, 2**32), got %d" % noise_seed)
        if int(generator_batch) < 1:
            raise ValueError("generator_batch must be >= 1, got %d" % generator_batch)
        self.comodgan = isinstance(model, comodgan.Generator)
        self.noise_seed, self.generator_batch, self.noise_index = int(noise_seed), int(generator_batch), 0

    def take(self, name: str, n: int, seeds) -> Optional[np.ndarray]:
        """The uint64 seeds of the next n images (None for MI-GAN); `seeds` overrides the counter, which then stays."""
        if not self.comodgan:
            if seeds is not None:
                raise ValueError("%s.forward_batch: seeds= needs a Co-Mod-GAN generator; MI-GAN draws no noise" % name)
            return None
        if seeds is not None:
            out = comodgan.seed_array(seeds)
            if len(out) != n:
                raise ValueError("%s.forward_batch: %d seeds for %d images" % (name, len(out), n))
            return out
        k0, self.noise_index = self.noise_index, self.noise_index + n
        return np.array([(self.noise_seed << 32) + k for k in range(k0, k0 + n)], dtype=np.uint64)

    def run(self, model, x: torch.Tensor, seeds: Optional[np.ndarray]) -> Tuple[torch.Tensor, int]:
        """(y, launches): the generator over x [n, 4, R, R], in chunks for Co-Mod-GAN, and its kernel launches."""
        if seeds is None:
            y = model(x)
            return y, model.last_launch_count()
        n, gb = x.shape[0], self.generator_batch
        y = torch.empty((n, 3, x.shape[2], x.shape[3]), dtype=torch.float32, device=x.device)
        launches = 0
        for c in range(0, n, gb):
            model(x[c:c + gb], seeds=seeds[c:c + gb], _out=y[c:c + gb])
            launches += model.last_launch_count()
        return y, launches


def _to(t: torch.Tensor, device, non_blocking: bool) -> torch.Tensor:
    """`t` contiguous on `device`.  A non-blocking copy from pageable memory would wait for the stream, so a pageable CPU
    tensor is first staged by a host copy into pinned memory."""
    if non_blocking and not t.is_cuda and not t.is_pinned():
        t = t.pin_memory()
    return t.to(device, non_blocking=non_blocking).contiguous()


class _Call:
    """One enqueued call: the event after its last copy (None when it enqueued nothing), its per-request record, and the
    tensors its enqueued work reads or writes (kept alive until the call is waited for)."""

    def __init__(self, event, record: list, keep):
        self.event, self.record, self.keep = event, record, keep


class _Queued(torch.nn.Module):
    """A pipeline whose calls may only be enqueued (`forward_batch(..., wait=False)`) and waited for later."""

    def __init__(self, model_or_state_dict, resolution: int, device, accept_comodgan: bool = False):
        super().__init__()
        self.model = load_generator(self, model_or_state_dict, resolution, device, accept_comodgan)
        self.res = int(resolution)
        self._pending: List[_Call] = []                     # calls of forward_batch(..., wait=False) not yet waited for

    def _set_record(self, record: list) -> None:
        """Set the pipeline's `last_*` record from the joined records of the calls just waited for."""
        raise NotImplementedError

    def _finish(self, calls) -> None:
        """Wait for `calls` in order; the `last_*` record becomes theirs when they have one."""
        record = []
        for call in calls:
            if call.event is not None:
                call.event.synchronize()
            record += call.record
        if record:
            self._set_record(record)

    def wait(self, calls: Optional[int] = None) -> None:
        """Block until every call enqueued with `forward_batch(..., wait=False)` has finished: its results are written and
        the per-request record of those calls (`last_boxes`, `last_sizes`, `last_extents` or `last_windows`) is set, in
        submission order.  `calls`: wait only for the oldest that many calls; the later ones stay queued."""
        k = len(self._pending) if calls is None else max(0, min(int(calls), len(self._pending)))
        done, self._pending = self._pending[:k], self._pending[k:]
        self._finish(done)


class _PhotoPipeline(_Queued):
    """What the photo pipelines share: HWC uint8 photos as numpy arrays or CPU / CUDA tensors, their checks, one generator
    workspace and the copy of the results back to the host."""

    def __init__(self, model_or_state_dict, resolution: int, device, accept_comodgan: bool = False):
        super().__init__(model_or_state_dict, resolution, device, accept_comodgan)
        self._ws = None                                      # the generator workspace, grown to the largest chunk seen

    @classmethod
    def _name(cls) -> str:
        return cls.__name__

    def __call__(self, img, mask, invert: bool = False):
        return self.forward_batch([img], [mask], invert=invert)[0]

    def _device(self) -> torch.device:
        return next(self.model.parameters()).device

    def _extent(self, eng, i: int, H: int, W: int, what: str = "") -> Tuple[Tuple[int, int], int]:
        """((Hp, Wp), largest batch there) of an H x W photo (or window) of request i; ValueError when it is too large
        for one forward."""
        Hp, Wp, mx = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        if eng.lib.migan_fullres_extent(eng.handle, H, W, ctypes.byref(Hp), ctypes.byref(Wp), ctypes.byref(mx)) != 0:
            raise ValueError("%s: request %d: %s%s" % (self._name(), i, what, eng.lib.migan_last_error().decode()))
        return (Hp.value, Wp.value), mx.value

    def _check(self, i, img, mask):
        """(photo tensor [H,W,3], mask tensor [Hm,Wm,C]) of request i."""
        name = self._name()
        img = torch.from_numpy(np.ascontiguousarray(img)) if isinstance(img, np.ndarray) else img
        mask = torch.from_numpy(np.ascontiguousarray(mask)) if isinstance(mask, np.ndarray) else mask
        if not isinstance(img, torch.Tensor) or not isinstance(mask, torch.Tensor):
            raise TypeError("%s: request %d: photo and mask must be numpy arrays or torch tensors" % (name, i))
        if img.dtype != torch.uint8 or mask.dtype != torch.uint8:
            raise ValueError("%s: request %d: photo and mask must be uint8" % (name, i))
        if img.dim() != 3 or img.shape[2] != 3 or img.shape[0] < 1 or img.shape[1] < 1:
            raise ValueError("%s: request %d: photo of shape %s, expected [H, W, 3]" % (name, i, tuple(img.shape)))
        if mask.dim() == 2:
            mask = mask.unsqueeze(2)
        if mask.dim() != 3 or not 1 <= mask.shape[2] <= 4:
            raise ValueError("%s: request %d: mask of shape %s, expected [H, W] or [H, W, 1..4]" % (name, i, tuple(mask.shape)))
        self._check_mask_size(i, img, mask)
        if img.is_cuda and img.device != self._device():
            raise ValueError("%s: request %d: photo on %s, the pipeline runs on %s" % (name, i, img.device, self._device()))
        return img, mask

    def _check_mask_size(self, i, img, mask) -> None:
        """The mask has the photo's H x W."""
        if tuple(mask.shape[:2]) != tuple(img.shape[:2]):
            raise ValueError("%s: request %d: mask of %d x %d, photo of %d x %d (H x W); they must match"
                             % (self._name(), i, mask.shape[0], mask.shape[1], img.shape[0], img.shape[1]))

    def _kind(self, i: int, img, wait: bool) -> str:
        """"numpy", "cpu" or "cuda" for photo i; refuses a photo that cannot be copied asynchronously when wait=False."""
        if not isinstance(img, (np.ndarray, torch.Tensor)):
            raise TypeError("%s: request %d: photo and mask must be numpy arrays or torch tensors" % (self._name(), i))
        kind = "numpy" if isinstance(img, np.ndarray) else ("cuda" if img.is_cuda else "cpu")
        if not wait and kind != "cuda" and not (kind == "cpu" and img.is_pinned() and img.is_contiguous()):
            raise RuntimeError("%s.forward_batch(wait=False): CPU photo %d must be a pinned contiguous tensor (it is "
                               "copied asynchronously); use torch.from_numpy(img).pin_memory() or wait=True" % (self._name(), i))
        return kind

    def _requests(self, imgs, masks, invert, wait: bool):
        """(kinds, [(photo, mask)], inverts) of a forward_batch call, after every per-request check."""
        imgs, masks = list(imgs), list(masks)
        name = self._name()
        if len(imgs) != len(masks):
            raise ValueError("%s.forward_batch: %d photos and %d masks" % (name, len(imgs), len(masks)))
        inverts = [bool(invert)] * len(imgs) if isinstance(invert, (bool, int)) else [bool(v) for v in invert]
        if len(inverts) != len(imgs):
            raise ValueError("%s.forward_batch: %d invert flags for %d requests" % (name, len(inverts), len(imgs)))
        kinds, checked = [], []
        for i, (img, mask) in enumerate(zip(imgs, masks)):
            kinds.append(self._kind(i, img, wait))
            checked.append(self._check(i, img, mask))
        return kinds, checked, inverts

    def _workspace(self, eng, passes) -> torch.Tensor:
        """The one workspace, 1024-byte aligned, grown (never shrunk) to what the largest chunk of `passes` needs.  A grown
        workspace is a new address, so the plans cached for the old one are no longer hit; the old memory is released in
        stream order."""
        nbytes = max(eng.lib.migan_workspace_bytes_hw(eng.handle, len(c.requests), c.Hp, c.Wp) for p in passes for c in p)
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            raw = torch.empty(nbytes + 1024, dtype=torch.uint8, device=eng.device)
            off = (-raw.data_ptr()) % 1024
            self._ws = raw[off:off + nbytes]
        return self._ws

    def _complete(self, kinds, outs_d, record: list, keep, stream, wait: bool) -> list:
        """Enqueue the copy of each result to pinned host memory (except for CUDA photos) and the call's completion event
        on `stream`, then finish the call (wait=True) or queue it for `wait()`.  Returns the results: numpy for numpy
        photos once finished, tensors otherwise."""
        results = []
        for kind, out in zip(kinds, outs_d):
            if kind == "cuda":
                results.append(out)
            else:
                host = torch.empty(out.shape, dtype=torch.uint8, pin_memory=True)
                host.copy_(out, non_blocking=True)
                results.append(host)
        event = torch.cuda.Event()
        event.record(stream)
        call = _Call(event, record, keep)
        if wait:
            self._finish([call])
            return [r.numpy() if kind == "numpy" else r for kind, r in zip(kinds, results)]
        self._pending.append(call)
        return results
