"""`FullResPipeline`: inpaint photos of any size at their own resolution, on the GPU.

    pipe = FullResPipeline(state_dict_or_generator, resolution=512)
    out = pipe(img, mask, invert=False)               # img uint8 [H,W,3]; mask uint8 [H,W] / [H,W,1..4]; out [H,W,3]
    outs = pipe.forward_batch(imgs, masks)            # many photos of mixed sizes
    pipe.forward_batch(imgs_t, masks_t, wait=False)   # only enqueue (serving loop) ...
    pipe.wait()                                       # ... outputs written, pipe.last_extents set

The generator's fully convolutional forward (`Generator.forward_fc`) runs at any H, W >= R that are multiples of R/4.  A
photo of another size is padded to the smallest such extent, (Hp, Wp) = (max(R, q ceil(H/q)), max(R, q ceil(W/q))) with
q = R/4, and the result is cropped back:

1. the mask's per-pixel steps are those of demo.py's `read_mask` without its resize: the channel (alpha of LA / RGBA, R of
   RGB, L itself), 255 - v if `invert`, then v < 255 -> 0; a pixel is known where the result is 255;
2. the photo stays at the origin; the bottom and right are filled by reflection without repeating the edge, iterated when
   the pad is longer than the side: numpy's `np.pad(..., mode="reflect")`.  The known-mask is reflected with the photo, so
   a hole that touches the border continues into the pad as a hole;
3. x = cat([mask - 0.5, img * mask]) at (Hp, Wp) -> `forward_fc` -> (y*0.5+0.5).clamp(0,1)*255 -> uint8 on the top-left
   H x W, with the known pixels taken from the photo (demo.py's composite).

So the result is byte for byte `forward_fc_u8` on the reflect-padded photo and mask, cropped to H x W; a photo that is
already a valid size is not padded and gets `forward_fc_u8`'s bytes.  The padding rule decides the pixels the network sees
past the bottom and right edges, so results near those edges depend on it.

Requests are taken in passes of up to 32.  Within a pass they are grouped by extent in order of first appearance and each
group is split into chunks of at most the largest batch the forward accepts at that extent.  A pass is one pre-process
launch for every request, one `migan_forward_hw` per chunk and one post-process launch (kernels in csrc/fullres.cu behind
include/migan_b200.h).  The pipeline keeps one generator workspace, grown to the largest chunk seen, so the library's
per-shape plan cache serves every chunk and pass.  There is no CPU path.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, NamedTuple, Sequence, Tuple, Union

import numpy as np
import torch

from . import _abi
from .demo import _Call, _to
from .generator import Generator


class Chunk(NamedTuple):
    """One `migan_forward_hw` call of a pass: the extent and the requests in slot order (slot s is x[s] / y[s])."""
    Hp: int
    Wp: int
    requests: List[int]


def plan_passes(extents: Sequence[Tuple[int, int]], max_n: Dict[Tuple[int, int], int],
                pass_size: int = _abi.PIPE_MAX_BATCH) -> List[List[Chunk]]:
    """The passes of a call: requests [k * pass_size, (k + 1) * pass_size) form pass k; within a pass, requests are grouped
    by extent in order of first appearance and each group is split into chunks of at most max_n[extent]."""
    passes = []
    for p0 in range(0, len(extents), pass_size):
        groups: Dict[Tuple[int, int], List[int]] = {}
        for i in range(p0, min(p0 + pass_size, len(extents))):
            groups.setdefault(tuple(extents[i]), []).append(i)
        chunks = []
        for (Hp, Wp), idx in groups.items():
            m = max_n[(Hp, Wp)]
            chunks += [Chunk(Hp, Wp, idx[c:c + m]) for c in range(0, len(idx), m)]
        passes.append(chunks)
    return passes


class _PhotoPipeline(torch.nn.Module):
    """What the photo pipelines share: the generator, the per-request input checks, one workspace and `wait()`.
    `model_or_state_dict`: a `migan_b200.Generator`, a state_dict, or a file `torch.load` reads one from."""

    def __init__(self, model_or_state_dict, resolution: int, device: Union[str, torch.device] = "cuda"):
        super().__init__()
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("migan_b200.%s runs on a CUDA device (there is no CPU path); got %s" % (self._name(), device))
        if isinstance(model_or_state_dict, Generator):
            if model_or_state_dict.resolution != resolution:
                raise RuntimeError("generator resolution %d != pipeline resolution %d" % (model_or_state_dict.resolution, resolution))
            self.model = model_or_state_dict
        else:
            self.model = Generator(resolution=resolution)
            sd = model_or_state_dict if isinstance(model_or_state_dict, dict) else torch.load(model_or_state_dict, map_location="cpu")
            self.model.load_state_dict(sd)
        self.model = self.model.to(device).eval()
        self.res = int(resolution)
        self._ws = None                                      # the generator workspace, grown to the largest chunk seen
        self._pending: List[_Call] = []

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
        """(photo tensor [H,W,3], mask tensor [H,W,C]) of request i."""
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
        if tuple(mask.shape[:2]) != tuple(img.shape[:2]):
            raise ValueError("%s: request %d: mask of %d x %d, photo of %d x %d (H x W); they must match"
                             % (name, i, mask.shape[0], mask.shape[1], img.shape[0], img.shape[1]))
        if img.is_cuda and img.device != self._device():
            raise ValueError("%s: request %d: photo on %s, the pipeline runs on %s" % (name, i, img.device, self._device()))
        return img, mask

    def _kind(self, i: int, img, wait: bool) -> str:
        """"numpy", "cpu" or "cuda" for photo i; refuses a photo that cannot be copied asynchronously when wait=False."""
        if not isinstance(img, (np.ndarray, torch.Tensor)):
            raise TypeError("%s: request %d: photo and mask must be numpy arrays or torch tensors" % (self._name(), i))
        kind = "numpy" if isinstance(img, np.ndarray) else ("cuda" if img.is_cuda else "cpu")
        if not wait and kind != "cuda" and not (kind == "cpu" and img.is_pinned() and img.is_contiguous()):
            raise RuntimeError("%s.forward_batch(wait=False): CPU photo %d must be a pinned contiguous tensor (it is "
                               "copied asynchronously); use torch.from_numpy(img).pin_memory() or wait=True" % (self._name(), i))
        return kind

    def _workspace(self, eng, nbytes: int) -> torch.Tensor:
        """The one workspace, 1024-byte aligned, grown (never shrunk) to nbytes.  A grown workspace is a new address, so
        the plans cached for the old one are no longer hit; the old memory is released in stream order."""
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            raw = torch.empty(nbytes + 1024, dtype=torch.uint8, device=eng.device)
            off = (-raw.data_ptr()) % 1024
            self._ws = raw[off:off + nbytes]
        return self._ws

    def _finish(self, calls) -> None:
        raise NotImplementedError

    def wait(self) -> None:
        """Block until every call enqueued with `forward_batch(..., wait=False)` has finished: its outputs are written and
        the per-request record of those calls (`last_extents` / `last_windows`) is set, in submission order."""
        calls, self._pending = self._pending, []
        self._finish(calls)


class FullResPipeline(_PhotoPipeline):
    """`model_or_state_dict`: a `migan_b200.Generator`, a state_dict, or a file `torch.load` reads one from."""

    def __init__(self, model_or_state_dict, resolution: int, device: Union[str, torch.device] = "cuda"):
        super().__init__(model_or_state_dict, resolution, device)
        self.last_extents: List[Tuple[int, int]] = []      # (Hp, Wp) of every result of the last completed call(s)
        self.last_launches = 0                              # kernel launches of the last pass, generator included

    def _pass(self, eng, chunks: List[Chunk], imgs, masks, inverts, outs, ws, stream) -> list:
        """Enqueue one pass; returns the tensors its work reads or writes."""
        lib = eng.lib
        dev = eng.device
        n = sum(len(c.requests) for c in chunks)
        reqs = (_abi.FullResRequest * n)()
        xs, ys, k = [], [], 0
        for c in chunks:
            x = torch.empty((len(c.requests), 4, c.Hp, c.Wp), dtype=torch.float32, device=dev)
            y = torch.empty((len(c.requests), 3, c.Hp, c.Wp), dtype=torch.float32, device=dev)
            xs.append(x)
            ys.append(y)
            for slot, i in enumerate(c.requests):
                r = reqs[k]
                k += 1
                img, m = imgs[i], masks[i]
                r.img, r.H, r.W = img.data_ptr(), int(img.shape[0]), int(img.shape[1])
                r.mask, r.mask_channels, r.invert = m.data_ptr(), int(m.shape[2]), int(bool(inverts[i]))
                r.x, r.y, r.Hp, r.Wp, r.out = x[slot].data_ptr(), y[slot].data_ptr(), c.Hp, c.Wp, outs[i].data_ptr()
        path = _abi.path_id(self.model.path)
        _abi.check(lib.b200_fullres_preprocess(reqs, n, stream))
        launches = 2
        for c, x, y in zip(chunks, xs, ys):
            _abi.check(lib.migan_forward_hw(eng.handle, x.data_ptr(), y.data_ptr(), len(c.requests), c.Hp, c.Wp,
                                            ws.data_ptr(), ws.numel(), path, stream))
            launches += int(lib.migan_last_launch_count(eng.handle))
        _abi.check(lib.b200_fullres_postprocess(reqs, n, stream))
        self.last_launches = launches
        return xs + ys

    @torch.no_grad()
    def forward_batch(self, imgs: Sequence, masks: Sequence, invert: Union[bool, Sequence[bool]] = False,
                      wait: bool = True) -> list:
        """Many photos of any sizes.  imgs[i]: uint8 [H,W,3]; masks[i]: uint8 [H,W] or [H,W,C] (C in 1..4) of the same
        H x W; numpy arrays or CPU / CUDA tensors; `invert` one flag or one per request.  Returns the inpainted photos, uint8
        [H,W,3]: numpy for numpy photos, a tensor on the photo's device otherwise.  `last_extents` holds every (Hp, Wp).
        Every refusal (TypeError for a non-array, ValueError naming the request otherwise) comes before anything is enqueued.

        wait=False only enqueues the work on the current stream and returns the output tensors, which hold the results
        (and `last_extents` is set) after `wait()`.  CPU photos must then be pinned tensors (`pin_memory()`), since they are
        copied asynchronously; pageable CPU masks are staged through pinned memory."""
        imgs, masks = list(imgs), list(masks)
        if len(imgs) != len(masks):
            raise ValueError("FullResPipeline.forward_batch: %d photos and %d masks" % (len(imgs), len(masks)))
        inverts = [bool(invert)] * len(imgs) if isinstance(invert, (bool, int)) else [bool(v) for v in invert]
        if len(inverts) != len(imgs):
            raise ValueError("FullResPipeline.forward_batch: %d invert flags for %d requests" % (len(inverts), len(imgs)))
        dev = self._device()
        with torch.cuda.device(dev):
            eng = self.model._engine(dev)
            kinds, checked, extents, max_n = [], [], [], {}
            for i, (img, mask) in enumerate(zip(imgs, masks)):
                kinds.append(self._kind(i, img, wait))
                img, mask = self._check(i, img, mask)
                ext, mx = self._extent(eng, i, int(img.shape[0]), int(img.shape[1]))
                checked.append((img, mask))
                extents.append(ext)
                max_n[ext] = mx
            if not imgs:
                return []
            passes = plan_passes(extents, max_n)
            need = max(eng.lib.migan_workspace_bytes_hw(eng.handle, len(c.requests), c.Hp, c.Wp) for p in passes for c in p)
            ws = self._workspace(eng, need)
            nb = not wait
            imgs_d = [_to(t, dev, nb) for t, _ in checked]
            masks_d = [_to(m, dev, nb) for _, m in checked]
            outs_d = [torch.empty((int(t.shape[0]), int(t.shape[1]), 3), dtype=torch.uint8, device=dev) for t, _ in checked]
            stream = torch.cuda.current_stream(dev).cuda_stream
            keep = [imgs_d, masks_d, outs_d, ws]
            for chunks in passes:
                keep.append(self._pass(eng, chunks, imgs_d, masks_d, inverts, outs_d, ws, stream))
            results = []
            for kind, out in zip(kinds, outs_d):
                if kind == "cuda":
                    results.append(out)
                else:
                    host = torch.empty(out.shape, dtype=torch.uint8, pin_memory=True)
                    host.copy_(out, non_blocking=True)
                    results.append(host)
            event = torch.cuda.Event()
            event.record(torch.cuda.current_stream(dev))
        call = _Call(event, extents, keep)
        if wait:
            self._finish([call])
            return [r.numpy() if kind == "numpy" else r for kind, r in zip(kinds, results)]
        self._pending.append(call)
        return results

    def _finish(self, calls) -> None:
        extents = []
        for call in calls:
            call.event.synchronize()
            extents += call.sizes
        if extents:
            self.last_extents = extents
