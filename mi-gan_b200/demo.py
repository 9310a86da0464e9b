"""`DemoPipeline`: the reference demo's request path (scripts/demo.py:26-66, :120-143) at any photo size, on the GPU.

    pipe = DemoPipeline(state_dict_or_generator, resolution=512)
    composed = pipe(img, mask, invert=False)          # img uint8 [H,W,3]; mask uint8 [H,W] / [H,W,2|3|4]
    outs = pipe.forward_batch(imgs, masks)            # many photos of any sizes, one generator forward per 32
    pipe.forward_batch(imgs_t, masks_t, wait=False)   # only enqueue (serving loop) ...
    pipe.wait()                                       # ... outputs written, pipe.last_sizes set

`img` is `np.array(Image.open(p).convert("RGB"))` and `mask` is `np.array(Image.open(mask_path))` in any mode `read_mask`
handles (L, LA, RGB, RGBA; it may have its own size).  The result is byte for byte the image demo.py saves: its size is
that of `resize(img, max_size=R)`.  Per pass of up to 32 requests (kernels in csrc/demo_resize.cu behind
include/migan_b200.h, one launch per stage for every request):

    tables -> [PIL BICUBIC down-scale of the photos larger than R: width pass, height pass] -> PIL BICUBIC to R x R + the
    mask's NEAREST chain + x  ->  Generator.forward at the pass's batch size  ->  uint8 + OpenCV INTER_CUBIC width pass
    -> height pass + composite

OpenCV's cubic resize is reproduced as its scalar path computes it (`cv2.setUseOptimized(False)`); OpenCV's default
optimised path differs from it by at most 1 in a small fraction of values.  The generator's output does not depend on the
batch size, so request i of a batch gets the bytes of a call with request i alone.  There is no CPU path.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple, Union

import numpy as np
import torch

from . import _abi
from .generator import Generator

MASK_MAX = 512          # read_mask's first resize (demo.py:28)


def resized_size(w: int, h: int, max_size: int) -> Tuple[int, int]:
    """demo.py `resize` (:48-53): the (w, h) of an image after its down-scale to at most max_size."""
    if w > max_size or h > max_size:
        ratio = max_size / w if w > h else max_size / h
        return int(w * ratio), int(h * ratio)
    return w, h


class DemoPipeline(torch.nn.Module):
    """`model_or_state_dict`: a `migan_b200.Generator`, a state_dict, or a file `torch.load` reads one from."""

    def __init__(self, model_or_state_dict, resolution: int, device: Union[str, torch.device] = "cuda"):
        super().__init__()
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("migan_b200.DemoPipeline runs on a CUDA device (there is no CPU path); got %s" % device)
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
        self.device_ = device
        self._pending: List["_Call"] = []
        self.last_sizes: List[Tuple[int, int]] = []       # (w', h') of every result of the last completed call(s)
        self.last_launches = 0                             # kernel launches (generator excluded) of the last pass

    def __call__(self, img, mask, invert: bool = False):
        return self.forward_batch([img], [mask], invert=invert)[0]

    # -- one pass ---------------------------------------------------------------------------------------------------
    def _pass(self, imgs, masks, inverts, outs) -> None:
        """Enqueue one pass over <= 32 requests: imgs [H,W,3] / masks [Hm,Wm,C] uint8 CUDA contiguous, outs [h',w',3]
        uint8 CUDA contiguous, all on one device."""
        lib = _abi.load()
        n = len(imgs)
        dev = imgs[0].device
        stream = torch.cuda.current_stream(dev).cuda_stream
        reqs = (_abi.DemoRequest * n)()
        for r, img, m, inv, out in zip(reqs, imgs, masks, inverts, outs):
            r.img, r.H, r.W = img.data_ptr(), int(img.shape[0]), int(img.shape[1])
            r.mask, r.Hm, r.Wm, r.mask_channels = m.data_ptr(), int(m.shape[0]), int(m.shape[1]), int(m.shape[2])
            r.invert = int(bool(inv))
            r.out, r.out_h, r.out_w = out.data_ptr(), int(out.shape[0]), int(out.shape[1])
        need = int(lib.b200_demo_scratch_bytes(reqs, n, self.res))
        if need == 0:
            _abi.check(_abi.ERR_INVALID)
        with torch.cuda.device(dev):
            # the caching allocator hands the scratch to the next pass on this stream in order
            scratch = torch.empty(need, dtype=torch.uint8, device=dev)
            x = torch.empty((n, 4, self.res, self.res), dtype=torch.float32, device=dev)
            _abi.check(lib.b200_demo_preprocess(reqs, n, self.res, x.data_ptr(), scratch.data_ptr(), need, stream))
            y = self.model(x)
            if y.dtype != torch.float32 or tuple(y.shape) != (n, 3, self.res, self.res) or not y.is_contiguous():
                raise RuntimeError("generator output must be contiguous float32 (%d,3,%d,%d)" % (n, self.res, self.res))
            _abi.check(lib.b200_demo_postprocess(y.data_ptr(), reqs, n, self.res, scratch.data_ptr(), need, stream))
        down = any((int(r.out_w), int(r.out_h)) != (int(r.W), int(r.H)) for r in reqs)
        self.last_launches = 2 + (2 if down else 0) + 2

    # -- public calls -----------------------------------------------------------------------------------------------
    def _check(self, i, img, mask):
        """(photo tensor [H,W,3], mask tensor [Hm,Wm,C], (w', h')) of request i; ValueError where demo.py fails."""
        img = torch.from_numpy(np.ascontiguousarray(img)) if isinstance(img, np.ndarray) else img
        mask = torch.from_numpy(np.ascontiguousarray(mask)) if isinstance(mask, np.ndarray) else mask
        if not isinstance(img, torch.Tensor) or not isinstance(mask, torch.Tensor):
            raise TypeError("DemoPipeline: request %d: photo and mask must be numpy arrays or torch tensors" % i)
        if img.dtype != torch.uint8 or mask.dtype != torch.uint8:
            raise ValueError("DemoPipeline: request %d: photo and mask must be uint8" % i)
        if img.dim() != 3 or img.shape[2] != 3 or img.shape[0] < 1 or img.shape[1] < 1:
            raise ValueError("DemoPipeline: request %d: photo of shape %s, expected [H, W, 3]" % (i, tuple(img.shape)))
        if mask.dim() == 2:
            mask = mask.unsqueeze(2)
        if mask.dim() != 3 or not 1 <= mask.shape[2] <= 4 or mask.shape[0] < 1 or mask.shape[1] < 1:
            raise ValueError("DemoPipeline: request %d: mask of shape %s, expected [H, W] or [H, W, 1..4]" % (i, tuple(mask.shape)))
        H, W, Hm, Wm = int(img.shape[0]), int(img.shape[1]), int(mask.shape[0]), int(mask.shape[1])
        w1, h1 = resized_size(W, H, self.res)
        wb, hb = resized_size(*resized_size(Wm, Hm, MASK_MAX), self.res)
        if min(w1, h1, wb, hb) < 1 or min(resized_size(Wm, Hm, MASK_MAX)) < 1:
            raise ValueError("DemoPipeline: request %d: photo %dx%d or mask %dx%d resizes to a 0-pixel side at resolution %d"
                             % (i, W, H, Wm, Hm, self.res))
        if (wb, hb) != (w1, h1):
            raise ValueError("DemoPipeline: request %d: the mask resizes to %dx%d and the photo to %dx%d (w x h); demo.py "
                             "cannot compose them" % (i, wb, hb, w1, h1))
        return img, mask, (w1, h1)

    @torch.no_grad()
    def forward_batch(self, imgs: Sequence, masks: Sequence, invert: Union[bool, Sequence[bool]] = False,
                      wait: bool = True) -> list:
        """Many requests of any sizes, one pass per 32.  imgs[i]: uint8 [H,W,3]; masks[i]: uint8 [Hm,Wm] or [Hm,Wm,C];
        numpy arrays or CPU / CUDA tensors; `invert` one flag or one per request.  Returns the composed images, uint8
        [h',w',3]: numpy for numpy photos, a tensor on the photo's device otherwise.  `last_sizes` holds every (w', h').

        wait=False only enqueues the work on the current stream and returns the output tensors, which hold the results
        (and `last_sizes` is set) after `wait()`.  CPU photos must then be pinned tensors (`pin_memory()`), since they are
        copied asynchronously; pageable CPU masks are staged through pinned memory."""
        imgs, masks = list(imgs), list(masks)
        if len(imgs) != len(masks):
            raise ValueError("DemoPipeline.forward_batch: %d photos and %d masks" % (len(imgs), len(masks)))
        inverts = [bool(invert)] * len(imgs) if isinstance(invert, (bool, int)) else [bool(v) for v in invert]
        if len(inverts) != len(imgs):
            raise ValueError("DemoPipeline.forward_batch: %d invert flags for %d requests" % (len(inverts), len(imgs)))
        kinds, checked = [], []
        for i, (img, mask) in enumerate(zip(imgs, masks)):
            kinds.append("numpy" if isinstance(img, np.ndarray) else ("cuda" if img.is_cuda else "cpu"))
            if not wait and kinds[-1] != "cuda" and not (kinds[-1] == "cpu" and img.is_pinned() and img.is_contiguous()):
                raise RuntimeError("DemoPipeline.forward_batch(wait=False): CPU photo %d must be a pinned contiguous tensor "
                                   "(it is copied asynchronously); use torch.from_numpy(img).pin_memory() or wait=True" % i)
            checked.append(self._check(i, img, mask))
        if not imgs:
            return []
        dev = next((t.device for t, _, _ in checked if t.is_cuda), self.device_)
        nb = not wait
        imgs_d = [_to(t, dev, nb) for t, _, _ in checked]
        masks_d = [_to(m, dev, nb) for _, m, _ in checked]
        outs_d = [torch.empty((h, w, 3), dtype=torch.uint8, device=dev) for _, _, (w, h) in checked]
        for c in range(0, len(imgs), _abi.PIPE_MAX_BATCH):
            s = slice(c, c + _abi.PIPE_MAX_BATCH)
            self._pass(imgs_d[s], masks_d[s], inverts[s], outs_d[s])
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
        call = _Call(event, [size for _, _, size in checked], (imgs_d, masks_d, outs_d))
        if wait:
            self._finish([call])
            return [r.numpy() if kind == "numpy" else r for kind, r in zip(kinds, results)]
        self._pending.append(call)
        return results

    def _finish(self, calls) -> None:
        sizes = []
        for call in calls:
            call.event.synchronize()
            sizes += call.sizes
        if sizes:
            self.last_sizes = sizes

    def wait(self) -> None:
        """Block until every call enqueued with `forward_batch(..., wait=False)` has finished: its outputs are written and
        `last_sizes` holds the sizes of all those calls' results, in submission order."""
        calls, self._pending = self._pending, []
        self._finish(calls)


class _Call:
    """One enqueued call: the event after its last copy, the result sizes, and the tensors its enqueued work reads or
    writes (kept alive until the call is waited for)."""

    def __init__(self, event, sizes, keep):
        self.event, self.sizes, self.keep = event, sizes, keep


def _to(t: torch.Tensor, device, non_blocking: bool) -> torch.Tensor:
    """`t` contiguous on `device`.  A non-blocking copy from pageable memory would wait for the stream, so a pageable CPU
    tensor is first staged by a host copy into pinned memory."""
    if non_blocking and not t.is_cuda and not t.is_pinned():
        t = t.pin_memory()
    return t.to(device, non_blocking=non_blocking).contiguous()
