"""Device-planned crop pipeline on the H100: `MIGAN_Pipeline.forward_batch(..., wait=False)` and the planned C entry points.

* the planning kernel's windows equal `migan_crop_box` on the host flags for edge cases of its load scheme (flag offsets
  at every alignment, widths below / not a multiple of 16, all-known and all-hole masks, holes at the borders, a 4K mask);
* a planned pass with the generator output given: the reference vectors bit for bit, and a 24-request random batch equal
  to the host-box batched calls, boxes and model input included;
* the real generator: two `forward_batch(..., wait=False)` calls back to back, pinned CPU requests among them, then `wait()`,
  equal the sequential `pipe(...)` calls byte for byte;
* no host synchronisation: with the stream held busy, `forward_batch(..., wait=False)` returns before it drains;
* pageable CPU images are refused with wait=False."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from migan_b200 import _abi, ops, synthetic
from migan_b200.pipeline import MIGAN_Pipeline

sys.path.insert(0, os.path.dirname(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import make_golden_pipeline as MG  # noqa: E402  (case table + seeded inputs only)
from test_pipeline_batch_gpu import GivenOutput, _mixed_requests, _sequential  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = MG.load_fixture()
_PIPES = {}


def _pipe(res, pad, device):
    if res not in _PIPES:
        _PIPES[res] = MIGAN_Pipeline(synthetic.export_style_state_dict(res, seed=11), res, padding=pad, device=device)
    p = _PIPES[res]
    p.padding = pad
    return p


def _reqs(images, masks):
    reqs = (_abi.PipeRequest * len(images))()
    for r, im, m in zip(reqs, images, masks):
        r.image, r.mask, r.H, r.W = im.data_ptr(), m.data_ptr(), int(m.shape[0]), int(m.shape[1])
    return reqs


def _planned_boxes(masks, res, pad):
    """Flags + planning launch on device masks [H,W]; returns the boxes and the flags on the host."""
    lib = _abi.load()
    dev = masks[0].device
    stream = torch.cuda.current_stream(dev).cuda_stream
    n = len(masks)
    reqs = _reqs(masks, masks)                                          # the plan does not read the images
    flags = torch.empty(sum(r.W + r.H for r in reqs), dtype=torch.uint8, device=dev)
    _abi.check(lib.b200_hole_flags_batch(reqs, n, flags.data_ptr(), stream))
    need = lib.b200_pipeline_batch_scratch_bound(reqs, n, res)
    scratch = torch.empty(need, dtype=torch.uint8, device=dev)
    boxes = torch.full((n, 4), -1, dtype=torch.int32, device=dev)
    _abi.check(lib.b200_pipeline_plan_batch(reqs, n, res, pad, flags.data_ptr(), boxes.data_ptr(), scratch.data_ptr(), need, stream))
    return boxes.cpu(), flags.cpu()


def _host_boxes(flags, masks, res, pad):
    lib = _abi.load()
    out, off = [], 0
    box = torch.zeros(4, dtype=torch.int32)
    for m in masks:
        H, W = int(m.shape[0]), int(m.shape[1])
        _abi.check(lib.migan_crop_box(flags.data_ptr() + off, H, W, res, pad, box.data_ptr()))
        out.append(tuple(int(v) for v in box))
        off += W + H
    return out


def test_planned_boxes_edge_cases(cuda_device):
    g = torch.Generator(device="cpu").manual_seed(9)

    def holes(H, W, *rects):
        m = torch.full((H, W), 255, dtype=torch.uint8)
        for a, b, c, d in rects:
            m[a:b, c:d] = 0
        return m

    cases = [torch.full((40, 50), 255, dtype=torch.uint8), torch.zeros((40, 50), dtype=torch.uint8),
             holes(40, 50, (0, 1, 10, 20)), holes(40, 50, (39, 40, 10, 20)), holes(40, 50, (5, 9, 0, 1)),
             holes(40, 50, (5, 9, 49, 50)), holes(3, 3), torch.zeros((3, 3), dtype=torch.uint8), holes(3, 3, (1, 2, 1, 2)),
             holes(3, 200, (0, 3, 150, 151)), holes(3, 1001, (1, 2, 0, 1), (2, 3, 1000, 1001)),
             holes(2160, 3840, (700, 1300, 1000, 1900), (2159, 2160, 3839, 3840)), holes(2160, 3840)]
    for W in (1, 5, 15, 16, 17, 31, 33, 47, 64, 100, 515):                # flag offsets at every alignment
        m = torch.full((7, W + 2), 255, dtype=torch.uint8)
        m[torch.rand(7, W + 2, generator=g) < 0.05] = 0
        cases.append(m)
    cases = cases[:_abi.PIPE_MAX_BATCH]
    masks = [c.to(cuda_device) for c in cases]
    for res, pad in ((64, 0), (64, 128), (3, 0), (512, 16)):
        boxes, flags = _planned_boxes(masks, res, pad)
        assert [tuple(int(v) for v in b) for b in boxes] == _host_boxes(flags, cases, res, pad), (res, pad)


def test_reference_cases_planned(cuda_device):
    cases = [c for c in MG.CASES if c[1] == 64]
    pipe = _pipe(64, cases[0][2], cuda_device)
    real = pipe.model
    inputs = [MG.case_inputs(c) for c in cases]
    try:
        pipe.model = GivenOutput(torch.from_numpy(np.concatenate([GOLD["y_" + c[0]] for c in cases])).to(cuda_device))
        images = [im.to(cuda_device) for im, _ in inputs]
        out = pipe.forward_batch(images, [m.to(cuda_device) for _, m in inputs], wait=False)
        pipe.wait()
        for i, c in enumerate(cases):
            tag = c[0]
            assert pipe.last_boxes[i] == tuple(int(v) for v in GOLD["box_" + tag]), tag
            x = pipe.model.x[i:i + 1].cpu()
            assert torch.equal(MG.on_stored_rows(GOLD, "x", tag, x), torch.from_numpy(GOLD["x_" + tag])), tag
            assert np.array_equal(MG.on_stored_rows(GOLD, "final", tag, out[i].cpu().numpy()), GOLD["final_" + tag]), tag
    finally:
        pipe.model = real


def _host_box_pass(images, masks, res, pad, y):
    """The host-box batched calls on device images [3,H,W] (updated in place) and masks [H,W]; returns (boxes, x)."""
    lib = _abi.load()
    dev = images[0].device
    stream = torch.cuda.current_stream(dev).cuda_stream
    n = len(images)
    reqs = _reqs(images, masks)
    flags = torch.empty(sum(r.W + r.H for r in reqs), dtype=torch.uint8, device=dev)
    _abi.check(lib.b200_hole_flags_batch(reqs, n, flags.data_ptr(), stream))
    flags_h = flags.cpu()
    off = 0
    for r in reqs:
        _abi.check(lib.migan_crop_box(flags_h.data_ptr() + off, r.H, r.W, res, pad, ctypes.addressof(r.box)))
        off += r.W + r.H
    need = lib.b200_pipeline_batch_scratch_bytes(reqs, n, res)
    scratch = torch.empty(need, dtype=torch.uint8, device=dev)
    x = torch.empty((n, 4, res, res), dtype=torch.float32, device=dev)
    _abi.check(lib.b200_pipeline_preprocess_batch(reqs, n, res, x.data_ptr(), scratch.data_ptr(), need, stream))
    k = ops.feather_kernel(5, 1.0).contiguous()
    _abi.check(lib.b200_pipeline_postprocess_batch(y.data_ptr(), reqs, n, res, k.data_ptr(), scratch.data_ptr(), need, stream))
    return [tuple(int(v) for v in r.box) for r in reqs], x


def test_random_batch_planned_equals_host_boxes(cuda_device):
    rng = np.random.RandomState(654)
    sizes = [(257, 255), (720, 1280), (64, 64), (65, 1000), (1100, 90), (333, 777), (3, 3), (9, 500)]
    reqs = _mixed_requests(rng, 24, sizes)
    y = torch.randn(24, 3, 64, 64, generator=torch.Generator().manual_seed(655)).to(cuda_device)
    pipe = _pipe(64, 16, cuda_device)
    real = pipe.model
    try:
        pipe.model = GivenOutput(y)
        images = [im.clone().to(cuda_device) for im, _ in reqs]
        masks = [m.to(cuda_device) for _, m in reqs]
        out = pipe.forward_batch(images, masks)
        masks_full = []
        for im, m in zip(images, masks):                                # the host-box calls take masks at the image size
            H, W = int(im.shape[2]), int(im.shape[3])
            m = m[0, 0]
            if tuple(m.shape) != (H, W):
                m2 = torch.empty((H, W), dtype=torch.uint8, device=cuda_device)
                _abi.check(_abi.load().b200_resize_nearest_u8(m.data_ptr(), int(m.shape[0]), int(m.shape[1]), m2.data_ptr(), H, W,
                                                              torch.cuda.current_stream(cuda_device).cuda_stream))
                m = m2
            masks_full.append(m)
        want_images = [im.clone().to(cuda_device)[0] for im, _ in reqs]
        want_boxes, want_x = _host_box_pass(want_images, masks_full, 64, 16, y)
        assert pipe.last_boxes == want_boxes
        assert torch.equal(pipe.model.x, want_x)
        for i in range(24):
            assert torch.equal(out[i][0], want_images[i]), (i, int((out[i][0] != want_images[i]).sum()))
    finally:
        pipe.model = real


def test_wait_false_equals_sequential_calls(cuda_device):
    """Real generator: 40 mixed-size requests, some as pinned CPU tensors, as two wait=False calls (passes of 32 + 2, then
    6), then one wait()."""
    rng = np.random.RandomState(56)
    sizes = [(256, 256), (300, 420), (120, 100), (90, 700), (64, 64), (500, 333), (41, 45), (720, 1280)]
    reqs = [(im.to(cuda_device), m.to(cuda_device)) for im, m in _mixed_requests(rng, 40, sizes)]
    for i in (3, 17, 35, 38):
        reqs[i] = (reqs[i][0].cpu().pin_memory(), reqs[i][1].cpu().pin_memory())
    reqs[20] = (reqs[20][0], reqs[20][1].cpu())                         # a pageable CPU mask is staged
    pipe = _pipe(64, 32, cuda_device)
    want, want_boxes = _sequential(pipe, reqs)
    images = [im.clone() for im, _ in reqs]
    for i in (3, 17, 35, 38):
        images[i] = images[i].pin_memory()
    masks = [m for _, m in reqs]
    first = pipe.forward_batch(images[:34], masks[:34], wait=False)
    second = pipe.forward_batch(images[34:], masks[34:], wait=False)
    pipe.wait()
    out = first + second
    assert out[3] is images[3] and not out[3].is_cuda
    assert pipe.last_boxes == want_boxes
    assert pipe.last_box == want_boxes[-1]
    for i in range(40):
        assert torch.equal(out[i].cpu(), want[i]), (i, int((out[i].cpu() != want[i]).sum()))
    pipe.wait()                                                         # nothing outstanding: a no-op
    assert pipe.last_boxes == want_boxes


def test_wait_false_does_not_synchronise(cuda_device):
    """With the stream held busy by a sleep kernel, the call returns while the stream still has work queued."""
    rng = np.random.RandomState(57)
    reqs = _mixed_requests(rng, 6, [(200, 300), (64, 64), (480, 640)])
    pipe = _pipe(64, 32, cuda_device)
    for on_gpu in (True, False):
        if on_gpu:
            src = [(im.to(cuda_device), m.to(cuda_device)) for im, m in reqs]
        else:
            src = [(im.pin_memory(), m.pin_memory()) for im, m in reqs]
        want = [im.clone() for im, _ in src]
        pipe.forward_batch(want, [m for _, m in src])                   # warm-up at the same sizes, and the expected bytes
        torch.cuda.synchronize(cuda_device)
        images = [im.clone() for im, _ in src]
        if not on_gpu:
            images = [im.pin_memory() for im in images]
        stream = torch.cuda.current_stream(cuda_device)
        torch.cuda._sleep(1_000_000_000)
        pipe.forward_batch(images, [m for _, m in src], wait=False)
        busy = not stream.query()
        pipe.wait()
        assert busy, "forward_batch(wait=False) waited for the stream (%s requests)" % ("CUDA" if on_gpu else "pinned CPU")
        for a, b in zip(images, want):
            assert torch.equal(a.cpu(), b.cpu())


def test_pageable_images_refused_without_wait(cuda_device):
    pipe = _pipe(64, 16, cuda_device)
    image = torch.full((1, 3, 40, 50), 7, dtype=torch.uint8)
    mask = torch.zeros((1, 1, 40, 50), dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="pinned"):
        pipe.forward_batch([image], [mask], wait=False)
    assert bool((image == 7).all())
    assert pipe.forward_batch([image], [mask], wait=True)[0] is image   # the synchronous form takes pageable memory
    assert not bool((image == 7).all())
