"""Batched crop pipeline on the H100: `MIGAN_Pipeline.forward_batch` and the batched C entry points under it.

* the batched hole-flags kernel against torch on the edge cases of its load scheme (widths below / not a multiple of 16,
  3 rows, unaligned mask bases, all-known and all-hole masks, a 4K mask, widths over one column tile);
* the reference vectors and random mixed-size requests in one call, generator output given: bit-exact;
* the real generator: `forward_batch` equals the sequential `pipe(...)` calls byte for byte, CPU requests included, over
  a 32 + 8 split, on a non-default stream; overlapping images are refused."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from migan_b200 import _abi, synthetic
from migan_b200.pipeline import MIGAN_Pipeline
from oracle import pipeline_oracle as PO

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import make_golden_pipeline as MG  # noqa: E402  (case table + seeded inputs only)

pytestmark = pytest.mark.gpu
GOLD = MG.load_fixture()


class GivenOutput(torch.nn.Module):
    """Stands in for the generator: records the model input, returns a fixed y."""

    def __init__(self, y):
        super().__init__()
        self.y, self.x = y, None

    def forward(self, x):
        self.x = x.clone()
        return self.y


_PIPES = {}


def _pipe(res, pad, device):
    if res not in _PIPES:
        _PIPES[res] = MIGAN_Pipeline(synthetic.export_style_state_dict(res, seed=11), res, padding=pad, device=device)
    p = _PIPES[res]
    p.padding = pad
    return p


def _flags_batch(masks):
    lib = _abi.load()
    reqs = (_abi.PipeRequest * len(masks))()
    for r, m in zip(reqs, masks):
        r.image, r.mask, r.H, r.W = m.data_ptr(), m.data_ptr(), int(m.shape[0]), int(m.shape[1])
    flags = torch.full((sum(r.W + r.H for r in reqs),), 7, dtype=torch.uint8, device=masks[0].device)
    _abi.check(lib.b200_hole_flags_batch(reqs, len(masks), flags.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return flags.cpu()


def test_hole_flags_batch_edge_cases(cuda_device):
    g = torch.Generator(device="cpu").manual_seed(5)

    def sparse(H, W, p):
        m = torch.full((H, W), 255, dtype=torch.uint8)
        m[torch.rand(H, W, generator=g) < p] = torch.randint(0, 255, (1,), generator=g).to(torch.uint8)
        return m

    stack = sparse(2 * 7 * 13, 1, 0.02).view(2, 7, 13)                 # H*W odd: stack[1] starts 91 bytes in (not 16-aligned)
    big = torch.full((2160, 3840), 255, dtype=torch.uint8)
    big[700:1300, 1000:1900] = 0
    big[2159, 3839] = 254
    cases = [
        sparse(3, 3, 0.3), sparse(3, 5, 0.3), sparse(3, 15, 0.1), sparse(5, 17, 0.05), sparse(3, 16, 0.1),
        sparse(64, 31, 0.002), sparse(33, 1000, 0.0005), sparse(17, 257, 0.003),
        torch.full((40, 37), 255, dtype=torch.uint8), torch.zeros((19, 45), dtype=torch.uint8),
        sparse(3, 20000, 0.0002), big,                                  # one / several column tiles of 8192
    ]
    dev = [c.to(cuda_device) for c in cases]
    stack_d = stack.to(cuda_device)
    dev += [stack_d[0], stack_d[1]]
    cases += [stack[0], stack[1]]
    assert stack_d[1].data_ptr() % 16 != 0
    offsets = [1, 2, 3, 5, 7, 9, 11, 13, 15]                            # unaligned copies of a mask with holes in the row heads / tails
    base = torch.full((9, 45), 255, dtype=torch.uint8)
    base[:, 0] = 0; base[4, 44] = 3; base[8, 20] = 254
    for o in offsets:
        buf = torch.full((o + base.numel(),), 255, dtype=torch.uint8, device=cuda_device)
        buf[o:] = base.flatten().to(cuda_device)
        dev.append(buf[o:].view(9, 45))
        cases.append(base)
    assert len(dev) <= _abi.PIPE_MAX_BATCH
    flags = _flags_batch(dev)
    off = 0
    for i, m in enumerate(cases):
        H, W = m.shape
        want = torch.cat([(m < 255).any(dim=0), (m < 255).any(dim=1)]).to(torch.uint8)
        assert torch.equal(flags[off:off + W + H], want), (i, H, W)
        off += W + H


def test_reference_cases_in_one_batch(cuda_device):
    cases = [c for c in MG.CASES if c[1] == 64]
    pipe = _pipe(64, cases[0][2], cuda_device)
    real = pipe.model
    inputs = [MG.case_inputs(c) for c in cases]
    try:
        pipe.model = GivenOutput(torch.from_numpy(np.concatenate([GOLD["y_" + c[0]] for c in cases])).to(cuda_device))
        images = [im.to(cuda_device) for im, _ in inputs]
        ptrs = [im.data_ptr() for im in images]
        out = pipe.forward_batch(images, [m.to(cuda_device) for _, m in inputs])
        assert [o.data_ptr() for o in out] == ptrs                      # in place
        for i, c in enumerate(cases):
            tag = c[0]
            assert pipe.last_boxes[i] == tuple(int(v) for v in GOLD["box_" + tag]), tag
            x = pipe.model.x[i:i + 1].cpu()
            assert torch.equal(MG.on_stored_rows(GOLD, "x", tag, x), torch.from_numpy(GOLD["x_" + tag])), tag
            assert np.array_equal(MG.on_stored_rows(GOLD, "final", tag, out[i].cpu().numpy()), GOLD["final_" + tag]), tag
        assert pipe.last_box == pipe.last_boxes[-1]
    finally:
        pipe.model = real


def _mixed_requests(rng, n, sizes):
    reqs = []
    for i in range(n):
        H, W = sizes[i % len(sizes)]
        image = torch.from_numpy(rng.randint(0, 256, size=(1, 3, H, W), dtype=np.uint8))
        mask = torch.full((1, 1, H, W), 255, dtype=torch.uint8)
        kind = i % 4
        if kind == 1:                                                   # at a border
            mask[:, :, : H // 3, W - W // 4:] = 0
        elif kind >= 2:
            a, b = sorted(rng.randint(0, H, 2)); c, d = sorted(rng.randint(0, W, 2))
            mask[:, :, a:b + 1, c:d + 1] = 0
        if i % 5 == 4:                                                  # mask at another size
            mask = torch.nn.functional.interpolate(mask.float(), size=(max(3, H // 2), max(3, W // 2)), mode="nearest").to(torch.uint8)
        reqs.append((image, mask))
    return reqs


def test_random_mixed_batch_against_oracle(cuda_device):
    rng = np.random.RandomState(321)
    sizes = [(257, 255), (720, 1280), (64, 64), (65, 1000), (1100, 90), (333, 777), (3, 3), (9, 500)]
    reqs = _mixed_requests(rng, 24, sizes)
    y = torch.randn(24, 3, 64, 64, generator=torch.Generator().manual_seed(322))
    pipe = _pipe(64, 16, cuda_device)
    real = pipe.model
    try:
        pipe.model = GivenOutput(y.to(cuda_device))
        out = pipe.forward_batch([im.clone().to(cuda_device) for im, _ in reqs], [m.to(cuda_device) for _, m in reqs])
        for i, (image, mask) in enumerate(reqs):
            taps = {}
            want = PO.forward(lambda _x: y[i:i + 1], image.clone(), mask, 64, 16, taps)
            assert pipe.last_boxes[i] == taps["box"], i
            assert torch.equal(pipe.model.x[i:i + 1].cpu(), taps["x"]), i
            got = out[i].cpu()
            assert torch.equal(got, want), (i, int((got != want).sum()))
    finally:
        pipe.model = real


def _sequential(pipe, reqs):
    outs, boxes = [], []
    for image, mask in reqs:
        outs.append(pipe(image.clone(), mask.clone()).cpu())
        boxes.append(pipe.last_box)
    return outs, boxes


def test_forward_batch_equals_sequential_calls(cuda_device):
    """Real generator: 40 mixed-size requests (two of them CPU tensors) run as 32 + 8, against one call per request."""
    rng = np.random.RandomState(55)
    sizes = [(256, 256), (300, 420), (120, 100), (90, 700), (64, 64), (500, 333), (41, 45), (720, 1280)]
    reqs = [(im.to(cuda_device), m.to(cuda_device)) for im, m in _mixed_requests(rng, 40, sizes)]
    reqs[3] = (reqs[3][0].cpu(), reqs[3][1].cpu())
    reqs[35] = (reqs[35][0].cpu(), reqs[35][1].cpu())
    pipe = _pipe(64, 32, cuda_device)
    want, want_boxes = _sequential(pipe, reqs)
    images = [im.clone() for im, _ in reqs]
    out = pipe.forward_batch(images, [m for _, m in reqs])
    assert out[3] is images[3] and not out[3].is_cuda
    assert pipe.last_boxes == want_boxes
    for i in range(40):
        assert torch.equal(out[i].cpu(), want[i]), (i, int((out[i].cpu() != want[i]).sum()))
    # 8 requests on a non-default stream
    images = [im.clone() for im, _ in reqs[:8]]
    s = torch.cuda.Stream(device=cuda_device)
    s.wait_stream(torch.cuda.current_stream(cuda_device))
    with torch.cuda.stream(s):
        out = pipe.forward_batch(images, [m for _, m in reqs[:8]])
    s.synchronize()
    for i in range(8):
        assert torch.equal(out[i].cpu(), want[i]), i
    # forward with N > 1 takes the same path
    same = torch.stack([reqs[k][0][0].cpu() for k in (0, 8, 16)])
    masks = torch.stack([reqs[k][1][0].cpu() for k in (0, 8, 16)])
    both = pipe(same.clone().to(cuda_device), masks.to(cuda_device)).cpu()
    for j, k in enumerate((0, 8, 16)):
        assert torch.equal(both[j:j + 1], want[k])


def test_overlapping_images_are_refused(cuda_device):
    pipe = _pipe(64, 16, cuda_device)
    buf = torch.full((1, 3, 100, 120), 7, dtype=torch.uint8, device=cuda_device)
    mask = torch.full((1, 1, 100, 120), 0, dtype=torch.uint8, device=cuda_device)
    with pytest.raises(RuntimeError, match="overlaps"):
        pipe.forward_batch([buf, buf[:, :, 10:]], [mask, mask])
    flat = torch.full((3 * 100 * 120 + 100 * 120,), 255, dtype=torch.uint8, device=cuda_device)
    with pytest.raises(RuntimeError, match="overlaps"):                  # an image that is also a mask
        pipe.forward_batch([flat[:3 * 100 * 120].view(1, 3, 100, 120)], [flat[100 * 120:2 * 100 * 120].view(1, 1, 100, 120)])
    assert bool((buf == 7).all())
    with pytest.raises(RuntimeError):
        pipe.forward_batch([buf], [mask, mask])
