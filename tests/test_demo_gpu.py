"""The demo request path on the H100 (mi-gan_b200/csrc/demo_resize.cu, migan_b200.demo.DemoPipeline):

* every stage equals the fixture of the reference's own functions (tests/golden/demo.npz) byte for byte;
* at R = 256 and 512, the 20 photo sizes of the reference's places2_512_object set plus a 1080 x 1920 and a 2160 x 3840
  photo in one pass: x, and the output of the post stage on the GPU generator's own y, equal oracle/demo_oracle.py;
* square R x R requests give exactly `Generator.forward_u8`'s bytes;
* `forward_batch` of 24 mixed requests equals the 24 single calls;
* two back-to-back `forward_batch(..., wait=False)` calls equal sequential ones, and the call returns before the stream
  drains; pageable CPU photos are refused with wait=False;
* a non-array photo is a TypeError, and a CUDA photo on another GPU than the pipeline's a ValueError, before any work."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from migan_b200 import _abi, synthetic
from migan_b200.demo import DemoPipeline
from migan_b200.generator import Generator

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from oracle import demo_oracle as O  # noqa: E402
import make_golden_demo as MG  # noqa: E402  (case table + seeded inputs only)

pytestmark = pytest.mark.gpu

# (W, H, mask channels) of examples/places2_512_object/{images,masks}/1..20.png, then a 1080p and a 4K photo
SIZES = [(512, 343, 3), (512, 380, 3), (512, 357, 3), (512, 340, 3), (512, 384, 3), (512, 384, 1), (512, 384, 1),
         (374, 512, 1), (384, 512, 1), (383, 512, 3), (512, 340, 3), (512, 332, 3), (512, 383, 3), (512, 340, 3),
         (401, 512, 3), (512, 384, 3), (512, 384, 3), (512, 340, 3), (512, 512, 3), (512, 512, 3),
         (1080, 1920, 4), (3840, 2160, 2)]
_PIPES = {}


def _pipe(res, device):
    if res not in _PIPES:
        _PIPES[res] = DemoPipeline(synthetic.export_style_state_dict(res, seed=5), res, device=device)
    return _PIPES[res]


def _request(rng, W, H, C):
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    m = np.full((H, W, C), 255, np.uint8)
    y0, x0 = int(rng.integers(0, H // 2)), int(rng.integers(0, W // 2))
    m[y0:y0 + H // 3, x0:x0 + W // 4] = rng.integers(0, 255, C, dtype=np.uint8)
    m = np.where(rng.random((H, W, 1)) < 0.03, 0, m).astype(np.uint8)
    return img, np.ascontiguousarray(m[..., 0] if C == 1 else m)


def _stages(reqs_np, inverts, res, dev, y=None, model=None):
    """The two C entry points on one pass: (x, outs, y) with y given or the model's own."""
    lib = _abi.load()
    stream = torch.cuda.current_stream(dev).cuda_stream
    n = len(reqs_np)
    imgs = [torch.from_numpy(i).to(dev) for i, _ in reqs_np]
    masks = [torch.from_numpy(m if m.ndim == 3 else m[..., None]).contiguous().to(dev) for _, m in reqs_np]
    outs = []
    reqs = (_abi.DemoRequest * n)()
    for r, img, m, inv in zip(reqs, imgs, masks, inverts):
        w1, h1 = O.resized_size(int(img.shape[1]), int(img.shape[0]), res)
        out = torch.full((h1, w1, 3), 3, dtype=torch.uint8, device=dev)
        outs.append(out)
        r.img, r.H, r.W = img.data_ptr(), int(img.shape[0]), int(img.shape[1])
        r.mask, r.Hm, r.Wm, r.mask_channels = m.data_ptr(), int(m.shape[0]), int(m.shape[1]), int(m.shape[2])
        r.invert, r.out, r.out_w, r.out_h = int(inv), out.data_ptr(), w1, h1
    need = lib.b200_demo_scratch_bytes(reqs, n, res)
    assert need > 0
    scratch = torch.empty(need, dtype=torch.uint8, device=dev)
    x = torch.full((n, 4, res, res), float("nan"), device=dev)
    _abi.check(lib.b200_demo_preprocess(reqs, n, res, x.data_ptr(), scratch.data_ptr(), need, stream))
    if y is None:
        y = model(x)
    y = y.to(dev).contiguous()
    _abi.check(lib.b200_demo_postprocess(y.data_ptr(), reqs, n, res, scratch.data_ptr(), need, stream))
    torch.cuda.synchronize(dev)
    return x.cpu().numpy(), [o.cpu().numpy() for o in outs], y.cpu().numpy()


def test_stages_equal_fixture(cuda_device):
    gold = MG.load_fixture()
    for i, (R, W, H, mode, invert) in enumerate(MG.CASES):
        img, mask, y = MG.case_inputs(i)
        x, outs, _ = _stages([(img, mask)], [invert], R, cuda_device, y=torch.from_numpy(y)[None])
        assert np.array_equal(x[0], gold["%d_x" % i]), i
        assert np.array_equal(outs[0], gold["%d_out" % i]), i
        assert np.abs(outs[0].astype(int) - gold["%d_out_default" % i].astype(int)).max() <= 1, i


@pytest.mark.parametrize("res", [256, 512])
def test_example_sizes_with_generator(cuda_device, res):
    rng = np.random.default_rng(res)
    reqs = [_request(rng, W, H, C) for W, H, C in SIZES]
    inverts = [k % 3 == 0 for k in range(len(reqs))]
    model = _pipe(res, cuda_device).model
    x, outs, y = _stages(reqs, inverts, res, cuda_device, model=model)
    for k, ((img, mask), inv) in enumerate(zip(reqs, inverts)):
        rs, m, ox = O.demo_pre(img, mask, inv, res)
        assert np.array_equal(x[k], ox), SIZES[k]
        assert np.array_equal(outs[k], O.demo_post(y[k], rs, m)), SIZES[k]


def test_square_requests_equal_forward_u8(cuda_device):
    res = 256
    pipe = _pipe(res, cuda_device)
    rng = np.random.default_rng(3)
    reqs = [_request(rng, res, res, 1) for _ in range(3)]
    got = pipe.forward_batch([i for i, _ in reqs], [m for _, m in reqs])
    img = torch.from_numpy(np.stack([i for i, _ in reqs]))
    mask = torch.from_numpy(np.stack([m for _, m in reqs]))
    want = pipe.model.forward_u8(img, mask)
    for k in range(3):
        assert np.array_equal(got[k], want[k].numpy()), k


def _mixed(rng, n, res):
    out = []
    while len(out) < n:
        W, H = int(rng.integers(8, 3 * res)), int(rng.integers(8, 3 * res))
        C = int(rng.choice([1, 2, 3, 4]))
        out.append(_request(rng, W, H, C) + (bool(rng.integers(0, 2)),))
    return out


def test_forward_batch_equals_single_calls(cuda_device):
    res = 256
    pipe = _pipe(res, cuda_device)
    reqs = _mixed(np.random.default_rng(4), 24, res)
    got = pipe.forward_batch([r[0] for r in reqs], [r[1] for r in reqs], invert=[r[2] for r in reqs])
    assert pipe.last_sizes == [O.resized_size(r[0].shape[1], r[0].shape[0], res) for r in reqs]
    for k, (img, mask, inv) in enumerate(reqs):
        assert np.array_equal(got[k], pipe(img, mask, invert=inv)), k


def test_wait_false_back_to_back(cuda_device):
    res = 256
    pipe = _pipe(res, cuda_device)
    reqs = _mixed(np.random.default_rng(6), 10, res)
    want = [pipe(i, m, invert=v) for i, m, v in reqs]
    a, b = reqs[:6], reqs[6:]
    imgs_a = [torch.from_numpy(i).pin_memory() for i, _, _ in a]          # pinned CPU photos
    imgs_b = [torch.from_numpy(i).to(cuda_device) for i, _, _ in b]       # CUDA photos
    stream = torch.cuda.current_stream(cuda_device)
    torch.cuda._sleep(1_000_000_000)
    out_a = pipe.forward_batch(imgs_a, [m for _, m, _ in a], invert=[v for _, _, v in a], wait=False)
    busy = not stream.query()
    out_b = pipe.forward_batch(imgs_b, [torch.from_numpy(m) for _, m, _ in b], invert=[v for _, _, v in b], wait=False)
    pipe.wait()
    assert busy, "forward_batch(wait=False) waited for the stream"
    assert pipe.last_sizes == [O.resized_size(r[0].shape[1], r[0].shape[0], res) for r in reqs]
    for k, o in enumerate(out_a + out_b):
        assert np.array_equal(o.cpu().numpy(), want[k]), k


def test_pageable_photo_refused_without_wait(cuda_device):
    pipe = _pipe(256, cuda_device)
    img = torch.full((40, 50, 3), 7, dtype=torch.uint8)
    mask = torch.full((40, 50), 255, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="pinned"):
        pipe.forward_batch([img], [mask], wait=False)
    with pytest.raises(RuntimeError, match="pinned"):
        pipe.forward_batch([img.numpy()], [mask], wait=False)
    assert torch.equal(pipe.forward_batch([img], [mask])[0], img)       # all known: the photo itself


def test_mask_size_mismatch_is_value_error(cuda_device):
    pipe = _pipe(256, cuda_device)
    with pytest.raises(ValueError, match="mask resizes"):
        pipe(np.zeros((300, 700, 3), np.uint8), np.zeros((300, 600), np.uint8))


def test_non_array_photo_is_type_error(cuda_device):
    pipe = _pipe(256, cuda_device)
    img, mask = np.zeros((40, 50, 3), np.uint8), np.full((40, 50), 255, np.uint8)
    with pytest.raises(TypeError, match="DemoPipeline: request 1: photo and mask must be"):
        pipe.forward_batch([img, [[1, 2, 3]]], [mask, mask])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_photo_on_another_gpu_refused_before_any_work(cuda_device):
    pipe = _pipe(256, cuda_device)
    other = torch.device("cuda", 1)
    img = torch.zeros((40, 50, 3), dtype=torch.uint8, device=other)
    mask = torch.full((40, 50), 255, dtype=torch.uint8)
    torch.cuda.synchronize(other)
    mem0 = torch.cuda.memory_allocated(other)
    with pytest.raises(ValueError, match="DemoPipeline: request 0: photo on cuda:1, the pipeline runs on cuda:0"):
        pipe.forward_batch([img], [mask])
    torch.cuda.synchronize(other)
    assert torch.cuda.memory_allocated(other) == mem0
