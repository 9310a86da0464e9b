"""uint8 request path (SURVEY.md 8(f) rank 1) on the H100: the pre/post-processing kernels are bit-exact against the
oracle restatement of scripts/demo.py:56-66 / :135-142; the fused host call equals kernel-by-kernel composition."""
import os

import numpy as np
import pytest
import torch

import migan_b200
from migan_b200 import ops, synthetic
from oracle import migan_oracle as O
from oracle import prepost_oracle as P

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def test_prepost_kernels_bit_exact(cuda_device):
    gold = np.load(os.path.join(GOLDEN, "prepost.npz"))
    img, mask, y = torch.from_numpy(gold["img"]), torch.from_numpy(gold["mask"]), torch.from_numpy(gold["y"])
    x = ops.preprocess_u8(img.to(cuda_device), mask.to(cuda_device)).cpu()
    assert torch.equal(x, torch.from_numpy(gold["x"]))
    out = ops.postprocess_u8(y.to(cuda_device), img.to(cuda_device), mask.to(cuda_device)).cpu()
    assert torch.equal(out, torch.from_numpy(gold["out"]))
    rng = np.random.RandomState(0)
    img = torch.from_numpy(rng.randint(0, 256, size=(3, 128, 128, 3), dtype=np.uint8))
    mask = torch.from_numpy(rng.choice(np.array([0, 1, 128, 254, 255], np.uint8), size=(3, 128, 128)))
    x = ops.preprocess_u8(img.to(cuda_device), mask.to(cuda_device)).cpu()
    assert torch.equal(x, P.preprocess(img.numpy(), mask.numpy()))
    y = torch.linspace(-1.2, 1.2, 3 * 3 * 128 * 128).reshape(3, 3, 128, 128).contiguous()
    out = ops.postprocess_u8(y.to(cuda_device), img.to(cuda_device), mask.to(cuda_device)).cpu()
    assert np.array_equal(out.numpy(), P.postprocess(y, img.numpy(), mask.numpy()))


@pytest.mark.parametrize("R,N", [(64, 3), (256, 2)])
def test_forward_u8_equals_composition(cuda_device, R, N):
    model = migan_b200.Generator(R)
    sd = O.make_state_dict(R, seed=1)
    model.load_state_dict(sd)
    model = model.to(cuda_device).eval()
    rng = np.random.RandomState(R)
    img = torch.from_numpy(rng.randint(0, 256, size=(N, R, R, 3), dtype=np.uint8))
    mask = torch.from_numpy(((rng.rand(N, R, R) > 0.4) * 255).astype(np.uint8))
    out = model.forward_u8(img.pin_memory(), mask.pin_memory())
    assert out.shape == (N, R, R, 3) and out.dtype == torch.uint8 and not out.is_cuda
    # (a) same kernels, called one by one on the device: identical
    x = ops.preprocess_u8(img.to(cuda_device), mask.to(cuda_device))
    step = ops.postprocess_u8(model(x), img.to(cuda_device), mask.to(cuda_device)).cpu()
    assert torch.equal(out, step)
    # (b) against the CPU oracle chain: the generator output differs by ~1e-5, so a value sitting on a uint8 boundary may
    # truncate to the neighbouring level; known pixels are copied and must be identical.
    y_or = O.generator_forward(sd, P.preprocess(img.numpy(), mask.numpy()), R)
    want = torch.from_numpy(P.postprocess(y_or, img.numpy(), mask.numpy()))
    diff = (out.int() - want.int()).abs()
    assert int(diff.max()) <= 1 and float((diff > 0).float().mean()) < 1e-3
    known = (mask == 255)
    assert torch.equal(out[known], img[known])
    with pytest.raises(RuntimeError):
        model.forward_u8(img.float(), mask)


def test_forward_u8_async_serving_loop(cuda_device):
    """Back-to-back uint8 requests alternate staging slots (copies of request t+1 / t-1 under the kernels of t); every output
    must be complete after host_wait() and equal to the synchronous call."""
    R, N = 128, 4
    model = migan_b200.Generator(R)
    model.load_state_dict(O.make_state_dict(R, seed=2))
    model = model.to(cuda_device).eval()
    rng = np.random.RandomState(11)
    imgs = [torch.from_numpy(rng.randint(0, 256, size=(N, R, R, 3), dtype=np.uint8)).pin_memory() for _ in range(5)]
    masks = [torch.from_numpy(((rng.rand(N, R, R) > 0.5) * 255).astype(np.uint8)).pin_memory() for _ in range(5)]
    outs = [torch.empty(N, R, R, 3, dtype=torch.uint8).pin_memory() for _ in range(5)]
    for i, m, o in zip(imgs, masks, outs):
        model.forward_u8(i, m, out=o, wait=False)
    model.host_wait()
    for i, m, o in zip(imgs, masks, outs):
        assert torch.equal(o, model.forward_u8(i, m))


def test_feather_composite_reference_pipeline(cuda_device):
    """ops.feather_composite == the blend of the deployed pipeline (create_onnx_pipeline.py:233-245): vectors produced by the
    reference's own MIGAN_Pipeline.postprocess (tests/golden/feather.npz) and the oracle on a 512 x 512 free-form-mask case."""
    gold = np.load(os.path.join(GOLDEN, "feather.npz"))
    for tag in ("a", "b"):
        image, mask, y = (torch.from_numpy(gold[n + "_" + tag]) for n in ("image", "mask", "y"))
        out = ops.feather_composite(y.to(cuda_device), image.to(cuda_device), mask.to(cuda_device)).cpu()
        diff = (out.int() - torch.from_numpy(gold["out_" + tag]).int()).abs()
        assert int(diff.max()) <= 1 and float((diff > 0).float().mean()) < 1e-3
    rng = np.random.RandomState(9)
    R = 512
    image = torch.from_numpy(rng.randint(0, 256, size=(2, 3, R, R), dtype=np.uint8))
    mask = torch.from_numpy(np.stack([synthetic.free_form_mask(R, rng) for _ in range(2)])[:, None].astype(np.uint8) * 255)
    y = torch.from_numpy((rng.randn(2, 3, R, R) * 0.7).astype(np.float32))
    out = ops.feather_composite(y.to(cuda_device), image.to(cuda_device), mask.to(cuda_device)).cpu()
    want = P.feather_composite(image, mask, y)
    diff = (out.int() - want.int()).abs()
    assert int(diff.max()) <= 1 and float((diff > 0).float().mean()) < 1e-3
    far = torch.nn.functional.avg_pool2d((mask == 255).float(), 9, stride=1, padding=4) == 1.0     # 4 pixels away from any hole
    assert torch.equal(out[far.expand_as(out)], image[far.expand_as(image)])
