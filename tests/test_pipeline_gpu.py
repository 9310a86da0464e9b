"""Arbitrary-resolution crop pipeline (SURVEY.md 8(f) row f4, scripts/create_onnx_pipeline.py:121-264) on the H100, through
`migan_b200.pipeline.MIGAN_Pipeline` and the C ABI underneath it, against the vectors the reference's own MIGAN_Pipeline
produced (tests/golden/pipeline.npz) and against the oracle on shapes the fixtures do not hold.

Bar: with the generator's output given (the reference's y from the fixture) every stage is BIT-EXACT -- crop window, model
input x, final uint8 image.  End to end (generator on the GPU, whose output differs from the CPU reference by ~5e-5) the
blended pixels may land on the neighbouring uint8 level: <= 1 level, on < 2 % of the crop; everything outside is untouched."""
import os
import sys

import numpy as np
import pytest
import torch

import migan_b200
from migan_b200 import synthetic
from migan_b200.pipeline import MIGAN_Pipeline
from oracle import pipeline_oracle as PO

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import make_golden_pipeline as MG  # noqa: E402  (case table + seeded inputs only; main() needs the reference)

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


@pytest.mark.parametrize("case", MG.CASES, ids=[c[0] for c in MG.CASES])
def test_stages_bit_exact_with_reference_vectors(cuda_device, case):
    tag, res, pad = case[0], case[1], case[2]
    image, mask = MG.case_inputs(case)
    pipe = _pipe(res, pad, cuda_device)
    real = pipe.model
    try:
        pipe.model = GivenOutput(torch.from_numpy(GOLD["y_" + tag]).to(cuda_device))
        img_d = image.to(cuda_device)
        out = pipe(img_d, mask.to(cuda_device))
        assert out.data_ptr() == img_d.data_ptr()                       # in place, like the reference
        assert pipe.last_box == tuple(int(v) for v in GOLD["box_" + tag])
        assert torch.equal(MG.on_stored_rows(GOLD, "x", tag, pipe.model.x.cpu()), torch.from_numpy(GOLD["x_" + tag]))
        assert np.array_equal(MG.on_stored_rows(GOLD, "final", tag, out.cpu().numpy()), GOLD["final_" + tag])
    finally:
        pipe.model = real


@pytest.mark.parametrize("case", MG.CASES, ids=[c[0] for c in MG.CASES])
def test_end_to_end_against_reference_vectors(cuda_device, case):
    tag, res, pad = case[0], case[1], case[2]
    image, mask = MG.case_inputs(case)
    pipe = _pipe(res, pad, cuda_device)
    before = image.clone()
    out = pipe(image, mask)                                             # CPU tensors in: copied to the device and back, in place
    assert out is image and not out.is_cuda
    want = torch.from_numpy(GOLD["final_" + tag])
    x0, x1, y0, y1 = [int(v) for v in GOLD["box_" + tag]]
    outside = torch.ones_like(image, dtype=torch.bool)
    outside[:, :, y0:y1, x0:x1] = False
    assert torch.equal(out[outside], before[outside])
    inside = ~MG.on_stored_rows(GOLD, "final", tag, outside)
    diff = (MG.on_stored_rows(GOLD, "final", tag, out).int() - want.int()).abs()
    assert int(diff.max()) <= 1, int(diff.max())
    assert float((diff[inside] > 0).float().mean()) < 0.02


def test_random_requests_against_oracle(cuda_device):
    """Larger and odder shapes than the fixtures, generator output given (bit-exact bar)."""
    rng = np.random.RandomState(123)
    g = torch.Generator().manual_seed(124)
    pipe = _pipe(64, 16, cuda_device)
    real = pipe.model
    try:
        for t, (H, W) in enumerate([(257, 255), (720, 1280), (64, 64), (65, 1000), (1100, 90), (333, 777)]):
            image = torch.from_numpy(rng.randint(0, 256, size=(1, 3, H, W), dtype=np.uint8))
            mask = torch.full((1, 1, H, W), 255, dtype=torch.uint8)
            a, b = sorted(rng.randint(0, H, 2)); c, d = sorted(rng.randint(0, W, 2))
            mask[:, :, a:b + 1, c:d + 1] = 0
            pipe.padding = int(rng.choice([0, 16, 128]))
            y = torch.randn(1, 3, 64, 64, generator=g)
            taps = {}
            want = PO.forward(lambda x: y, image.clone(), mask, 64, pipe.padding, taps)
            pipe.model = GivenOutput(y.to(cuda_device))
            out = pipe(image.to(cuda_device), mask.to(cuda_device)).cpu()
            assert pipe.last_box == taps["box"], t
            assert torch.equal(pipe.model.x.cpu(), taps["x"]), t
            assert torch.equal(out, want), (t, int((out != want).sum()))
    finally:
        pipe.model = real


def test_batch_and_argument_checks(cuda_device):
    pipe = _pipe(64, 16, cuda_device)
    rng = np.random.RandomState(9)
    image = torch.from_numpy(rng.randint(0, 256, size=(2, 3, 100, 120), dtype=np.uint8))
    mask = torch.full((2, 1, 100, 120), 255, dtype=torch.uint8)
    mask[0, :, 10:30, 20:60] = 0
    mask[1, :, 70:95, 5:40] = 0
    both = pipe(image.clone().to(cuda_device), mask.to(cuda_device)).cpu()
    for i in range(2):                                                  # N > 1 = the requests one after the other
        one = pipe(image[i:i + 1].clone().to(cuda_device), mask[i:i + 1].to(cuda_device)).cpu()
        assert torch.equal(both[i:i + 1], one)
    with pytest.raises(RuntimeError):
        pipe(image.float(), mask)
    with pytest.raises(RuntimeError):
        pipe(image[:, :2], mask)
    with pytest.raises(RuntimeError):
        MIGAN_Pipeline(synthetic.export_style_state_dict(64, seed=11), 64, device="cpu")
