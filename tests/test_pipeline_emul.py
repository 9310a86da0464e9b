"""CPU checks of the arbitrary-resolution crop pipeline (SURVEY.md 8(f) row f4, scripts/create_onnx_pipeline.py:121-264):

* the oracle (oracle/pipeline_oracle.py) against the vectors the reference's own MIGAN_Pipeline produced
  (tests/golden/pipeline.npz, written by tests/golden/make_golden_pipeline.py where a checkout of the reference exists);
* the kernel functors of mi-gan_b200/csrc/pipeline.cu, compiled for the host by the emulation build (test infrastructure),
  against the same vectors -- bit for bit: crop window, model input x, final image given the reference generator's y;
* the host crop arithmetic of the PRODUCT library (`migan_crop_box`, no GPU involved) on the 300 pinned random masks.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from oracle import pipeline_oracle as PO  # noqa: E402
from migan_b200 import _abi, ops  # noqa: E402
import build_emul  # noqa: E402
import make_golden_pipeline as MG  # noqa: E402  (case table + seeded inputs; its main() needs the reference and is not run here)

GOLD = MG.load_fixture()
PIPE_SYMBOLS = [s for s in _abi.SYMBOLS if s[0] in ("b200_pipeline_scratch_bytes", "b200_resize_nearest_u8", "b200_hole_flags",
                                                    "migan_crop_box", "b200_pipeline_preprocess", "b200_pipeline_postprocess")]


@pytest.fixture(scope="module")
def emul():
    return _abi.bind(ctypes.CDLL(build_emul.build()), PIPE_SYMBOLS)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def random_bbox_masks():
    """The masks of the `bbox_cases` table (seed 5), regenerated exactly as make_golden_pipeline.py drew them."""
    rng = np.random.RandomState(5)
    for t in range(300):
        H, W = int(rng.randint(8, 400)), int(rng.randint(8, 400))
        mask = np.full((H, W), 255, np.uint8)
        for _ in range(int(rng.randint(0, 3))):
            a, b = sorted(rng.randint(0, H, 2)); c, d = sorted(rng.randint(0, W, 2))
            mask[a:b + 1, c:d + 1] = rng.choice([0, 0, 128, 254])
        pad = int(rng.choice([0, 5, 16, 128]))
        yield t, mask, pad


def test_oracle_bbox_matches_reference_vectors():
    table = GOLD["bbox_cases"]
    for t, mask, pad in random_bbox_masks():
        H, W, p, x0, x1, y0, y1 = [int(v) for v in table[t]]
        assert (H, W, p) == (mask.shape[0], mask.shape[1], pad)
        assert PO.masked_bbox(mask, 64, pad) == (x0, x1, y0, y1), t


@pytest.mark.parametrize("case", MG.CASES, ids=[c[0] for c in MG.CASES])
def test_oracle_matches_reference_pipeline(case):
    tag, res, pad = case[0], case[1], case[2]
    image, mask = MG.case_inputs(case)
    y_ref = torch.from_numpy(GOLD["y_" + tag])
    taps = {}
    final = PO.forward(lambda x: y_ref, image.clone(), mask, res, pad, taps)      # the generator's output is the reference's
    assert taps["box"] == tuple(int(v) for v in GOLD["box_" + tag])
    assert torch.equal(MG.on_stored_rows(GOLD, "x", tag, taps["x"]), torch.from_numpy(GOLD["x_" + tag]))
    assert np.array_equal(MG.on_stored_rows(GOLD, "final", tag, final.numpy()), GOLD["final_" + tag])


def test_aa_weights_against_torch():
    """The weight table (oracle restatement of ATen's) reproduces the weights torch applies: impulse responses."""
    import torch.nn.functional as F
    for (L, O) in [(420, 256), (256, 420), (150, 64), (45, 64), (64, 210)]:
        eye = torch.eye(L).view(1, L, 1, L)
        wt = F.interpolate(eye, size=(1, O), mode="bilinear", align_corners=False, antialias=True)[0, :, 0, :].numpy()
        xmin, xsize, w = PO.aa_weights(L, O)
        mine = np.zeros((L, O), np.float32)
        for i in range(O):
            mine[xmin[i]:xmin[i] + xsize[i], i] = w[i, :xsize[i]]
        assert np.array_equal(wt, mine), (L, O)


def _run_emul_pipeline(lib, image, mask, res, pad, y):
    """The request through the C entry points (host pointers: the emulation library runs the kernel functors on the CPU)."""
    image = np.ascontiguousarray(image[0]); mask = np.ascontiguousarray(mask[0, 0])
    H, W = image.shape[1], image.shape[2]
    if mask.shape != (H, W):
        m2 = np.empty((H, W), np.uint8)
        assert lib.b200_resize_nearest_u8(_ptr(mask), mask.shape[0], mask.shape[1], _ptr(m2), H, W, None) == 0
        mask = m2
    flags = np.empty(W + H, np.uint8)
    assert lib.b200_hole_flags(_ptr(mask), H, W, _ptr(flags), None) == 0
    box = np.zeros(4, np.int32)
    assert lib.migan_crop_box(_ptr(flags), H, W, res, pad, _ptr(box)) == 0
    nbytes = lib.b200_pipeline_scratch_bytes(H, W, res)
    raw = np.empty(nbytes + 256, np.uint8)
    scratch = raw[(-raw.ctypes.data) % 256:][:nbytes]
    x = np.empty((1, 4, res, res), np.float32)
    assert lib.b200_pipeline_preprocess(_ptr(image), _ptr(mask), H, W, _ptr(box), res, _ptr(x), _ptr(scratch), nbytes, None) == 0
    k = np.ascontiguousarray(ops.feather_kernel().numpy())
    yy = np.ascontiguousarray(y)
    assert lib.b200_pipeline_postprocess(_ptr(yy), _ptr(image), _ptr(mask), H, W, _ptr(box), res, _ptr(k), _ptr(scratch), nbytes, None) == 0
    return tuple(int(v) for v in box), x, image[None]


@pytest.mark.parametrize("case", MG.CASES, ids=[c[0] for c in MG.CASES])
def test_kernels_match_reference_pipeline(emul, case):
    tag, res, pad = case[0], case[1], case[2]
    image, mask = MG.case_inputs(case)
    box, x, final = _run_emul_pipeline(emul, image.numpy().copy(), mask.numpy(), res, pad, GOLD["y_" + tag])
    assert box == tuple(int(v) for v in GOLD["box_" + tag])
    x, final = MG.on_stored_rows(GOLD, "x", tag, x), MG.on_stored_rows(GOLD, "final", tag, final)
    assert np.array_equal(x, GOLD["x_" + tag]), "model input differs on %d values" % int((x != GOLD["x_" + tag]).sum())
    want = GOLD["final_" + tag]
    assert np.array_equal(final, want), "final image differs on %d bytes (max %d)" % (
        int((final != want).sum()), int(np.abs(final.astype(int) - want.astype(int)).max()))


def test_kernels_match_oracle_on_random_requests(emul):
    """Shapes the fixtures do not hold: odd sizes, strong down / up scaling, holes at the borders; y is random."""
    rng = np.random.RandomState(77)
    g = torch.Generator().manual_seed(78)
    for t in range(6):
        res = int(rng.choice([32, 64]))
        H, W = int(rng.randint(20, 260)), int(rng.randint(20, 260))
        image = torch.from_numpy(rng.randint(0, 256, size=(1, 3, H, W), dtype=np.uint8))
        mask = torch.full((1, 1, H, W), 255, dtype=torch.uint8)
        a, b = sorted(rng.randint(0, H, 2)); c, d = sorted(rng.randint(0, W, 2))
        mask[:, :, a:b + 1, c:d + 1] = 0
        pad = int(rng.choice([0, 8, 40]))
        y = torch.randn(1, 3, res, res, generator=g)
        taps = {}
        want = PO.forward(lambda x: y, image.clone(), mask, res, pad, taps)
        box, x, final = _run_emul_pipeline(emul, image.numpy().copy(), mask.numpy(), res, pad, y.numpy())
        assert box == taps["box"], t
        assert np.array_equal(x, taps["x"].numpy()), t
        assert np.array_equal(final, want.numpy()), (t, int((final != want.numpy()).sum()))


def test_product_crop_box_is_host_arithmetic(emul):
    """The product's `migan_crop_box` is host code: same 300 pinned masks as the oracle."""
    lib = emul
    table = GOLD["bbox_cases"]
    for t, mask, pad in random_bbox_masks():
        H, W = mask.shape
        flags = np.concatenate([(mask < 255).any(axis=0), (mask < 255).any(axis=1)]).astype(np.uint8)
        box = np.zeros(4, np.int32)
        assert lib.migan_crop_box(_ptr(flags), H, W, 64, pad, _ptr(box)) == 0
        assert tuple(int(v) for v in box) == tuple(int(v) for v in table[t][3:]), t
