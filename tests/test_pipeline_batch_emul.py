"""CPU checks of the batched crop-pipeline entry points (b200_hole_flags_batch, b200_pipeline_batch_scratch_bytes,
b200_pipeline_preprocess_batch, b200_pipeline_postprocess_batch) in the emulation build of mi-gan_b200/csrc/pipeline.cu:
many requests of different sizes in ONE call of each stage, bit-exact with the reference vectors and with the oracle run
request by request, and the argument checks."""
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
import make_golden_pipeline as MG  # noqa: E402  (case table + seeded inputs only)

GOLD = MG.load_fixture()
NAMES = ("b200_resize_nearest_u8", "migan_crop_box", "b200_hole_flags_batch", "b200_pipeline_batch_scratch_bytes",
         "b200_pipeline_preprocess_batch", "b200_pipeline_postprocess_batch")
BATCH_SYMBOLS = [s for s in _abi.SYMBOLS if s[0] in NAMES]


@pytest.fixture(scope="module")
def emul():
    return _abi.bind(ctypes.CDLL(build_emul.build()), BATCH_SYMBOLS)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _requests(images, masks):
    reqs = (_abi.PipeRequest * len(images))()
    for r, image, mask in zip(reqs, images, masks):
        r.image, r.mask, r.H, r.W = image.ctypes.data, mask.ctypes.data, image.shape[1], image.shape[2]
    return reqs


def _scratch(nbytes):
    raw = np.empty(nbytes + 256, np.uint8)
    return raw[(-raw.ctypes.data) % 256:][:nbytes]


def run_batch(lib, images, masks, res, pad, y):
    """images [3,H,W] uint8 (updated in place), masks [h,w] uint8 at any size, y [n,3,res,res]: the whole batch through one
    call of each batched stage.  Returns (boxes, x)."""
    n = len(images)
    masks = list(masks)
    for i, (image, mask) in enumerate(zip(images, masks)):
        H, W = image.shape[1], image.shape[2]
        if mask.shape != (H, W):
            m2 = np.empty((H, W), np.uint8)
            assert lib.b200_resize_nearest_u8(_ptr(mask), mask.shape[0], mask.shape[1], _ptr(m2), H, W, None) == 0
            masks[i] = m2
    reqs = _requests(images, masks)
    flags = np.empty(sum(r.W + r.H for r in reqs), np.uint8)
    assert lib.b200_hole_flags_batch(reqs, n, _ptr(flags), None) == 0
    off = 0
    for r, mask in zip(reqs, masks):
        want = np.concatenate([(mask < 255).any(axis=0), (mask < 255).any(axis=1)]).astype(np.uint8)
        assert np.array_equal(flags[off:off + r.W + r.H], want)
        assert lib.migan_crop_box(flags.ctypes.data + off, r.H, r.W, res, pad, ctypes.addressof(r.box)) == 0
        off += r.W + r.H
    nbytes = lib.b200_pipeline_batch_scratch_bytes(reqs, n, res)
    assert nbytes > 0
    scratch = _scratch(nbytes)
    x = np.empty((n, 4, res, res), np.float32)
    assert lib.b200_pipeline_preprocess_batch(reqs, n, res, _ptr(x), _ptr(scratch), nbytes, None) == 0
    k = np.ascontiguousarray(ops.feather_kernel().numpy())
    yy = np.ascontiguousarray(y, dtype=np.float32)
    assert lib.b200_pipeline_postprocess_batch(_ptr(yy), reqs, n, res, _ptr(k), _ptr(scratch), nbytes, None) == 0
    return [tuple(int(v) for v in r.box) for r in reqs], x


def test_reference_cases_in_one_batch(emul):
    """The six resolution-64 reference requests (one with its mask at half size) in one call of each stage."""
    cases = [c for c in MG.CASES if c[1] == 64]
    assert len(cases) == 6 and len({c[2] for c in cases}) == 1
    inputs = [MG.case_inputs(c) for c in cases]
    images = [np.ascontiguousarray(im.numpy()[0]) for im, _ in inputs]
    masks = [np.ascontiguousarray(m.numpy()[0, 0]) for _, m in inputs]
    y = np.concatenate([GOLD["y_" + c[0]] for c in cases])
    boxes, x = run_batch(emul, images, masks, 64, cases[0][2], y)
    for i, c in enumerate(cases):
        tag = c[0]
        assert boxes[i] == tuple(int(v) for v in GOLD["box_" + tag]), tag
        assert np.array_equal(MG.on_stored_rows(GOLD, "x", tag, x[i:i + 1]), GOLD["x_" + tag]), tag
        assert np.array_equal(MG.on_stored_rows(GOLD, "final", tag, images[i][None]), GOLD["final_" + tag]), tag


def _random_request(rng, kind):
    if kind == "tiny":
        H, W = int(rng.randint(3, 12)), int(rng.randint(3, 12))          # strong up-scaling
    elif kind == "large":
        H, W = int(rng.randint(200, 420)), int(rng.randint(200, 420))    # strong down-scaling
    else:
        H, W = int(rng.randint(13, 200)), int(rng.randint(13, 200))
    image = rng.randint(0, 256, size=(1, 3, H, W), dtype=np.uint8)
    mh, mw = (H, W) if rng.rand() < 0.7 else (int(rng.randint(3, 2 * H)), int(rng.randint(3, 2 * W)))
    mask = np.full((1, 1, mh, mw), 255, np.uint8)
    hole = rng.randint(0, 4)
    if hole == 1:                                                       # at a border
        a = int(rng.randint(0, mh)); c = int(rng.randint(0, mw))
        mask[:, :, a:, :c + 1] = 0
    elif hole >= 2:
        a, b = sorted(rng.randint(0, mh, 2)); c, d = sorted(rng.randint(0, mw, 2))
        mask[:, :, a:b + 1, c:d + 1] = 0
    return image, mask


@pytest.mark.parametrize("n,res,pad", [(32, 32, 8), (7, 64, 0)])
def test_random_batch_matches_oracle(emul, n, res, pad):
    """Odd sizes, strong down / up scaling, masks at other sizes, holes at the borders and no hole; y is random."""
    rng = np.random.RandomState(1000 + n)
    kinds = ["tiny", "large", "mid"]
    reqs = [_random_request(rng, kinds[i % 3]) for i in range(n)]
    y = torch.randn(n, 3, res, res, generator=torch.Generator().manual_seed(n))
    images = [np.ascontiguousarray(im[0]).copy() for im, _ in reqs]
    boxes, x = run_batch(emul, images, [np.ascontiguousarray(m[0, 0]) for _, m in reqs], res, pad, y.numpy())
    for i, (image, mask) in enumerate(reqs):
        taps = {}
        want = PO.forward(lambda _x: y[i:i + 1], torch.from_numpy(image.copy()), torch.from_numpy(mask), res, pad, taps)
        assert boxes[i] == taps["box"], i
        assert np.array_equal(x[i:i + 1], taps["x"].numpy()), i
        assert np.array_equal(images[i][None], want.numpy()), (i, int((images[i][None] != want.numpy()).sum()))


def test_batch_argument_checks(emul):
    rng = np.random.RandomState(3)
    images = [rng.randint(0, 256, size=(3, 40, 50), dtype=np.uint8) for _ in range(33)]
    masks = [np.full((40, 50), 255, np.uint8) for _ in range(33)]
    reqs = _requests(images, masks)
    for r in reqs:
        r.box[:] = [0, 50, 0, 40]
    flags = np.empty(33 * 90, np.uint8)
    x = np.empty((33, 4, 16, 16), np.float32)
    y = np.zeros((33, 3, 16, 16), np.float32)
    k = np.ascontiguousarray(ops.feather_kernel().numpy())
    for n in (0, 33):
        assert emul.b200_hole_flags_batch(reqs, n, _ptr(flags), None) == _abi.ERR_INVALID
        assert emul.b200_pipeline_batch_scratch_bytes(reqs, n, 16) == 0
        assert emul.b200_pipeline_preprocess_batch(reqs, n, 16, _ptr(x), _ptr(flags), flags.nbytes, None) == _abi.ERR_INVALID
        assert emul.b200_pipeline_postprocess_batch(_ptr(y), reqs, n, 16, _ptr(k), _ptr(flags), flags.nbytes, None) == _abi.ERR_INVALID
    need = emul.b200_pipeline_batch_scratch_bytes(reqs, 32, 16)
    assert need > 0
    scratch = _scratch(need)
    assert emul.b200_pipeline_preprocess_batch(reqs, 32, 16, _ptr(x), _ptr(scratch), need - 1, None) == _abi.ERR_WORKSPACE
    assert emul.b200_pipeline_postprocess_batch(_ptr(y), reqs, 32, 16, _ptr(k), _ptr(scratch), need - 1, None) == _abi.ERR_WORKSPACE
    reqs[5].box[:] = [0, 51, 0, 40]                                     # outside the image
    assert emul.b200_pipeline_preprocess_batch(reqs, 32, 16, _ptr(x), _ptr(scratch), need, None) == _abi.ERR_INVALID
    reqs[5].box[:] = [0, 50, 0, 40]
    reqs[7].H = 2                                                       # too small for the feathering
    assert emul.b200_hole_flags_batch(reqs, 32, _ptr(flags), None) == _abi.ERR_INVALID
