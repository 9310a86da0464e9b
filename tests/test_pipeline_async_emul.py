"""CPU checks of the device-planned crop-pipeline entry points (b200_pipeline_batch_scratch_bound, b200_pipeline_plan_batch,
b200_pipeline_preprocess_planned, b200_pipeline_postprocess_planned) in the emulation build of mi-gan_b200/csrc/pipeline.cu:
the planned crop windows equal `migan_crop_box` on pinned random masks and edge cases, the scratch bound holds every window
an image allows, and a planned pass is bit-exact with the reference vectors and with the host-box batched calls."""
import ctypes
import itertools
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from migan_b200 import _abi, ops  # noqa: E402
import build_emul  # noqa: E402
import make_golden_pipeline as MG  # noqa: E402  (case table + seeded inputs only)
from test_pipeline_batch_emul import _random_request, run_batch  # noqa: E402
from test_pipeline_emul import random_bbox_masks  # noqa: E402

GOLD = MG.load_fixture()
NAMES = ("b200_resize_nearest_u8", "migan_crop_box", "b200_hole_flags_batch", "b200_pipeline_batch_scratch_bytes",
         "b200_pipeline_preprocess_batch", "b200_pipeline_postprocess_batch", "b200_pipeline_batch_scratch_bound",
         "b200_pipeline_plan_batch", "b200_pipeline_preprocess_planned", "b200_pipeline_postprocess_planned")
SYMBOLS = [s for s in _abi.SYMBOLS if s[0] in NAMES]
SIZE6 = ctypes.c_size_t * 6


@pytest.fixture(scope="module")
def emul():
    lib = _abi.bind(ctypes.CDLL(build_emul.build()), SYMBOLS)
    lib.migan_emul_planned_regions.restype = None
    lib.migan_emul_planned_regions.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                               ctypes.c_void_p]
    return lib


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


def _host_boxes(lib, masks, res, pad):
    out = []
    for m in masks:
        H, W = m.shape
        flags = np.ascontiguousarray(np.concatenate([(m < 255).any(axis=0), (m < 255).any(axis=1)]).astype(np.uint8))
        box = np.zeros(4, np.int32)
        assert lib.migan_crop_box(_ptr(flags), H, W, res, pad, _ptr(box)) == 0
        out.append(tuple(int(v) for v in box))
    return out


def plan(lib, images, masks, res, pad):
    """Flags and planning step of one pass (masks already at the image sizes).  Returns (reqs, boxes [n,4], scratch)."""
    n = len(images)
    reqs = _requests(images, masks)
    for r in reqs:
        r.box[:] = [-7, -7, -7, -7]                                     # not read
    flags = np.empty(sum(r.W + r.H for r in reqs), np.uint8)
    assert lib.b200_hole_flags_batch(reqs, n, _ptr(flags), None) == 0
    nbytes = lib.b200_pipeline_batch_scratch_bound(reqs, n, res)
    assert nbytes > 0
    scratch = _scratch(nbytes)
    boxes = np.full((n, 4), -1, np.int32)
    assert lib.b200_pipeline_plan_batch(reqs, n, res, pad, _ptr(flags), _ptr(boxes), _ptr(scratch), nbytes, None) == 0
    for (x0, x1, y0, y1), image in zip(boxes, images):                  # inside the image, at least 3 x 3
        H, W = image.shape[1], image.shape[2]
        assert 0 <= x0 and x1 <= W and 0 <= y0 and y1 <= H and x1 - x0 >= 3 and y1 - y0 >= 3, (x0, x1, y0, y1, H, W)
    return reqs, boxes, scratch


def run_planned(lib, images, masks, res, pad, y):
    """The whole planned pass: images [3,H,W] uint8 updated in place, masks [H,W], y [n,3,res,res].  Returns (boxes, x)."""
    n = len(images)
    reqs, boxes, scratch = plan(lib, images, masks, res, pad)
    x = np.empty((n, 4, res, res), np.float32)
    assert lib.b200_pipeline_preprocess_planned(reqs, n, res, _ptr(x), _ptr(scratch), scratch.nbytes, None) == 0
    k = np.ascontiguousarray(ops.feather_kernel().numpy())
    yy = np.ascontiguousarray(y, dtype=np.float32)
    assert lib.b200_pipeline_postprocess_planned(_ptr(yy), reqs, n, res, _ptr(k), _ptr(scratch), scratch.nbytes, None) == 0
    return [tuple(int(v) for v in b) for b in boxes], x


def test_planned_boxes_on_pinned_masks(emul):
    """The 300 masks of the `bbox_cases` table, planned 32 per call, against the stored boxes and migan_crop_box."""
    table = GOLD["bbox_cases"]
    cases = list(random_bbox_masks())
    pads = {}
    for t, mask, pad in cases:
        pads.setdefault(pad, []).append((t, mask))
    for pad, group in sorted(pads.items()):
        for c in range(0, len(group), 32):
            part = group[c:c + 32]
            masks = [np.ascontiguousarray(m) for _, m in part]
            images = [np.zeros((3,) + m.shape, np.uint8) for m in masks]
            _, boxes, _ = plan(emul, images, masks, 64, pad)
            want = _host_boxes(emul, masks, 64, pad)
            for (t, _), got, w in zip(part, boxes, want):
                assert tuple(int(v) for v in got) == w == tuple(int(v) for v in table[t][3:]), t


def _edge_masks():
    def holes(H, W, *rects):
        m = np.full((H, W), 255, np.uint8)
        for a, b, c, d in rects:
            m[a:b, c:d] = 0
        return m
    return [
        np.full((40, 50), 255, np.uint8), np.zeros((40, 50), np.uint8),           # all known, all hole
        holes(40, 50, (0, 1, 10, 20)), holes(40, 50, (39, 40, 10, 20)),           # top / bottom row
        holes(40, 50, (5, 9, 0, 1)), holes(40, 50, (5, 9, 49, 50)),               # left / right column
        holes(40, 50, (0, 40, 0, 1), (0, 1, 0, 50)), holes(33, 17, (32, 33, 16, 17)),
        np.full((3, 3), 255, np.uint8), np.zeros((3, 3), np.uint8), holes(3, 3, (1, 2, 1, 2)),
        holes(3, 200, (0, 3, 150, 151)), holes(3, 1001, (1, 2, 0, 1), (2, 3, 1000, 1001)),
        holes(2160, 3840, (700, 1300, 1000, 1900), (2159, 2160, 3839, 3840)),
    ]


@pytest.mark.parametrize("res,pad", [(64, 0), (64, 128), (3, 0), (512, 16)])
def test_planned_boxes_on_edge_cases(emul, res, pad):
    masks = [np.ascontiguousarray(m) for m in _edge_masks()]
    images = [np.zeros((3,) + m.shape, np.uint8) for m in masks]
    _, boxes, _ = plan(emul, images, masks, res, pad)
    assert [tuple(int(v) for v in b) for b in boxes] == _host_boxes(emul, masks, res, pad)


def _reachable_boxes(lib, H, W, res, pad):
    """Every window migan_crop_box returns for an H x W image: all column / row hole extents, and none."""
    xs = [None] + [(a, b) for a in range(W) for b in range(a, W)]
    ys = [None] + [(a, b) for a in range(H) for b in range(a, H)]
    flags = np.zeros(W + H, np.uint8)
    box = np.zeros(4, np.int32)
    out = set()
    for xe, ye in itertools.product(xs, ys):
        flags[:] = 0
        if xe:
            flags[xe[0]] = flags[xe[1]] = 1
        if ye:
            flags[W + ye[0]] = flags[W + ye[1]] = 1
        assert lib.migan_crop_box(_ptr(flags), H, W, res, pad, _ptr(box)) == 0
        out.add(tuple(int(v) for v in box))
    return out


@pytest.mark.parametrize("H,W,res", [(16, 16, 16), (12, 20, 16), (20, 12, 16), (17, 15, 16), (9, 30, 8), (5, 5, 8), (3, 13, 4),
                                     (3, 3, 3)])
def test_scratch_bound_holds_every_window(emul, H, W, res):
    """Sides at, just above and below the resolution, where the tap count of a table is not monotone in the crop size
    (1 tap when a side equals the resolution, 3 just below it, more above)."""
    image = np.zeros((3, H, W), np.uint8)
    mask = np.full((H, W), 255, np.uint8)
    reqs = _requests([image], [mask])
    bound = emul.b200_pipeline_batch_scratch_bound(reqs, 1, res)
    assert bound > 0
    have, need = SIZE6(), SIZE6()
    boxes = set()
    for pad in (0, 1, 3):
        boxes |= _reachable_boxes(emul, H, W, res, pad)
    for b in sorted(boxes):
        reqs[0].box[:] = list(b)
        exact = emul.b200_pipeline_batch_scratch_bytes(reqs, 1, res)
        assert 0 < exact <= bound, (b, exact, bound)
        emul.migan_emul_planned_regions(H, W, res, ctypes.cast(reqs[0].box, ctypes.c_void_p), have, need)
        for i in range(6):                                             # every table and width-pass buffer on its own
            assert need[i] <= have[i], (b, i, need[i], have[i])


def test_reference_cases_in_one_planned_pass(emul):
    """The six resolution-64 reference requests (one with its mask at half size) in one planned pass."""
    cases = [c for c in MG.CASES if c[1] == 64]
    assert len(cases) == 6 and len({c[2] for c in cases}) == 1
    inputs = [MG.case_inputs(c) for c in cases]
    images = [np.ascontiguousarray(im.numpy()[0]) for im, _ in inputs]
    masks = []
    for image, (_, m) in zip(images, inputs):
        m = np.ascontiguousarray(m.numpy()[0, 0])
        H, W = image.shape[1:]
        if m.shape != (H, W):
            m2 = np.empty((H, W), np.uint8)
            assert emul.b200_resize_nearest_u8(_ptr(m), m.shape[0], m.shape[1], _ptr(m2), H, W, None) == 0
            m = m2
        masks.append(m)
    y = np.concatenate([GOLD["y_" + c[0]] for c in cases])
    boxes, x = run_planned(emul, images, masks, 64, cases[0][2], y)
    for i, c in enumerate(cases):
        tag = c[0]
        assert boxes[i] == tuple(int(v) for v in GOLD["box_" + tag]), tag
        assert np.array_equal(MG.on_stored_rows(GOLD, "x", tag, x[i:i + 1]), GOLD["x_" + tag]), tag
        assert np.array_equal(MG.on_stored_rows(GOLD, "final", tag, images[i][None]), GOLD["final_" + tag]), tag


@pytest.mark.parametrize("n,res,pad", [(32, 32, 8), (7, 64, 0)])
def test_random_planned_batch_matches_host_boxes(emul, n, res, pad):
    """Mixed sizes, strong down / up scaling, holes at the borders and no hole: the planned pass against the host-box
    batched calls on copies of the same requests."""
    rng = np.random.RandomState(2000 + n)
    kinds = ["tiny", "large", "mid"]
    reqs = [_random_request(rng, kinds[i % 3]) for i in range(n)]
    y = torch.randn(n, 3, res, res, generator=torch.Generator().manual_seed(n)).numpy()
    masks = []
    for image, m in reqs:
        m = np.ascontiguousarray(m[0, 0])
        H, W = image.shape[2:]
        if m.shape != (H, W):
            m2 = np.empty((H, W), np.uint8)
            assert emul.b200_resize_nearest_u8(_ptr(m), m.shape[0], m.shape[1], _ptr(m2), H, W, None) == 0
            m = m2
        masks.append(m)
    host_images = [np.ascontiguousarray(im[0]).copy() for im, _ in reqs]
    want_boxes, want_x = run_batch(emul, host_images, masks, res, pad, y)
    images = [np.ascontiguousarray(im[0]).copy() for im, _ in reqs]
    boxes, x = run_planned(emul, images, masks, res, pad, y)
    assert boxes == want_boxes
    assert np.array_equal(x, want_x)
    for i in range(n):
        assert np.array_equal(images[i], host_images[i]), (i, int((images[i] != host_images[i]).sum()))


def test_planned_argument_checks(emul):
    rng = np.random.RandomState(4)
    images = [rng.randint(0, 256, size=(3, 40, 50), dtype=np.uint8) for _ in range(33)]
    masks = [np.full((40, 50), 255, np.uint8) for _ in range(33)]
    reqs = _requests(images, masks)
    flags = np.zeros(33 * 90, np.uint8)
    boxes = np.zeros((33, 4), np.int32)
    x = np.empty((33, 4, 16, 16), np.float32)
    y = np.zeros((33, 3, 16, 16), np.float32)
    k = np.ascontiguousarray(ops.feather_kernel().numpy())
    need = emul.b200_pipeline_batch_scratch_bound(reqs, 32, 16)
    assert need > 0
    scratch = _scratch(need)
    S = (_ptr(scratch), need, None)

    def calls(n, res=16, s=S):
        return [emul.b200_pipeline_plan_batch(reqs, n, res, 4, _ptr(flags), _ptr(boxes), *s),
                emul.b200_pipeline_preprocess_planned(reqs, n, res, _ptr(x), *s),
                emul.b200_pipeline_postprocess_planned(_ptr(y), reqs, n, res, _ptr(k), *s)]

    for n in (0, 33):
        assert emul.b200_pipeline_batch_scratch_bound(reqs, n, 16) == 0
        assert calls(n) == [_abi.ERR_INVALID] * 3
    assert calls(32, s=(_ptr(scratch), need - 1, None)) == [_abi.ERR_WORKSPACE] * 3
    assert emul.b200_pipeline_batch_scratch_bound(reqs, 32, 2) == 0               # a window must be at least 3 x 3
    assert calls(32, res=2) == [_abi.ERR_INVALID] * 3
    assert emul.b200_pipeline_batch_scratch_bound(None, 32, 16) == 0
    assert emul.b200_pipeline_plan_batch(None, 32, 16, 4, _ptr(flags), _ptr(boxes), *S) == _abi.ERR_INVALID
    assert emul.b200_pipeline_plan_batch(reqs, 32, 16, 4, None, _ptr(boxes), *S) == _abi.ERR_INVALID
    assert emul.b200_pipeline_plan_batch(reqs, 32, 16, 4, _ptr(flags), None, *S) == _abi.ERR_INVALID
    assert emul.b200_pipeline_plan_batch(reqs, 32, 16, -1, _ptr(flags), _ptr(boxes), *S) == _abi.ERR_INVALID
    assert emul.b200_pipeline_preprocess_planned(reqs, 32, 16, None, *S) == _abi.ERR_INVALID
    assert emul.b200_pipeline_postprocess_planned(None, reqs, 32, 16, _ptr(k), *S) == _abi.ERR_INVALID
    assert emul.b200_pipeline_postprocess_planned(_ptr(y), reqs, 32, 16, None, *S) == _abi.ERR_INVALID
    assert calls(32, s=(None, need, None)) == [_abi.ERR_INVALID] * 3
    reqs[7].H = 2                                                       # too small for the feathering
    assert calls(32) == [_abi.ERR_INVALID] * 3
    reqs[7].H = 40
    reqs[9].mask = None
    assert calls(32) == [_abi.ERR_INVALID] * 3
    reqs[9].mask = masks[9].ctypes.data
    assert calls(32) == [_abi.OK] * 3
