"""CPU checks of the crop pipeline on decoded photos (csrc/pipeline.cu, emulation build): the stages at MIGAN_LAYOUT_HWC
give the bytes of MIGAN_LAYOUT_CHW on the transposed photo and of the oracle and the stored reference vectors, host-
planned and device-planned; the CHW entry points are unchanged; and b200_pipeline_mask_planes is create_onnx_pipeline.py's
`read_mask` followed by the NEAREST resize to the photo's size."""
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

from migan_b200 import _abi, ops  # noqa: E402
from oracle import pipeline_oracle as PO  # noqa: E402
import build_emul  # noqa: E402
import make_golden_pipeline as MG  # noqa: E402  (case table + seeded inputs only)
from test_pipeline_batch_emul import _random_request, run_batch  # noqa: E402

GOLD = MG.load_fixture()
NAMES = ("b200_resize_nearest_u8", "migan_crop_box", "b200_hole_flags_batch", "b200_pipeline_batch_scratch_bytes",
         "b200_pipeline_preprocess_batch", "b200_pipeline_postprocess_batch", "b200_pipeline_batch_scratch_bound",
         "b200_pipeline_plan_batch", "b200_pipeline_preprocess_planned", "b200_pipeline_postprocess_planned",
         "b200_pipeline_mask_planes", "b200_pipeline_preprocess_batch_layout", "b200_pipeline_postprocess_batch_layout",
         "b200_pipeline_plan_batch_layout")


@pytest.fixture(scope="module")
def emul():
    return _abi.bind(ctypes.CDLL(build_emul.build()), [s for s in _abi.SYMBOLS if s[0] in NAMES])


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _scratch(nbytes):
    raw = np.empty(nbytes + 256, np.uint8)
    return raw[(-raw.ctypes.data) % 256:][:nbytes]


def _requests(images, masks, boxes=None):
    """images [3,H,W] or [H,W,3] (the sizes come from the masks, which are at the image size)."""
    reqs = (_abi.PipeRequest * len(images))()
    for i, (r, image, mask) in enumerate(zip(reqs, images, masks)):
        r.image, r.mask, r.H, r.W = image.ctypes.data, mask.ctypes.data, mask.shape[0], mask.shape[1]
        if boxes is not None:
            r.box[:] = list(boxes[i])
    return reqs


def _at_size(lib, masks, images_chw):
    out = []
    for m, im in zip(masks, images_chw):
        H, W = im.shape[1:]
        if m.shape != (H, W):
            m2 = np.empty((H, W), np.uint8)
            assert lib.b200_resize_nearest_u8(_ptr(m), m.shape[0], m.shape[1], _ptr(m2), H, W, None) == 0
            m = m2
        out.append(np.ascontiguousarray(m))
    return out


def run_layout(lib, images, masks, boxes, res, layout, y):
    """The host-box batched stages with an explicit layout; images updated in place.  Returns x."""
    n = len(images)
    reqs = _requests(images, masks, boxes)
    nbytes = lib.b200_pipeline_batch_scratch_bytes(reqs, n, res)
    scratch = _scratch(nbytes)
    x = np.empty((n, 4, res, res), np.float32)
    assert lib.b200_pipeline_preprocess_batch_layout(reqs, n, res, layout, _ptr(x), _ptr(scratch), nbytes, None) == 0
    k = np.ascontiguousarray(ops.feather_kernel().numpy())
    yy = np.ascontiguousarray(y, dtype=np.float32)
    assert lib.b200_pipeline_postprocess_batch_layout(_ptr(yy), reqs, n, res, layout, _ptr(k), _ptr(scratch), nbytes,
                                                      None) == 0
    return x


def run_planned_layout(lib, images, masks, res, pad, layout, y):
    """The device-planned pass with an explicit layout; images updated in place.  Returns (boxes, x)."""
    n = len(images)
    reqs = _requests(images, masks)
    flags = np.empty(sum(r.W + r.H for r in reqs), np.uint8)
    assert lib.b200_hole_flags_batch(reqs, n, _ptr(flags), None) == 0
    nbytes = lib.b200_pipeline_batch_scratch_bound(reqs, n, res)
    scratch = _scratch(nbytes)
    boxes = np.full((n, 4), -1, np.int32)
    assert lib.b200_pipeline_plan_batch_layout(reqs, n, res, pad, layout, _ptr(flags), _ptr(boxes), _ptr(scratch), nbytes,
                                               None) == 0
    x = np.empty((n, 4, res, res), np.float32)
    assert lib.b200_pipeline_preprocess_planned(reqs, n, res, _ptr(x), _ptr(scratch), nbytes, None) == 0
    k = np.ascontiguousarray(ops.feather_kernel().numpy())
    yy = np.ascontiguousarray(y, dtype=np.float32)
    assert lib.b200_pipeline_postprocess_planned(_ptr(yy), reqs, n, res, _ptr(k), _ptr(scratch), nbytes, None) == 0
    return [tuple(int(v) for v in b) for b in boxes], x


def _hwc(chw):
    return np.ascontiguousarray(chw.transpose(1, 2, 0))


def _reference_cases(lib):
    cases = [c for c in MG.CASES if c[1] == 64]
    inputs = [MG.case_inputs(c) for c in cases]
    images = [np.ascontiguousarray(im.numpy()[0]) for im, _ in inputs]
    masks = _at_size(lib, [np.ascontiguousarray(m.numpy()[0, 0]) for _, m in inputs], images)
    y = np.concatenate([GOLD["y_" + c[0]] for c in cases])
    return cases, images, masks, y


@pytest.mark.parametrize("planned", [False, True])
def test_hwc_reproduces_the_reference_vectors(emul, planned):
    """The six resolution-64 reference requests as [H,W,3] photos, in one pass, against the stored x and final image."""
    cases, images, masks, y = _reference_cases(emul)
    photos = [_hwc(im) for im in images]
    boxes = [tuple(int(v) for v in GOLD["box_" + c[0]]) for c in cases]
    if planned:
        got_boxes, x = run_planned_layout(emul, photos, masks, 64, cases[0][2], _abi.LAYOUT_HWC, y)
        assert got_boxes == boxes
    else:
        x = run_layout(emul, photos, masks, boxes, 64, _abi.LAYOUT_HWC, y)
    for i, c in enumerate(cases):
        tag = c[0]
        assert np.array_equal(MG.on_stored_rows(GOLD, "x", tag, x[i:i + 1]), GOLD["x_" + tag]), tag
        final = np.ascontiguousarray(photos[i].transpose(2, 0, 1))[None]
        assert np.array_equal(MG.on_stored_rows(GOLD, "final", tag, final), GOLD["final_" + tag]), tag


@pytest.mark.parametrize("n,res,pad", [(32, 32, 8), (7, 64, 0)])
def test_hwc_equals_chw_on_the_transposed_photo(emul, n, res, pad):
    """The random batches of test_pipeline_batch_emul (odd sizes, strong down / up scaling, holes at the borders): HWC
    against CHW (host-planned and planned) and against the oracle."""
    rng = np.random.RandomState(1000 + n)
    kinds = ["tiny", "large", "mid"]
    reqs = [_random_request(rng, kinds[i % 3]) for i in range(n)]
    y = torch.randn(n, 3, res, res, generator=torch.Generator().manual_seed(n))
    chw = [np.ascontiguousarray(im[0]).copy() for im, _ in reqs]
    masks = _at_size(emul, [np.ascontiguousarray(m[0, 0]) for _, m in reqs], chw)
    photos = [_hwc(im) for im in chw]
    boxes, x_chw = run_batch(emul, chw, masks, res, pad, y.numpy())        # the CHW entry points, as before
    x_hwc = run_layout(emul, photos, masks, boxes, res, _abi.LAYOUT_HWC, y.numpy())
    assert np.array_equal(x_hwc, x_chw)
    planned = [_hwc(np.ascontiguousarray(im[0])) for im, _ in reqs]
    pboxes, px = run_planned_layout(emul, planned, masks, res, pad, _abi.LAYOUT_HWC, y.numpy())
    assert pboxes == boxes and np.array_equal(px, x_chw)
    for i, (image, mask) in enumerate(reqs):
        want = PO.forward(lambda _x: y[i:i + 1], torch.from_numpy(image.copy()), torch.from_numpy(mask), res, pad)
        want_hwc = want.numpy()[0].transpose(1, 2, 0)
        assert np.array_equal(chw[i], want.numpy()[0]), i
        assert np.array_equal(photos[i], want_hwc), i
        assert np.array_equal(planned[i], want_hwc), i


def test_chw_entry_points_are_unchanged(emul):
    """The old entry points, the *_layout forms at CHW and the planned pass at CHW: the same bytes."""
    cases, images, masks, y = _reference_cases(emul)
    boxes = [tuple(int(v) for v in GOLD["box_" + c[0]]) for c in cases]
    a = [im.copy() for im in images]
    b = [im.copy() for im in images]
    c = [im.copy() for im in images]
    _, xa = run_batch(emul, a, masks, 64, cases[0][2], y)
    xb = run_layout(emul, b, masks, boxes, 64, _abi.LAYOUT_CHW, y)
    cb, xc = run_planned_layout(emul, c, masks, 64, cases[0][2], _abi.LAYOUT_CHW, y)
    assert cb == boxes
    assert np.array_equal(xa, xb) and np.array_equal(xa, xc)
    for i in range(len(cases)):
        assert np.array_equal(a[i], b[i]) and np.array_equal(a[i], c[i])
        assert np.array_equal(MG.on_stored_rows(GOLD, "final", cases[i][0], a[i][None]), GOLD["final_" + cases[i][0]])


def test_layout_is_checked(emul):
    cases, images, masks, y = _reference_cases(emul)
    reqs = _requests(images[:1], masks[:1], [tuple(int(v) for v in GOLD["box_" + cases[0][0]])])
    x = np.empty((1, 4, 64, 64), np.float32)
    s = _scratch(1 << 20)
    assert emul.b200_pipeline_preprocess_batch_layout(reqs, 1, 64, 2, _ptr(x), _ptr(s), s.nbytes, None) == _abi.ERR_INVALID
    flags = np.zeros(1024, np.uint8)
    boxes = np.zeros((1, 4), np.int32)
    assert emul.b200_pipeline_plan_batch_layout(reqs, 1, 64, 0, -1, _ptr(flags), _ptr(boxes), _ptr(s), s.nbytes,
                                                None) == _abi.ERR_INVALID


# -- raw masks --------------------------------------------------------------------------------------------------------

def read_mask_np(mask: np.ndarray, invert: bool) -> np.ndarray:
    """create_onnx_pipeline.py:27-45 on a decoded mask array, as the single plane `.convert("L")` gives."""
    if mask.ndim == 3:
        if mask.shape[2] == 4:
            v = mask[:, :, 3]
        elif mask.shape[2] == 2:
            v = mask[:, :, 1]
        elif mask.shape[2] == 3:
            v = mask[:, :, 0]
        else:
            v = mask[:, :, 0]
    else:
        v = mask
    v = np.dstack([v, v, v])
    if invert:
        v = 255 - v
    v[v < 255] = 0
    from PIL import Image
    return np.array(Image.fromarray(v).convert("L"))


def _raw_table(masks, invs, outs):
    t = (_abi.RawMask * len(masks))()
    for r, m, inv, o in zip(t, masks, invs, outs):
        r.mask, r.hm, r.wm, r.channels = m.ctypes.data, m.shape[0], m.shape[1], m.shape[2]
        r.invert, r.out, r.H, r.W = int(inv), o.ctypes.data, o.shape[0], o.shape[1]
    return t


@pytest.mark.parametrize("channels", [1, 2, 3, 4])
@pytest.mark.parametrize("invert", [False, True])
def test_mask_planes_match_read_mask_and_nearest(emul, channels, invert):
    """Masks above, below and at the photo's size (and of other aspect), with values 0, 255 and in between, in one
    launch; against numpy read_mask + tvF.resize(NEAREST) (the oracle's resize)."""
    rng = np.random.RandomState(channels * 10 + invert)
    sizes = [((40, 50), (40, 50)), ((80, 100), (40, 50)), ((20, 25), (40, 50)), ((7, 300), (33, 17)), ((1, 1), (5, 9)),
             ((3, 3), (3, 3)), ((500, 3), (9, 400))]
    masks, outs = [], []
    for (hm, wm), (H, W) in sizes:
        m = rng.choice(np.array([0, 1, 128, 254, 255], np.uint8), size=(hm, wm, channels), p=[.3, .05, .1, .05, .5])
        masks.append(np.ascontiguousarray(m))
        outs.append(np.full((H, W), 77, np.uint8))
    t = _raw_table(masks, [invert] * len(masks), outs)
    assert emul.b200_pipeline_mask_planes(t, len(masks), None) == 0
    for m, o in zip(masks, outs):
        plane = read_mask_np(m if channels > 1 else m[:, :, 0], invert)
        want = PO.resize_nearest(torch.from_numpy(plane)[None, None], o.shape[0], o.shape[1]).numpy()[0, 0]
        assert np.array_equal(o, want), (m.shape, o.shape)


def test_mask_planes_per_request_invert_and_checks(emul):
    m = np.ascontiguousarray(np.array([[[0], [255]], [[255], [0]]], np.uint8))
    outs = [np.empty((2, 2), np.uint8), np.empty((2, 2), np.uint8)]
    t = _raw_table([m, m], [False, True], outs)
    assert emul.b200_pipeline_mask_planes(t, 2, None) == 0
    assert outs[0].tolist() == [[0, 255], [255, 0]] and outs[1].tolist() == [[255, 0], [0, 255]]
    bad = _raw_table([m], [False], outs[:1])
    bad[0].channels = 5
    assert emul.b200_pipeline_mask_planes(bad, 1, None) == _abi.ERR_INVALID
    bad = _raw_table([m], [False], outs[:1])
    bad[0].H = 0
    assert emul.b200_pipeline_mask_planes(bad, 1, None) == _abi.ERR_INVALID
    assert emul.b200_pipeline_mask_planes(t, 0, None) == _abi.ERR_INVALID


# -- the known rounding difference of the crop resize ----------------------------------------------------------------

def test_known_resize_rounding_difference(emul):
    """The crop's anti-aliased resize rounds like torch's CPU `tvF.resize` except at rare values next to a half: on the
    seeded photos of test_crop_pipeline_gpu's Co-Mod-GAN check, x equals the oracle's for the first six, and the seventh
    (569 x 405, 3-channel mask) differs at one element, x[0, 1, 200, 216], where the kernel rounds the resized value to
    140 and torch to 139.  The CHW path, which MIGAN_Pipeline runs, gives the same 140: the difference is the resize
    kernel's, which the crop pipeline has in either layout, and the reference vectors do not reach it."""
    from test_crop_pipeline_gpu import _requests, read_mask
    R = 256
    for i, (img, mask) in enumerate(_requests(np.random.default_rng(21), 7)):
        plane = read_mask(mask, False)
        chw = np.ascontiguousarray(img.transpose(2, 0, 1))
        m = _at_size(emul, [np.ascontiguousarray(plane)], [chw])[0]
        y = np.zeros((1, 3, R, R), np.float32)
        _, x_hwc = run_planned_layout(emul, [img.copy()], [m], R, 128, _abi.LAYOUT_HWC, y)
        _, x_chw = run_planned_layout(emul, [chw.copy()], [m], R, 128, _abi.LAYOUT_CHW, y)
        assert np.array_equal(x_hwc, x_chw), i
        taps = {}
        PO.forward(lambda _x: torch.zeros(1, 3, R, R), torch.from_numpy(chw[None].copy()),
                   torch.from_numpy(plane[None, None]), R, 128, taps)
        want = taps["x"].numpy()
        diff = np.argwhere(x_hwc != want).tolist()
        if i < 6:
            assert diff == [], i
        else:
            assert img.shape == (569, 405, 3) and mask.shape[2] == 3
            assert diff == [[0, 1, 200, 216]]
            level = lambda v: round((float(v) / float(x_hwc[0, 0, 200, 216] + 0.5) + 1) * 255 / 2)  # noqa: E731
            assert (level(x_hwc[0, 1, 200, 216]), level(want[0, 1, 200, 216])) == (140, 139)
