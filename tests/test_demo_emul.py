"""CPU checks of the demo request path (mi-gan_b200/csrc/demo_resize.cu, scripts/demo.py:26-66, :120-143).

- oracle/demo_oracle.py equals Pillow and OpenCV (scalar path) on a sweep of random size pairs up to 4096, the NEAREST
  index map through a coordinate-ramp image (when Pillow / OpenCV are installed);
- the emulation build of demo_resize.cu (the same item functors, host loops) equals the oracle and the fixture of the
  reference's own functions byte for byte, and stays within 1 of OpenCV's default (optimised) path;
- a mixed batch of 32 equals the requests run one by one, and the argument checks refuse what demo.py cannot run."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from migan_b200 import _abi  # noqa: E402
from oracle import demo_oracle as O  # noqa: E402
import build_emul  # noqa: E402
import make_golden_demo as MG  # noqa: E402

NAMES = ("migan_demo_resized_size", "b200_demo_scratch_bytes", "b200_demo_preprocess", "b200_demo_postprocess")
SYMBOLS = [s for s in _abi.SYMBOLS if s[0] in NAMES]


@pytest.fixture(scope="module")
def emul():
    return _abi.bind(ctypes.CDLL(build_emul.build()), SYMBOLS)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def requests(imgs, masks, inverts, outs):
    reqs = (_abi.DemoRequest * len(imgs))()
    for r, img, m, inv, out in zip(reqs, imgs, masks, inverts, outs):
        r.img, r.H, r.W = img.ctypes.data, img.shape[0], img.shape[1]
        r.mask, r.Hm, r.Wm = m.ctypes.data, m.shape[0], m.shape[1]
        r.mask_channels = 1 if m.ndim == 2 else m.shape[2]
        r.invert = int(bool(inv))
        r.out, r.out_h, r.out_w = out.ctypes.data, out.shape[0], out.shape[1]
    return reqs


def run(lib, imgs, masks, inverts, ys, res):
    """One emulated pass: returns (x [n,4,R,R], outs)."""
    n = len(imgs)
    outs = []
    for img in imgs:
        w1, h1 = O.resized_size(img.shape[1], img.shape[0], res)
        outs.append(np.full((h1, w1, 3), 77, np.uint8))
    reqs = requests(imgs, masks, inverts, outs)
    nbytes = lib.b200_demo_scratch_bytes(reqs, n, res)
    assert nbytes > 0
    scratch = np.zeros(nbytes, np.uint8)
    x = np.full((n, 4, res, res), np.nan, np.float32)
    assert lib.b200_demo_preprocess(reqs, n, res, _ptr(x), _ptr(scratch), nbytes, None) == 0
    y = np.ascontiguousarray(np.stack(ys).astype(np.float32))
    assert lib.b200_demo_postprocess(_ptr(y), reqs, n, res, _ptr(scratch), nbytes, None) == 0
    return x, outs


def random_request(rng, res, max_side=None):
    """Photo, mask (random mode and size chain that demo.py accepts), invert, y."""
    max_side = max_side or 3 * res
    while True:
        W, H = int(rng.integers(1, max_side)), int(rng.integers(1, max_side))
        try:
            O.demo_sizes(W, H, W, H, res)
            break
        except ValueError:
            continue
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    C = int(rng.choice([1, 2, 3, 4]))
    m = np.where(rng.random((H, W, C)) < 0.6, 255, rng.choice(np.array([0, 254], np.uint8), (H, W, C))).astype(np.uint8)
    if C == 1:
        m = m[..., 0]
    y = (rng.standard_normal((3, res, res)) * 0.7).astype(np.float32)
    return img, np.ascontiguousarray(m), bool(rng.integers(0, 2)), y


def oracle(img, mask, invert, y, res):
    rs, m, x = O.demo_pre(img, mask, invert, res)
    return x, O.demo_post(y, rs, m)


# ---- the oracle against the libraries ---------------------------------------------------------------------------
def _size_pairs(seed, n):
    rng = np.random.default_rng(seed)
    pairs = [(512, 343), (343, 512), (1920, 512), (3840, 512), (1, 7), (7, 1), (4096, 1), (1, 4096)]
    while len(pairs) < n:
        a = int(rng.integers(1, 4097))
        b = int(rng.integers(1, 4097)) if rng.random() < 0.5 else max(1, int(a * rng.uniform(0.05, 2.0)))
        pairs.append((a, min(b, 4096)))
    return pairs


def test_oracle_pil_bicubic_sweep():
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(1)
    for i, (a, b) in enumerate(_size_pairs(2, 200)):
        if i % 2 == 0:   # width pass alone on 2 rows
            img = rng.integers(0, 256, (2, a, 3), dtype=np.uint8)
            size = (b, 2)
        else:            # height pass alone on 2 columns
            img = rng.integers(0, 256, (a, 2, 3), dtype=np.uint8)
            size = (2, b)
        ref = np.array(Image.fromarray(img).resize(size, Image.BICUBIC))
        assert np.array_equal(O.pil_bicubic(img, *size), ref), (a, b)
    for (W, H), (w, h) in [((512, 343), (512, 512)), ((343, 512), (256, 256)), ((1080, 1920), (288, 512)),
                           ((300, 200), (256, 256)), ((512, 512), (256, 256)), ((37, 90), (64, 64))]:
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        assert np.array_equal(O.pil_bicubic(img, w, h), np.array(Image.fromarray(img).resize((w, h), Image.BICUBIC)))


def test_oracle_pil_nearest_ramp():
    Image = pytest.importorskip("PIL.Image")
    for a, b in _size_pairs(3, 240):
        ramp = np.arange(a, dtype=np.int32)[None, :]
        ref = np.array(Image.fromarray(ramp, mode="I").resize((b, 1), Image.NEAREST))[0]
        assert np.array_equal(O.pil_nearest_index(a, b), ref), (a, b)


def test_oracle_cv_cubic_sweep():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(4)
    was = cv2.useOptimized()
    cv2.setUseOptimized(False)
    try:
        for i, (a, b) in enumerate(_size_pairs(5, 200)):
            img = rng.integers(0, 256, (2, a, 3) if i % 2 == 0 else (a, 2, 3), dtype=np.uint8)
            size = (b, 2) if i % 2 == 0 else (2, b)
            ref = cv2.resize(img, size, interpolation=cv2.INTER_CUBIC)
            assert np.array_equal(O.cv_cubic(img, *size), ref), (a, b)
        img = rng.integers(0, 256, (512, 512, 3), dtype=np.uint8)
        assert np.array_equal(O.cv_cubic(img, 343, 512), cv2.resize(img, (343, 512), interpolation=cv2.INTER_CUBIC))
    finally:
        cv2.setUseOptimized(was)


def test_resized_size_matches_python(emul):
    w, h = ctypes.c_int(), ctypes.c_int()
    rng = np.random.default_rng(6)
    for _ in range(500):
        a, b, m = int(rng.integers(1, 5000)), int(rng.integers(1, 5000)), int(rng.choice([32, 64, 256, 512, 1000]))
        assert emul.migan_demo_resized_size(a, b, m, ctypes.byref(w), ctypes.byref(h)) == 0
        assert (w.value, h.value) == O.resized_size(a, b, m)


# ---- the emulated functors --------------------------------------------------------------------------------------
def test_fixture(emul):
    gold = MG.load_fixture()
    assert float(gold["default_mismatch"]) < 0.05
    for i, (R, W, H, mode, invert) in enumerate(MG.CASES):
        img, mask, y = MG.case_inputs(i)
        x, outs = run(emul, [img], [mask], [invert], [y], R)
        ox, oout = oracle(img, mask, invert, y, R)
        assert np.array_equal(x[0], gold["%d_x" % i]), i
        assert np.array_equal(outs[0], gold["%d_out" % i]), i
        assert np.array_equal(x[0], ox) and np.array_equal(outs[0], oout), i
        d = np.abs(outs[0].astype(int) - gold["%d_out_default" % i].astype(int))
        assert d.max() <= 1, i


@pytest.mark.parametrize("res", [32, 64])
def test_random_requests_match_oracle(emul, res):
    rng = np.random.default_rng(res)
    for _ in range(12):
        img, mask, inv, y = random_request(rng, res)
        x, outs = run(emul, [img], [mask], [inv], [y], res)
        ox, oout = oracle(img, mask, inv, y, res)
        assert np.array_equal(x[0], ox)
        assert np.array_equal(outs[0], oout)


def test_large_photo_down_scale(emul):
    rng = np.random.default_rng(7)
    res = 64
    img = rng.integers(0, 256, (540, 960, 3), dtype=np.uint8)     # 15 x 15-tap down-scale to 64 x 36
    mask = np.where(rng.random((540, 960, 4)) < 0.7, 255, 0).astype(np.uint8)
    y = (rng.standard_normal((3, res, res)) * 0.7).astype(np.float32)
    x, outs = run(emul, [img], [mask], [False], [y], res)
    ox, oout = oracle(img, mask, False, y, res)
    assert np.array_equal(x[0], ox) and np.array_equal(outs[0], oout)


def test_mixed_batch_of_32_equals_single_calls(emul):
    rng = np.random.default_rng(8)
    res = 32
    reqs = [random_request(rng, res, max_side=120) for _ in range(32)]
    x, outs = run(emul, *[list(t) for t in zip(*reqs)], res)
    for k, (img, mask, inv, y) in enumerate(reqs):
        x1, o1 = run(emul, [img], [mask], [inv], [y], res)
        assert np.array_equal(x[k], x1[0]), k
        assert np.array_equal(outs[k], o1[0]), k


def test_argument_checks(emul):
    res = 32
    img = np.zeros((40, 50, 3), np.uint8)
    mask = np.full((40, 50), 255, np.uint8)
    w1, h1 = O.resized_size(50, 40, res)
    out = np.zeros((h1, w1, 3), np.uint8)
    x = np.zeros((1, 4, res, res), np.float32)

    def reqs(**kw):
        r = requests([img], [mask], [False], [out])
        for k, v in kw.items():
            setattr(r[0], k, v)
        return r

    good = reqs()
    nbytes = emul.b200_demo_scratch_bytes(good, 1, res)
    assert nbytes > 0
    scratch = np.zeros(nbytes, np.uint8)
    assert emul.b200_demo_preprocess(good, 1, res, _ptr(x), _ptr(scratch), nbytes, None) == 0
    bad = [dict(img=None), dict(mask=None), dict(out=None), dict(H=0), dict(Wm=0), dict(mask_channels=5),
           dict(mask_channels=0), dict(out_w=w1 + 1), dict(out_h=h1 - 1),
           dict(Wm=700, Hm=300)]                      # mask resizes to 32 x 13, photo to 32 x 25
    for kw in bad:
        r = reqs(**kw)
        assert emul.b200_demo_scratch_bytes(r, 1, res) == 0, kw
        assert emul.b200_demo_preprocess(r, 1, res, _ptr(x), _ptr(scratch), nbytes, None) == _abi.ERR_INVALID, kw
        assert emul.b200_demo_postprocess(_ptr(x), r, 1, res, _ptr(scratch), nbytes, None) == _abi.ERR_INVALID, kw
    assert emul.b200_demo_scratch_bytes(good, 0, res) == 0
    assert emul.b200_demo_scratch_bytes(good, 33, res) == 0
    assert emul.b200_demo_scratch_bytes(good, 1, 0) == 0
    assert emul.b200_demo_preprocess(good, 1, res, None, _ptr(scratch), nbytes, None) == _abi.ERR_INVALID
    assert emul.b200_demo_preprocess(good, 1, res, _ptr(x), _ptr(scratch), nbytes - 1, None) == _abi.ERR_WORKSPACE
    assert emul.b200_demo_postprocess(_ptr(x), good, 1, res, _ptr(scratch), nbytes - 1, None) == _abi.ERR_WORKSPACE
    # a strip that resizes to a 0-pixel side (demo.py's PIL resize refuses it)
    strip = np.zeros((1, 100, 3), np.uint8)
    r = requests([strip], [np.full((1, 100), 255, np.uint8)], [False], [out])
    r[0].out_w, r[0].out_h = 32, 0
    assert emul.b200_demo_scratch_bytes(r, 1, res) == 0
