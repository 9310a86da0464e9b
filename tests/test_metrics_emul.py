"""SSIM and PSNR without a GPU: the taps and the float64 oracle against the reference's own values
(tests/golden/metrics.npz), and the library's kernels in the emulation build (the same per-pixel arithmetic, tile
staging, block trees and per-image reduction as host loops) against the oracle, with every argument refusal of the C
ABI and the workspace sizes."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

import build_emul  # noqa: E402
from migan_b200 import _abi, metrics  # noqa: E402
from oracle import metrics_oracle as O  # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "metrics.npz"))
PSNR_MODES = {"none": (None, 2), "div2k2": ("div2k", 2), "bench2": ("benchmark", 2), "bench4": ("benchmark", 4)}


@pytest.fixture(scope="module")
def emul():
    path = build_emul._compile("metrics_emul", [os.path.join(build_emul.CSRC, s) for s in ("metrics.cu", "abi_error.cu")])
    L = metrics.lib(ctypes.CDLL(path))
    L.migan_last_error.restype = ctypes.c_char_p
    return L


class Workspace:
    """8-byte aligned host memory with guard bytes after the `nbytes` the call may use."""

    def __init__(self, nbytes, guard=256):
        self.buf = (ctypes.c_uint8 * (nbytes + guard + 8))()
        self.base = (ctypes.addressof(self.buf) + 7) // 8 * 8
        self.nbytes, self.guard = nbytes, guard
        ctypes.memset(self.base + nbytes, 0xA5, guard)

    def guard_intact(self):
        return bytes((ctypes.c_uint8 * self.guard).from_address(self.base + self.nbytes)) == b"\xa5" * self.guard


def emul_ssim(L, x, y, ws, taps=None):
    """(per-image [n] float32, mean float32) of the emulated library."""
    x, y = x.float().contiguous(), y.float().contiguous()
    n, C, H, W = x.shape
    g = (metrics.gaussian_taps(ws) if taps is None else taps).float().contiguous()
    w = Workspace(L.metrics_ssim_workspace_bytes(n, C, H, W, ws))
    per = torch.full((n + 2,), -7.5)
    mean = torch.full((3,), -7.5)
    _abi.check(L.metrics_ssim(x.data_ptr(), y.data_ptr(), n, C, H, W, g.data_ptr(), ws, per[1:].data_ptr(),
                              mean[1:].data_ptr(), w.base, w.nbytes, None), L)
    assert w.guard_intact() and per[0] == -7.5 and per[-1] == -7.5 and mean[0] == -7.5 and mean[2] == -7.5
    return per[1:n + 1].clone(), mean[1].clone()


def emul_psnr(L, x, y, for_dataset, scale, rgb_range):
    x, y = x.float().contiguous(), y.float().contiguous()
    n, C, H, W = x.shape
    shave = {None: 0, "div2k": scale + 6, "benchmark": scale}[for_dataset]
    w = Workspace(L.metrics_psnr_workspace_bytes(n, H, W, shave))
    out = torch.full((n + 2,), -7.5, dtype=torch.float64)
    _abi.check(L.metrics_psnr(x.data_ptr(), y.data_ptr(), n, C, H, W, int(for_dataset == "benchmark"), shave,
                              float(rgb_range), out[1:].data_ptr(), w.base, w.nbytes, None), L)
    assert w.guard_intact() and out[0] == -7.5 and out[-1] == -7.5
    return out[1:n + 1].clone()


def _golden_ssim_keys():
    return sorted(k for k in GOLDEN.files if k.startswith("ssim_") and k.endswith("_img"))


# ---- the taps and the oracle against the reference's own values -------------------------------------------------------
def test_taps_are_the_references_bytes():
    for ws in range(1, 32):
        want = torch.from_numpy(GOLDEN["taps%d" % ws])
        assert metrics.gaussian_taps(ws).dtype == torch.float32
        assert torch.equal(metrics.gaussian_taps(ws), want), ws
        assert torch.equal(O.gaussian_taps(ws), want), ws


@pytest.mark.parametrize("key", _golden_ssim_keys())
def test_ssim_oracle_matches_reference(key):
    _, case, w, _ = key.split("_")
    ws = int(w[1:])
    x, y = torch.from_numpy(GOLDEN["x_" + case]), torch.from_numpy(GOLDEN["y_" + case])
    # the float32 mode is the reference's own arithmetic: the same bits
    assert torch.equal(O.ssim(x, y, ws, size_average=False, fp32=True), torch.from_numpy(GOLDEN[key]))
    assert torch.equal(O.ssim(x, y, ws, size_average=True, fp32=True), torch.from_numpy(GOLDEN[key[:-4] + "_mean"]))
    # float64 against the reference: its own float32 error, at most 7.8e-6 on the bright pair, ~3e-7 elsewhere
    err = float((O.ssim(x, y, ws, size_average=False) - torch.from_numpy(GOLDEN[key]).double()).abs().max())
    assert err < (2e-5 if case == "bright" else 1e-6), err


@pytest.mark.parametrize("case", ["hole", "unrelated", "same"])
@pytest.mark.parametrize("mode", sorted(PSNR_MODES))
@pytest.mark.parametrize("rgb_range", [1, 255])
def test_psnr_oracle_matches_reference(case, mode, rgb_range):
    x = torch.from_numpy(GOLDEN["x_hole" if case == "same" else "x_" + case])
    y = x if case == "same" else torch.from_numpy(GOLDEN["y_" + case])
    xs, ys = (x * rgb_range).numpy(), (y * rgb_range).numpy()
    for_dataset, scale = PSNR_MODES[mode]
    want = GOLDEN["psnr_%s_%s_r%d" % (case, mode, rgb_range)]
    got32 = O.psnr(xs, ys, for_dataset, scale, rgb_range, fp32=True)
    assert got32.dtype == want.dtype and np.array_equal(got32, want)
    got = O.psnr(xs, ys, for_dataset, scale, rgb_range)
    if case == "same":
        assert np.isposinf(got).all()
    else:
        assert np.abs(got - want).max() < 1e-5   # float32 rounding of a value near 30 dB: ~2e-6


# ---- the emulated library against the oracle ---------------------------------------------------------------------------
SSIM_CASES = [  # (n, C, H, W, window)
    (2, 3, 40, 37, 11), (2, 3, 40, 37, 8), (2, 3, 40, 37, 7), (2, 3, 40, 37, 1), (1, 3, 7, 5, 11), (2, 1, 40, 37, 11),
    (2, 4, 33, 70, 8), (1, 3, 97, 131, 11), (1, 2, 3, 3, 31), (1, 1, 66, 65, 2),
]


@pytest.mark.parametrize("case", SSIM_CASES, ids=["%dx%dx%dx%d_w%d" % c for c in SSIM_CASES])
@pytest.mark.parametrize("kind", ["hole", "bright"])
def test_emulated_ssim_matches_oracle(emul, case, kind):
    n, C, H, W, ws = case
    if kind == "hole":
        x = O.images(n, C, H, W, seed=H + ws)
        y = O.images(n, C, H, W, seed=H + ws + 1)
        y[..., H // 4:H // 2, W // 3:W // 2] = x[..., H // 4:H // 2, W // 3:W // 2]
    else:
        x, y = O.bright(n, C, H, W, seed=W), O.bright(n, C, H, W, seed=W + 1)
    per, mean = emul_ssim(emul, x, y, ws)
    want_per, want = O.ssim(x, y, ws, size_average=False), O.ssim(x, y, ws, size_average=True)
    err = max(float((per.double() - want_per).abs().max()), abs(float(mean) - float(want)))
    ref_err = max(float((O.ssim(x, y, ws, size_average=False, fp32=True).double() - want_per).abs().max()),
                  abs(float(O.ssim(x, y, ws, fp32=True)) - float(want)))
    print("emulated ssim %s %s: err %.2e, the reference's fp32 err %.2e" % (case, kind, err, ref_err))
    assert err <= 6e-8   # float32 rounding of values below 1
    assert err <= ref_err or err <= 3e-8


def test_emulated_ssim_symmetry_identity_and_batch_invariance(emul):
    x = O.images(5, 3, 45, 38, seed=1)
    y = O.composed(x, seed=2)
    per, mean = emul_ssim(emul, x, y, 11)
    per_ba, mean_ba = emul_ssim(emul, y, x, 11)
    assert torch.equal(per, per_ba) and torch.equal(mean, mean_ba)
    for i in range(5):
        assert torch.equal(emul_ssim(emul, x[i:i + 1], y[i:i + 1], 11)[0], per[i:i + 1])
    same, same_mean = emul_ssim(emul, x, x.clone(), 11)
    assert (same == 1).all() and same_mean == 1


@pytest.mark.parametrize("mode", sorted(PSNR_MODES))
@pytest.mark.parametrize("rgb_range", [1, 255])
def test_emulated_psnr_matches_oracle(emul, mode, rgb_range):
    for_dataset, scale = PSNR_MODES[mode]
    x = O.images(3, 3, 41, 37, seed=3) * rgb_range
    y = O.composed(O.images(3, 3, 41, 37, seed=3), seed=4) * rgb_range
    y[2] = O.images(1, 3, 41, 37, seed=5)[0] * rgb_range
    got = emul_psnr(emul, x, y, for_dataset, scale, rgb_range)
    want = torch.from_numpy(O.psnr(x, y, for_dataset, scale, rgb_range))
    err = float((got - want).abs().max())
    print("emulated psnr %s r%d: err %.2e dB" % (mode, rgb_range, err))
    assert err < 1e-9
    same = emul_psnr(emul, x, x.clone(), for_dataset, scale, rgb_range)
    assert torch.isposinf(same).all()


def test_emulated_psnr_any_channels(emul):
    x, y = O.images(2, 4, 20, 19, seed=1), O.images(2, 4, 20, 19, seed=2)
    got = emul_psnr(emul, x, y, None, 0, 1)
    d = (x.float() - y.float()).double()
    want = -10 * torch.log10((d ** 2).mean((1, 2, 3)))
    assert float((got - want).abs().max()) < 1e-9


# ---- the C ABI's refusals and workspace sizes -------------------------------------------------------------------------
def _fail(L, rc, *words):
    assert rc == _abi.ERR_INVALID
    msg = L.migan_last_error().decode()
    for w in words:
        assert w in msg, (w, msg)


def test_ssim_refusals(emul):
    L = emul
    x = torch.rand(1, 3, 8, 8)
    g = metrics.gaussian_taps(3)
    out = torch.empty(2)
    w = Workspace(L.metrics_ssim_workspace_bytes(1, 3, 8, 8, 3))
    p = x.data_ptr()

    def call(img1=p, img2=p, n=1, C=3, H=8, W=8, taps=g.data_ptr(), ws=3, per=out.data_ptr(), mean=None, base=w.base,
             nbytes=w.nbytes):
        return L.metrics_ssim(img1, img2, n, C, H, W, taps, ws, per, mean, base, nbytes, None)

    assert call() == 0
    _fail(L, call(img1=None), "null img1")
    _fail(L, call(img2=None), "null img1 / img2")
    _fail(L, call(taps=None), "taps")
    _fail(L, call(per=None, mean=None), "both null")
    _fail(L, call(ws=0), "window 0 outside 1..31")
    _fail(L, call(ws=32), "window 32 outside 1..31")
    _fail(L, call(n=0), "bad batch n=0")
    _fail(L, call(C=0), "C=0")
    _fail(L, call(H=0), "H=0")
    _fail(L, call(base=None), "null workspace")
    _fail(L, call(base=w.base + 4), "8-byte aligned")
    _fail(L, call(nbytes=w.nbytes - 1), "workspace of %d bytes, %d needed" % (w.nbytes - 1, w.nbytes))


def test_psnr_refusals(emul):
    L = emul
    x = torch.rand(1, 3, 20, 20)
    out = torch.empty(1, dtype=torch.float64)
    w = Workspace(L.metrics_psnr_workspace_bytes(1, 20, 20, 2))
    p = x.data_ptr()

    def call(pred=p, gt=p, n=1, C=3, H=20, W=20, gray=0, shave=2, rgb=1.0, o=out.data_ptr(), base=w.base,
             nbytes=w.nbytes):
        return L.metrics_psnr(pred, gt, n, C, H, W, gray, shave, rgb, o, base, nbytes, None)

    assert call() == 0 and call(gray=1) == 0
    _fail(L, call(pred=None), "null pred")
    _fail(L, call(gt=None), "null pred / gt / out")
    _fail(L, call(o=None), "out")
    _fail(L, call(gray=1, C=1), "C == 3", "C=1")
    _fail(L, call(C=0), "C=0")
    _fail(L, call(rgb=0.0), "rgb_range 0")
    _fail(L, call(rgb=-1.0), "rgb_range -1")
    _fail(L, call(rgb=float("nan")), "rgb_range")
    _fail(L, call(shave=10), "empty region")
    _fail(L, call(shave=-1), "shave -1")
    _fail(L, call(n=0), "n=0")
    _fail(L, call(base=None), "null workspace")
    _fail(L, call(nbytes=w.nbytes - 8), "needed")


def test_workspace_sizes(emul):
    L = emul
    # SSIM: one double per 32 x 32 tile of each plane's map, then one per image
    for n, C, H, W, ws in ((1, 3, 256, 256, 11), (32, 3, 512, 512, 11), (2, 1, 40, 37, 8), (3, 4, 7, 5, 11),
                           (1, 1, 64, 64, 2)):
        Ho, Wo = metrics.map_size(H, W, ws)
        tiles = -(-Ho // 32) * -(-Wo // 32)
        assert L.metrics_ssim_workspace_bytes(n, C, H, W, ws) == 8 * (n * C * tiles + n)
    assert metrics.map_size(40, 37, 8) == (41, 38)
    for bad in ((0, 3, 8, 8, 11), (1, 0, 8, 8, 11), (1, 3, 8, 8, 0), (1, 3, 8, 8, 32)):
        assert L.metrics_ssim_workspace_bytes(*bad) == 0
    # PSNR: one double per 8 rows of the valid region of each image, then one per image
    for n, H, W, shave in ((32, 512, 512, 8), (1, 40, 37, 0), (3, 41, 37, 4)):
        assert L.metrics_psnr_workspace_bytes(n, H, W, shave) == 8 * (n * -(-(H - 2 * shave) // 8) + n)
    for bad in ((0, 8, 8, 0), (1, 8, 8, 4), (1, 8, 8, -1)):
        assert L.metrics_psnr_workspace_bytes(*bad) == 0


def test_python_refuses_before_the_device():
    x = torch.rand(2, 3, 16, 16)
    with pytest.raises(RuntimeError, match="no CPU"):
        metrics.compute_ssim(x, x)
    with pytest.raises(RuntimeError, match="no CPU"):
        metrics.compute_psnr(x, x)
    for ws in (0, 32, 2.5):
        with pytest.raises(ValueError, match="window_size"):
            metrics.compute_ssim(x, x, window_size=ws)
        with pytest.raises(ValueError, match="window_size"):
            metrics.SSIM(window_size=ws)
    with pytest.raises(ValueError, match="scale"):
        metrics.compute_psnr(x, x, scale=-1)
    for r in (0, -255):
        with pytest.raises(ValueError, match="rgb_range"):
            metrics.compute_psnr(x, x, rgb_range=r)
    with pytest.raises(NotImplementedError, match="for_dataset"):
        metrics.compute_psnr(x, x, for_dataset="set5")
