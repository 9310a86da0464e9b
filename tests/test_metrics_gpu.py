"""SSIM and PSNR on the H100: against the float64 oracle and the reference's own values (tests/golden/metrics.npz),
the reference's float32 error on the same inputs, bitwise batch invariance, symmetry and identity, guard bands around
every output and workspace, the two launches per call, the refusals, and the evaluation step end to end."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import migan_b200  # noqa: E402
from migan_b200 import _abi, metrics  # noqa: E402
from oracle import metrics_oracle as O  # noqa: E402
from oracle import migan_oracle as MO  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "metrics.npz"))
PSNR_MODES = {"none": (None, 2), "div2k2": ("div2k", 2), "bench2": ("benchmark", 2), "bench4": ("benchmark", 4)}
# Largest absolute error against the float64 oracle measured on an H100 (NVIDIA H100 80GB HBM3, 700 W) over
# test_ssim_matches_oracle, per-image values and the size_average mean: 2.95e-8, the float32 rounding of values below 1.
# Bound ~3x.  The reference's own float32 arithmetic measures up to 2.2e-5 on the same inputs (the bright pairs).
SSIM_TOL = 9e-8
# PSNR in dB, largest error measured on the same card: 9.4e-7 for None / "div2k" (the float32 result), 7.1e-15 for
# "benchmark" (double).  Bounds ~3x.
PSNR_TOL_F32, PSNR_TOL_F64 = 3e-6, 2.2e-14
GUARD = 4096


def _pair(kind, n, C, H, W, seed):
    if kind == "hole":
        x = O.images(n, C, H, W, seed=seed)
        y = O.images(n, C, H, W, seed=seed + 1)
        keep = torch.ones(1, 1, H, W, dtype=torch.bool)
        keep[..., H // 4:H // 4 + max(1, H // 3), W // 3:W // 3 + max(1, W // 3)] = False
        y = torch.where(keep, x, y)   # the composed image: the real one outside the hole
    elif kind == "unrelated":
        x, y = O.images(n, C, H, W, seed=seed), O.images(n, C, H, W, seed=seed + 1)
    else:
        x, y = O.bright(n, C, H, W, seed=seed), O.bright(n, C, H, W, seed=seed + 1)
    return x, y


SHAPES = [(1, 3, 256, 256), (3, 3, 512, 512), (33, 3, 97, 131), (2, 1, 7, 5), (3, 4, 40, 37)]


@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
@pytest.mark.parametrize("ws", [11, 7, 8, 1])
@pytest.mark.parametrize("kind", ["hole", "unrelated", "bright"])
def test_ssim_matches_oracle(shape, ws, kind):
    n, C, H, W = shape
    x, y = _pair(kind, n, C, H, W, seed=H + ws)
    xd, yd = x.to(DEV), y.to(DEV)
    per = metrics.compute_ssim(xd, yd, ws, size_average=False)
    mean = metrics.compute_ssim(xd, yd, ws)
    assert per.shape == (n,) and per.dtype == torch.float32 and per.is_cuda
    assert mean.shape == () and mean.dtype == torch.float32 and mean.is_cuda
    want_per, want = O.ssim(x, y, ws, size_average=False), O.ssim(x, y, ws)
    err = max(float((per.cpu().double() - want_per).abs().max()), abs(float(mean) - float(want)))
    ref_per, ref = O.ssim(x, y, ws, size_average=False, fp32=True), O.ssim(x, y, ws, fp32=True)
    ref_err = max(float((ref_per.double() - want_per).abs().max()), abs(float(ref) - float(want)))
    print("ssim %s w%d %s: err %.2e, the reference's fp32 err %.2e" % (shape, ws, kind, err, ref_err))
    assert err < SSIM_TOL
    assert err <= ref_err


@pytest.mark.parametrize("key", sorted(k for k in GOLDEN.files if k.startswith("ssim_") and k.endswith("_img")))
def test_ssim_matches_reference_values(key):
    _, case, w, _ = key.split("_")
    ws = int(w[1:])
    x, y = torch.from_numpy(GOLDEN["x_" + case]), torch.from_numpy(GOLDEN["y_" + case])
    per = metrics.compute_ssim(x.to(DEV), y.to(DEV), ws, size_average=False).cpu()
    mean = metrics.compute_ssim(x.to(DEV), y.to(DEV), ws).cpu()
    ref_per, ref = torch.from_numpy(GOLDEN[key]), torch.from_numpy(GOLDEN[key[:-4] + "_mean"])
    want_per = O.ssim(x, y, ws, size_average=False)
    # the reference's value differs from ours by at most its own error plus our rounding
    bound = float((ref_per.double() - want_per).abs().max()) + SSIM_TOL
    assert float((per.double() - ref_per.double()).abs().max()) <= bound
    assert abs(float(mean) - float(ref)) <= bound + abs(float(ref) - float(O.ssim(x, y, ws)))
    assert torch.equal(metrics.SSIM(ws, size_average=False)(x.to(DEV), y.to(DEV)).cpu(), per)


@pytest.mark.parametrize("case", ["hole", "unrelated", "same"])
@pytest.mark.parametrize("mode", sorted(PSNR_MODES))
@pytest.mark.parametrize("rgb_range", [1, 255])
def test_psnr_matches_reference_and_oracle(case, mode, rgb_range):
    x = torch.from_numpy(GOLDEN["x_hole" if case == "same" else "x_" + case])
    y = x.clone() if case == "same" else torch.from_numpy(GOLDEN["y_" + case])
    x, y = x * rgb_range, y * rgb_range
    for_dataset, scale = PSNR_MODES[mode]
    got = metrics.compute_psnr(x.to(DEV), y.to(DEV), for_dataset, scale, rgb_range)
    ref = GOLDEN["psnr_%s_%s_r%d" % (case, mode, rgb_range)]
    assert got.is_cuda and got.shape == (2,) and str(got.dtype) == "torch." + str(ref.dtype)
    got = got.cpu().double().numpy()
    if case == "same":
        assert np.isposinf(got).all() and np.isposinf(ref).all()
        return
    want = O.psnr(x, y, for_dataset, scale, rgb_range)
    tol = PSNR_TOL_F64 if for_dataset == "benchmark" else PSNR_TOL_F32
    err = float(np.abs(got - want).max())
    print("psnr %s %s r%d: err %.2e dB, the reference's %.2e" % (case, mode, rgb_range, err, np.abs(ref - want).max()))
    assert err < tol
    assert np.abs(got - ref).max() < 1e-5


@pytest.mark.parametrize("mode", sorted(PSNR_MODES))
def test_psnr_large(mode):
    for_dataset, scale = PSNR_MODES[mode]
    x, y = _pair("hole", 3, 3, 512, 512, seed=1)
    got = metrics.compute_psnr(x.to(DEV), y.to(DEV), for_dataset, scale).cpu().double().numpy()
    want = O.psnr(x, y, for_dataset, scale, 1)
    err = float(np.abs(got - want).max())
    print("psnr 3x3x512x512 %s: err %.2e dB" % (mode, err))
    assert err < (PSNR_TOL_F64 if for_dataset == "benchmark" else PSNR_TOL_F32)


def test_batch_invariance_symmetry_identity():
    x, y = _pair("hole", 33, 3, 97, 131, seed=3)
    x, y = x.to(DEV), y.to(DEV)
    for ws in (11, 8):
        full = metrics.compute_ssim(x, y, ws, size_average=False)
        for i in (0, 5, 17, 32):
            alone = metrics.compute_ssim(x[i:i + 1], y[i:i + 1], ws, size_average=False)
            assert torch.equal(alone[0], full[i])
            # the same image at another position of a batch of 33
            perm = torch.roll(torch.arange(33, device=DEV), 7)
            moved = metrics.compute_ssim(x[perm], y[perm], ws, size_average=False)
            assert torch.equal(moved, full[perm])
        assert torch.equal(metrics.compute_ssim(y, x, ws, size_average=False), full)
        assert torch.equal(metrics.compute_ssim(y, x, ws), metrics.compute_ssim(x, y, ws))
        assert (metrics.compute_ssim(x, x.clone(), ws, size_average=False) == 1).all()
        assert float(metrics.compute_ssim(x, x.clone(), ws)) == 1.0
    for for_dataset, scale in PSNR_MODES.values():
        full = metrics.compute_psnr(x, y, for_dataset, scale)
        assert torch.equal(metrics.compute_psnr(x[5:6], y[5:6], for_dataset, scale)[0], full[5])
        assert torch.equal(metrics.compute_psnr(y, x, for_dataset, scale), full)
        assert torch.isposinf(metrics.compute_psnr(x, x.clone(), for_dataset, scale)).all()


def test_guard_bands():
    L = metrics.lib()
    x, y = _pair("hole", 3, 3, 61, 70, seed=4)
    x, y = x.to(DEV), y.to(DEV)
    n, C, H, W = x.shape
    stream = torch.cuda.current_stream().cuda_stream
    taps = metrics.gaussian_taps(11)
    nbytes = L.metrics_ssim_workspace_bytes(n, C, H, W, 11)
    ws = torch.full((GUARD + nbytes // 8 + GUARD,), -7.5, dtype=torch.float64, device=DEV)
    out = torch.full((GUARD + n + 1 + GUARD,), -7.5, device=DEV)
    _abi.check(L.metrics_ssim(x.data_ptr(), y.data_ptr(), n, C, H, W, taps.data_ptr(), 11, out[GUARD:].data_ptr(),
                              out[GUARD + n:].data_ptr(), ws[GUARD:].data_ptr(), nbytes, stream), L)
    o, w = out.cpu(), ws.cpu()
    assert (o[:GUARD] == -7.5).all() and (o[GUARD + n + 1:] == -7.5).all()
    assert (w[:GUARD] == -7.5).all() and (w[GUARD + nbytes // 8:] == -7.5).all()
    assert torch.equal(o[GUARD:GUARD + n], metrics.compute_ssim(x, y, size_average=False).cpu())
    assert o[GUARD + n] == metrics.compute_ssim(x, y).cpu()
    for gray, shave in ((0, 0), (0, 8), (1, 2)):
        nbytes = L.metrics_psnr_workspace_bytes(n, H, W, shave)
        ws = torch.full((GUARD + nbytes // 8 + GUARD,), -7.5, dtype=torch.float64, device=DEV)
        out = torch.full((GUARD + n + GUARD,), -7.5, dtype=torch.float64, device=DEV)
        _abi.check(L.metrics_psnr(x.data_ptr(), y.data_ptr(), n, C, H, W, gray, shave, 1.0, out[GUARD:].data_ptr(),
                                  ws[GUARD:].data_ptr(), nbytes, stream), L)
        o, w = out.cpu(), ws.cpu()
        assert (o[:GUARD] == -7.5).all() and (o[GUARD + n:] == -7.5).all() and (o[GUARD:GUARD + n] > 0).all()
        assert (w[:GUARD] == -7.5).all() and (w[GUARD + nbytes // 8:] == -7.5).all()


def test_two_launches_per_call():
    x, y = _pair("hole", 4, 3, 128, 128, seed=5)
    x, y = x.to(DEV), y.to(DEV)
    metrics.compute_ssim(x, y)
    metrics.compute_psnr(x, y)
    torch.cuda.synchronize()
    counts = {}
    for name, fn in (("ssim", lambda: metrics.compute_ssim(x, y)), ("ssim_img", lambda: metrics.compute_ssim(x, y, 8, False)),
                     ("psnr", lambda: metrics.compute_psnr(x, y)), ("psnr_gray", lambda: metrics.compute_psnr(x, y, "benchmark", 4))):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            # a tracer started after an earlier session in the process can miss its first few kernel records: lead with
            # torch kernels that are not counted
            pad = torch.zeros(1, device=DEV)
            for _ in range(256):
                pad.add_(1)
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
        ours = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "metrics_" in e.name]
        counts[name] = ours
        assert len(ours) == 2, ours
        assert "metrics_reduce_kernel" in ours[-1]
    assert "metrics_ssim_tile_kernel" in counts["ssim"][0] and "metrics_psnr_kernel" in counts["psnr"][0]


def test_refusals():
    x = torch.rand(2, 3, 20, 20, device=DEV)
    with pytest.raises(RuntimeError, match="no CPU path"):
        metrics.compute_ssim(x.cpu(), x.cpu())
    with pytest.raises(RuntimeError, match="no CPU path"):
        metrics.compute_psnr(x.cpu(), x.cpu())
    with pytest.raises(RuntimeError, match="shape"):
        metrics.compute_ssim(x, x[:1])
    for ws in (0, 32):
        with pytest.raises(ValueError, match="window_size"):
            metrics.compute_ssim(x, x, ws)
    with pytest.raises(ValueError, match="nothing is left"):
        metrics.compute_psnr(x, x, "benchmark", 0)        # the reference's x[0:-0]
    with pytest.raises(ValueError, match="nothing is left"):
        metrics.compute_psnr(x, x, "div2k", 4)            # 10 pixels off each side of 20
    with pytest.raises(ValueError, match="scale"):
        metrics.compute_psnr(x, x, "div2k", -1)
    with pytest.raises(ValueError, match="rgb_range"):
        metrics.compute_psnr(x, x, rgb_range=0)
    with pytest.raises(ValueError, match="C=1"):
        metrics.compute_psnr(x[:, :1], x[:, :1], None)
    # an empty batch: empty per-image values, and torch's NaN mean of nothing
    e = x[:0]
    assert metrics.compute_ssim(e, e, size_average=False).shape == (0,)
    assert torch.isnan(metrics.compute_ssim(e, e)) and metrics.compute_ssim(e, e).shape == ()
    assert metrics.compute_psnr(e, e).shape == (0,) and metrics.compute_psnr(e, e, "benchmark").dtype == torch.float64


def test_evaluation_step_end_to_end():
    """EvalPipeline's (real, composed) at R = 64: SSIM and PSNR against the oracle on the same tensors."""
    R, n = 64, 6
    pipe = migan_b200.EvalPipeline(MO.make_state_dict(R, seed=1), resolution=R, device=DEV, seed=0)
    rng = np.random.default_rng(3)
    imgs = [rng.integers(0, 256, size=(R + 13 * i, R + 7 * i, 3), dtype=np.uint8) for i in range(n)]
    real, composed = pipe.forward_batch(imgs)
    assert real.shape == (n, 3, R, R)
    r, c = real.cpu(), composed.cpu()
    per = metrics.compute_ssim(real, composed, size_average=False).cpu().double()
    err = float((per - O.ssim(r, c, size_average=False)).abs().max())
    for for_dataset, scale in PSNR_MODES.values():
        got = metrics.compute_psnr(real, composed, for_dataset, scale).cpu().double().numpy()
        perr = float(np.abs(got - O.psnr(r, c, for_dataset, scale, 1)).max())
        print("evaluation step: PSNR %s err %.2e dB" % (for_dataset, perr))
        assert perr < (PSNR_TOL_F64 if for_dataset == "benchmark" else PSNR_TOL_F32), (for_dataset, perr)
    print("evaluation step: SSIM %s, err %.2e" % (np.round(per.numpy(), 5).tolist(), err))
    assert err < SSIM_TOL
