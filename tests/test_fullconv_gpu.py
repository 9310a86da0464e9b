"""Fully convolutional forward (`Generator.forward_fc`, `migan_forward_hw`) on the H100.

Bounds are those of test_generator_gpu.py: max-abs < 1e-3 and mean-abs < 1e-4 against the fp32 oracle for the
fp32-faithful paths, 2e-4 * scale per intermediate.  Shapes cover non-square and non-power-of-two extents: at migan-512,
640 x 896 has a 40 x 56 32-level and a 5 x 7 bottleneck, i.e. partial tiles at every level below 64.
"""
import gc
import os

import numpy as np
import pytest
import torch

import migan_b200
from migan_b200 import _abi
from oracle import fullconv_oracle as FC
from oracle import migan_oracle as O
from oracle import prepost_oracle as P

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "fullconv.npz")
PATHS = ["simt", "tc"]
TOL_MAX_ABS = 1e-3
TOL_MEAN_ABS = 1e-4

_models = {}


def make_model(R, path, seed=1, device="cuda:0"):
    key = (R, path, seed)
    if key not in _models:
        sd = O.make_state_dict(R, seed=seed)
        g = migan_b200.Generator(R, path=path)
        g.load_state_dict(sd)
        _models[key] = (g.to(device).eval(), sd)
    return _models[key]


def errs(got, want):
    d = (got.double().cpu() - want.double()).abs()
    return float(d.max()), float(d.mean())


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("case", range(4))
def test_reference_fixture(cuda_device, path, case):
    """Outputs of the reference itself with size-dependent filter_const / noise_const (make_golden_fullconv.py)."""
    z = np.load(GOLD)
    R, N, H, W, wseed, xseed = [int(v) for v in z["case%d_meta" % case]]
    g, _ = make_model(R, path, seed=wseed)
    x = FC.make_input_hw(R, N, H, W, seed=xseed)
    got = g.forward_fc(x.to(cuda_device))
    assert got.shape == (N, 3, H, W) and got.dtype == torch.float32 and got.is_contiguous()
    rows = torch.from_numpy(z["case%d_rows" % case]).to(cuda_device)     # the fixture keeps a row sample
    mx, mean = errs(got[:, :, rows], torch.from_numpy(z["case%d_y" % case]))
    print("fullconv fixture R=%d %dx%d n=%d path=%s max-abs=%.3e mean-abs=%.3e" % (R, H, W, N, path, mx, mean))
    assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("R,N,H,W", [(256, 1, 256, 384), (256, 1, 320, 256), (512, 1, 512, 768), (512, 1, 640, 896),
                                     (512, 1, 1024, 1536), (512, 3, 768, 512)])
def test_matches_oracle(cuda_device, path, R, N, H, W):
    g, sd = make_model(R, path)
    x = FC.make_input_hw(R, N, H, W, seed=H + W)
    want = FC.generator_forward_fc(sd, x, R)
    got = g.forward_fc(x.to(cuda_device))
    mx, mean = errs(got, want)
    print("path=%s R=%d %dx%d n=%d max-abs=%.3e mean-abs=%.3e (|y|max=%.2f)" % (path, R, H, W, N, mx, mean, float(want.abs().max())))
    assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("R,H,W", [(256, 640, 320), (128, 160, 224)])
def test_every_intermediate_matches_oracle(cuda_device, path, R, H, W):
    N = 2
    g, sd = make_model(R, path)
    x = FC.make_input_hw(R, N, H, W, seed=5)
    taps = {}
    FC.generator_forward_fc(sd, x, R, taps=taps)
    xd = x.to(cuda_device)
    names = g.tap_names()
    assert len(names) > 20
    bad = []
    for name, (c, h, w) in names:
        _, got = g.forward_fc(xd, tap=name)
        assert tuple(got.shape) == (N, c, h * H // R, w * W // R)
        if name.endswith("out_skip"):
            want = taps[name[: -len("_skip")]] + taps["feat%d" % h]
        else:
            want = taps[name]
        scale = max(float(want.abs().max()), 1.0)
        mx, _ = errs(got, want)
        if not (mx < 2e-4 * scale):
            bad.append((name, mx, scale))
    assert not bad, "first mismatching stages: %s" % bad[:5]


@pytest.mark.parametrize("R", [256, 512])
@pytest.mark.parametrize("N", [1, 3, 32])
def test_model_resolution_gives_forward_bytes(cuda_device, R, N):
    for path in PATHS:
        g, _ = make_model(R, path)
        x = O.make_input(R, N, seed=N).to(cuda_device)
        assert torch.equal(g.forward_fc(x), g(x)), (path, R, N)


@pytest.mark.parametrize("path", PATHS)
def test_batch_rows_equal_single_calls(cuda_device, path):
    g, _ = make_model(512, path)
    x = FC.make_input_hw(512, 4, 640, 896, seed=3).to(cuda_device)
    y4 = g.forward_fc(x)
    for i in range(4):
        assert torch.equal(y4[i:i + 1], g.forward_fc(x[i:i + 1].contiguous())), i


@pytest.mark.parametrize("path", PATHS)
def test_interleaved_shapes(cuda_device, path):
    """640 x 896, then 512 x 512 through forward (graph and plain), then 1024 x 512: each equals the same call alone, and
    forward / forward_u8 are unchanged by the shape changes around them."""
    g, _ = make_model(512, path)
    xa = FC.make_input_hw(512, 2, 640, 896, seed=1).to(cuda_device)
    xg = O.make_input(512, 2, seed=2).to(cuda_device)        # n <= graph_max_batch: the captured graph
    xp = O.make_input(512, 6, seed=3).to(cuda_device)        # the plain launch sequence
    xb = FC.make_input_hw(512, 2, 1024, 512, seed=4).to(cuda_device)
    rng = np.random.RandomState(0)
    img = torch.from_numpy(rng.randint(0, 256, size=(2, 512, 512, 3)).astype(np.uint8))
    mask = torch.from_numpy((rng.rand(2, 512, 512) > 0.3).astype(np.uint8) * 255)
    alone = [g.forward_fc(xa), g(xg), g(xp), g.forward_u8(img, mask).clone(), g.forward_fc(xb)]
    for _ in range(2):
        seq = [g.forward_fc(xa), g(xg), g(xp), g.forward_u8(img, mask).clone(), g.forward_fc(xb)]
        for i, (a, b) in enumerate(zip(alone, seq)):
            assert torch.equal(a, b), i


def test_launch_count(cuda_device):
    _models.clear()                 # n = 32 at 768 x 512 needs 15 GB of workspace: release the other models' first
    gc.collect()
    torch.cuda.empty_cache()
    g, _ = make_model(512, "tc")
    g(O.make_input(512, 32, seed=1).to(cuda_device))
    square = g.last_launch_count()
    assert square == 51
    for H, W in [(512, 512), (640, 896), (768, 512)]:
        g.forward_fc(FC.make_input_hw(512, 32, H, W, seed=2).to(cuda_device))
        assert g.last_launch_count() <= square + 1, (H, W, g.last_launch_count())
    g.forward_fc(O.make_input(512, 32, seed=1).to(cuda_device))
    assert g.last_launch_count() == square


def test_tc_fast_stated_accuracy(cuda_device):
    R, H, W = 512, 640, 896
    g, sd = make_model(R, "tc_fast")
    x = FC.make_input_hw(R, 1, H, W, seed=11)
    want = FC.generator_forward_fc(sd, x, R)
    mx, mean = errs(g.forward_fc(x.to(cuda_device)), want)
    print("tc_fast %dx%d max-abs=%.3e mean-abs=%.3e" % (H, W, mx, mean))
    assert mx < 1e-1 and mean < 1e-2
    assert mx > 1e-4


@pytest.mark.parametrize("path", PATHS)
def test_forward_fc_u8_equals_demo_expressions(cuda_device, path):
    g, _ = make_model(512, path)
    n, H, W = 2, 640, 896
    rng = np.random.RandomState(7)
    img = rng.randint(0, 256, size=(n, H, W, 3)).astype(np.uint8)
    mask = rng.choice(np.array([0, 100, 255, 255], np.uint8), size=(n, H, W))
    out = g.forward_fc_u8(torch.from_numpy(img).to(cuda_device), torch.from_numpy(mask).to(cuda_device))
    assert out.is_cuda and out.dtype == torch.uint8 and tuple(out.shape) == (n, H, W, 3)
    y = g.forward_fc(P.preprocess(img, mask).to(cuda_device))
    want = P.postprocess(y.cpu(), img, mask)
    assert np.array_equal(out.cpu().numpy(), want)


@pytest.mark.parametrize("H,W", [(640, 600), (384, 512), (512, 300)])
def test_refused_shapes(cuda_device, H, W):
    g, _ = make_model(512, "tc")
    eng = g._engine(torch.device(cuda_device))
    x = torch.zeros(1, 4, H, W, device=cuda_device)
    torch.cuda.synchronize()
    mem0, nws = torch.cuda.memory_allocated(), len(eng.workspaces)
    with pytest.raises(ValueError, match="nearest valid sizes"):
        g.forward_fc(x)
    with pytest.raises(ValueError, match="nearest valid sizes"):
        g.forward_fc_u8(torch.zeros(1, H, W, 3, dtype=torch.uint8, device=cuda_device),
                        torch.zeros(1, H, W, dtype=torch.uint8, device=cuda_device))
    assert torch.cuda.memory_allocated() == mem0 and len(eng.workspaces) == nws
    lib = eng.lib
    assert lib.migan_workspace_bytes_hw(eng.handle, 1, H, W) == 0
    y = torch.empty(1, 3, H, W, device=cuda_device)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=cuda_device)
    s = torch.cuda.current_stream().cuda_stream
    assert lib.migan_forward_hw(eng.handle, x.data_ptr(), y.data_ptr(), 1, H, W, ws.data_ptr(), ws.numel(),
                                _abi.PATH_TC, s) == _abi.ERR_INVALID


def test_element_limit_through_the_abi(cuda_device):
    """n = 8 at 2048 x 2048 is 2^31 elements in the largest activation: refused without allocating the input."""
    g, _ = make_model(512, "tc")
    eng = g._engine(torch.device(cuda_device))
    lib = eng.lib
    assert lib.migan_workspace_bytes_hw(eng.handle, 8, 2048, 2048) == 0
    assert b"2^31" in lib.migan_last_error()
    dummy = torch.empty(1 << 12, dtype=torch.uint8, device=cuda_device)
    p = dummy.data_ptr()
    assert lib.migan_forward_hw(eng.handle, p, p, 8, 2048, 2048, p, dummy.numel(), _abi.PATH_TC,
                                torch.cuda.current_stream().cuda_stream) == _abi.ERR_INVALID
    assert lib.migan_workspace_bytes_hw(eng.handle, 7, 2048, 2048) > 0


def test_input_errors(cuda_device):
    g, _ = make_model(256, "tc")
    with pytest.raises(RuntimeError):
        g.forward_fc(torch.zeros(1, 4, 256, 320))                                    # CPU tensor: no CPU path
    with pytest.raises(RuntimeError):
        g.forward_fc(torch.zeros(1, 4, 256, 320, device=cuda_device, dtype=torch.float16))
    with pytest.raises(RuntimeError):
        g.forward_fc(torch.zeros(1, 3, 256, 320, device=cuda_device))
