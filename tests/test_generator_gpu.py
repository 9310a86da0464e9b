"""Parity of the CUDA generator (through the C ABI) against the CPU oracle -- needs an H100.

Tolerance (north_star): max-abs error < 1e-3 vs the fp32 reference on identical inputs, for the
fp32-faithful paths ("simt": fp32 FMA, "tc": wgmma fp16 hi/lo 3-pass).  Outputs have
magnitude ~5-25, and the fp32-vs-fp64 noise floor of the reference itself is ~1e-5.
"""
import glob
import os

import numpy as np
import pytest
import torch

import migan_b200
from oracle import migan_oracle as O

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
PATHS = ["simt", "tc"]
TOL_MAX_ABS = 1e-3
TOL_MEAN_ABS = 1e-4


def make_model(R, path, seed=1, device="cuda:0"):
    sd = O.make_state_dict(R, seed=seed)
    g = migan_b200.Generator(R, path=path)
    g.load_state_dict(sd)
    return g.to(device).eval(), sd


def errs(got, want):
    d = (got.double().cpu() - want.double()).abs()
    return float(d.max()), float(d.mean())


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("R,N", [(64, 3), (128, 2), (256, 2)])
def test_forward_matches_oracle(cuda_device, path, R, N):
    g, sd = make_model(R, path)
    x = O.make_input(R, N, seed=11)
    want = O.generator_forward(sd, x, R)
    got = g(x.to(cuda_device))
    assert got.shape == want.shape and got.dtype == torch.float32 and got.is_contiguous()
    mx, mean = errs(got, want)
    print("path=%s R=%d N=%d max-abs=%.3e mean-abs=%.3e (|y|max=%.2f)" % (path, R, N, mx, mean, float(want.abs().max())))
    assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS


@pytest.mark.parametrize("path,R", [("simt", 64), ("tc", 64), ("tc", 256)])
def test_every_intermediate_matches_oracle(cuda_device, path, R):
    """Walk the plan stage by stage (debug taps) so a failure names the first bad kernel.
    R=256 on the tensor-core path also covers the fused torgb epilogue (C <= 128 levels)."""
    N = 2
    g, sd = make_model(R, path)
    x = O.make_input(R, N, seed=5)
    taps = {}
    O.generator_forward(sd, x, R, taps=taps)
    xd = x.to(cuda_device)
    names = g.tap_names()
    assert len(names) > 20
    bad = []
    for name, shape in names:
        _, got = g.forward_with_tap(xd, name, shape)
        if name.endswith("out_skip"):
            base = name[: -len("_skip")]
            res = shape[1]
            want = taps[base] + taps["feat%d" % res]
        else:
            want = taps[name]
        scale = max(float(want.abs().max()), 1.0)
        mx, _ = errs(got, want)
        if not (mx < 2e-4 * scale):
            bad.append((name, mx, scale))
    assert not bad, "first mismatching stages: %s" % bad[:5]


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("fixture", sorted(glob.glob(os.path.join(GOLDEN, "migan_R*.npz"))))
def test_golden_fixture(cuda_device, path, fixture):
    """Outputs of the REAL reference (generated in the build container) on seeded weights/inputs."""
    z = np.load(fixture)
    R, N = int(z["resolution"]), int(z["n"])
    g, sd = make_model(R, path, seed=int(z["wseed"]))
    x = O.make_input(R, N, seed=int(z["xseed"]))
    got = g(x.to(cuda_device))
    if "y_rows" in z.files:                              # large outputs are stored on a row sample (shrink_golden.py)
        got = got[:, :, torch.from_numpy(z["y_rows"]).to(cuda_device)]
    mx, mean = errs(got, torch.from_numpy(z["y"]))
    print("golden %s path=%s max-abs=%.3e mean-abs=%.3e" % (os.path.basename(fixture), path, mx, mean))
    assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS


@pytest.mark.parametrize("path", PATHS)
def test_clamp_saturation(cuda_device, path):
    """Random weights never reach the +-256 clamp (SURVEY 7.4(7)); scale the input until they do."""
    R, N = 64, 2
    g, sd = make_model(R, path)
    x = O.make_input(R, N, seed=3) * 3000.0
    taps = {}
    want = O.generator_forward(sd, x, R, taps=taps)
    assert float(taps["encoder.b64.conv1.dw_act"].abs().max()) == 256.0  # the case does saturate
    got = g(x.to(cuda_device))
    mx, _ = errs(got, want)
    assert mx < 1e-4 * float(want.abs().max())


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("mask_value", [0.0, 1.0])
def test_all_hole_and_all_known(cuda_device, path, mask_value):
    R, N = 64, 2
    g, sd = make_model(R, path)
    gen = torch.Generator().manual_seed(8)
    img = torch.rand(N, 3, R, R, generator=gen) * 2 - 1
    mask = torch.full((N, 1, R, R), mask_value)
    x = torch.cat([mask - 0.5, img * mask], 1)
    want = O.generator_forward(sd, x, R)
    mx, _ = errs(g(x.to(cuda_device)), want)
    assert mx < TOL_MAX_ABS


@pytest.mark.parametrize("path", PATHS)
def test_batch_independence_and_ragged_batches(cuda_device, path):
    """Images are independent (no batch statistics): N=1, N=5 and N=8 agree image by image."""
    R = 64
    g, sd = make_model(R, path)
    x = O.make_input(R, 8, seed=21).to(cuda_device)
    y8 = g(x)
    y5 = g(x[:5].contiguous())
    y1 = g(x[3:4].contiguous())
    assert torch.equal(y8[:5], y5)
    assert torch.equal(y8[3:4], y1)
    want = O.generator_forward(sd, x[3:4].cpu(), R)
    assert errs(y1, want)[0] < TOL_MAX_ABS


@pytest.mark.parametrize("path", PATHS)
def test_deterministic_and_input_untouched(cuda_device, path):
    R = 64
    g, _ = make_model(R, path)
    x = O.make_input(R, 2, seed=2).to(cuda_device)
    x0 = x.clone()
    a, b = g(x), g(x)
    assert torch.equal(a, b) and a.data_ptr() != b.data_ptr()
    assert torch.equal(x, x0)


def test_reload_weights_and_noncontiguous_input(cuda_device):
    R = 64
    g, sd = make_model(R, "simt")
    x = O.make_input(R, 2, seed=2)
    y1 = g(x.to(cuda_device))
    sd2 = O.make_state_dict(R, seed=9)
    g.load_state_dict(sd2)
    y2 = g(x.to(cuda_device))
    assert errs(y2, O.generator_forward(sd2, x, R))[0] < TOL_MAX_ABS
    assert not torch.equal(y1, y2)
    xt = x.to(cuda_device).permute(0, 1, 3, 2).contiguous().permute(0, 1, 3, 2)  # non-contiguous view
    assert not xt.is_contiguous()
    assert torch.equal(g(xt), y2)


def test_forward_host_end_to_end(cuda_device):
    R, N = 64, 3
    g, sd = make_model(R, "simt")
    x = O.make_input(R, N, seed=4).pin_memory()
    y = g.forward_host(x)
    assert not y.is_cuda and y.is_pinned()
    assert errs(y, O.generator_forward(sd, x, R))[0] < TOL_MAX_ABS


def test_forward_host_micro_batch_pipeline(cuda_device):
    """n = 16 takes the 2-micro-batch H2D / compute / D2H pipeline; results must equal the resident-input path."""
    R, N = 64, 16
    g, sd = make_model(R, "tc")
    x = O.make_input(R, N, seed=6).pin_memory()
    y = g.forward_host(x)
    want = g(x.to(cuda_device)).cpu()
    assert torch.equal(y, want)
    assert errs(y[[0, 15]], O.generator_forward(sd, x[[0, 15]], R))[0] < TOL_MAX_ABS


def test_forward_host_async_serving_loop(cuda_device):
    """Back-to-back submissions alternate staging slots; every output must be complete after host_wait()."""
    R, N = 64, 8
    g, sd = make_model(R, "tc")
    xs = [O.make_input(R, N, seed=40 + i).pin_memory() for i in range(5)]
    ys = [torch.empty(N, 3, R, R).pin_memory() for _ in range(5)]
    for x, y in zip(xs, ys):
        g.forward_host(x, out=y, wait=False)
    g.host_wait()
    for x, y in zip(xs, ys):
        assert torch.equal(y, g(x.to(cuda_device)).cpu())
    assert errs(ys[3][:2], O.generator_forward(sd, xs[3][:2], R))[0] < TOL_MAX_ABS


def test_tc_fast_mode_stated_accuracy(cuda_device):
    """path="tc_fast" = single fp16 tensor-core pass: NOT fp32-faithful (SURVEY F5 predicts ~1e-2 abs at
    output scale ~10); it must run and stay within its stated, looser bound."""
    R, N = 256, 2
    g, sd = make_model(R, "tc_fast")
    x = O.make_input(R, N, seed=11)
    want = O.generator_forward(sd, x, R)
    mx, mean = errs(g(x.to(cuda_device)), want)
    print("tc_fast R=%d max-abs=%.3e mean-abs=%.3e |y|max=%.2f" % (R, mx, mean, float(want.abs().max())))
    assert mx < 1e-1 and mean < 1e-2
    assert mx > 1e-4   # it really is the single-pass path


def test_from_img_mask(cuda_device):
    R = 64
    g, sd = make_model(R, "simt")
    gen = torch.Generator().manual_seed(1)
    img = torch.rand(1, 3, R, R, generator=gen) * 2 - 1
    mask = (torch.rand(1, 1, R, R, generator=gen) > 0.5).float()
    want = O.generator_forward(sd, torch.cat([mask - 0.5, img * mask], 1), R)
    assert errs(g.from_img_mask(img.to(cuda_device), mask.to(cuda_device)), want)[0] < TOL_MAX_ABS


def test_error_behaviour(cuda_device):
    R = 64
    g, _ = make_model(R, "simt")
    with pytest.raises(RuntimeError):
        g(torch.zeros(1, 4, R, R))                          # CPU tensor: no CPU path
    with pytest.raises(RuntimeError):
        g(torch.zeros(1, 4, R, R // 2, device=cuda_device))  # fixed resolution (SURVEY F9)
    with pytest.raises(RuntimeError):
        g(torch.zeros(1, 3, R, R, device=cuda_device))
    with pytest.raises(RuntimeError):
        g(torch.zeros(1, 4, R, R, device=cuda_device, dtype=torch.float16))
    sd = g.state_dict()
    sd["synthesis.b8.upsample.filter_const"] = torch.ones_like(sd["synthesis.b8.upsample.filter_const"])
    g.load_state_dict(sd)
    with pytest.raises(RuntimeError):                        # not the zero-insertion pattern
        g(torch.zeros(1, 4, R, R, device=cuda_device))


@pytest.mark.parametrize("path", PATHS)
def test_full_size_batch_properties(cuda_device, path):
    """BASELINE config sizes (migan-512, N=32): oracle on a 2-image sample + batch consistency."""
    R, N = 512, 32
    g, sd = make_model(R, path)
    x = O.make_input(R, N, seed=77)
    y = g(x.to(cuda_device))
    assert torch.isfinite(y).all()
    want = O.generator_forward(sd, x[[0, 31]], R)
    mx, mean = errs(y[[0, 31]], want)
    print("512/32 path=%s max-abs=%.3e mean-abs=%.3e" % (path, mx, mean))
    assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS
    y2 = g(x[16:].contiguous().to(cuda_device))              # same images, different batch slot
    assert torch.equal(y[16:], y2)


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("R", [8, 16, 32])
def test_small_resolutions(cuda_device, path, R):
    """R = 8 / 16 / 32 are valid constructor arguments (migan_inference.py:214-223): every level has 512 channels, the stem
    is 4 -> 512 and the top torgb runs un-fused.  Final output and every intermediate against the oracle."""
    N = 3
    g, sd = make_model(R, path)
    x = O.make_input(R, N, seed=13)
    taps = {}
    want = O.generator_forward(sd, x, R, taps=taps)
    xd = x.to(cuda_device)
    mx, mean = errs(g(xd), want)
    print("R=%d path=%s max-abs=%.3e mean-abs=%.3e" % (R, path, mx, mean))
    assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS
    bad = []
    for name, shape in g.tap_names():
        _, got = g.forward_with_tap(xd, name, shape)
        w = taps[name[: -len("_skip")]] + taps["feat%d" % shape[1]] if name.endswith("out_skip") else taps[name]
        e, _ = errs(got, w)
        if not (e < 2e-4 * max(float(w.abs().max()), 1.0)):
            bad.append((name, e))
    assert not bad, "first mismatching stages: %s" % bad[:5]


def test_migan256_batch32(cuda_device):
    """BASELINE.json configs[1] size (migan-256, 32 images, tensor-core path): oracle on a 3-image sample, finite everywhere,
    and image-by-image agreement with a different batch composition."""
    R, N = 256, 32
    g, sd = make_model(R, "tc")
    x = O.make_input(R, N, seed=91)
    y = g(x.to(cuda_device))
    assert torch.isfinite(y).all()
    pick = [0, 17, 31]
    mx, mean = errs(y[pick], O.generator_forward(sd, x[pick], R))
    print("256/32 tc max-abs=%.3e mean-abs=%.3e" % (mx, mean))
    assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS
    y2 = g(x[8:24].contiguous().to(cuda_device))
    assert torch.equal(y[8:24], y2)


def test_graph_replay_small_batches(cuda_device):
    """Batches <= graph_max_batch replay a captured CUDA graph of the forward (the demo's batch-1 latency path): same kernels,
    so bit-identical to the plain launch sequence; the graph follows weight reloads and batch-size changes."""
    R = 128
    g, sd = make_model(R, "tc")
    xs = [O.make_input(R, n, seed=60 + n).to(cuda_device) for n in (1, 2, 1, 3)]
    g.graph_max_batch = 0
    plain = [g(x) for x in xs]
    g.graph_max_batch = 4
    for _ in range(2):                                     # second round replays existing graphs / re-captures on a size change
        for x, want in zip(xs, plain):
            assert torch.equal(g(x), want)
    assert errs(plain[0], O.generator_forward(sd, xs[0].cpu(), R))[0] < TOL_MAX_ABS
    sd2 = O.make_state_dict(R, seed=5)
    g.load_state_dict(sd2)
    y = g(xs[1])                                           # new weights: the old graph must not be replayed
    assert errs(y, O.generator_forward(sd2, xs[1].cpu(), R))[0] < TOL_MAX_ABS
    name, shape = g.tap_names()[3]
    y_t, _ = g.forward_with_tap(xs[1], name, shape)        # taps fall back to the plain sequence
    assert torch.equal(y_t, y)
