"""The generator with asymmetric, per-channel FIR taps -- needs an H100, except the sensitivity check at the end.

The `*.filter.weight` taps are parameters of the reference (migan_inference.py:72, :96), so a trained checkpoint may carry
any values there.  The constructor's [1,3,3,1] filter is symmetric, separable and the same for every channel, so it cannot
show a kernel that flips the taps, swaps their axes or reads one channel's taps for every channel.  These tests load
asymmetric taps (`make_state_dict(..., fir="uniform" | "per_channel")`) and compare with the float64 oracle.

Which kernels see the taps depends on the plan.  Up-sampling taps that are the same for every channel go to the tensor-core
kernel's fused UP prologue at the levels r >= 16 with fewer than 512 channels (R >= 128 only); taps that differ between
channels send those levels through `up2_noise_act_skip` and an NHWC-source `sepconv_tc` launch instead.  R = 64 (every
level 512 channels) covers the unfused kernels, R = 256 (levels 128 and 256) the fused ones, and the plan labels confirm
which branch ran.

Bounds are those of test_generator_gpu.py: max-abs < 1e-3 and mean-abs < 1e-4 on outputs for the fp32-faithful paths,
2e-4 * scale per intermediate.
"""
import gc
import os

import numpy as np
import pytest
import torch

import migan_b200
from oracle import fullconv_oracle as FC
from oracle import migan_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden", "fir.npz")
PATHS = ["simt", "tc"]
TOL_MAX_ABS = 1e-3
TOL_MEAN_ABS = 1e-4
WSEED = 1

# (R, n, H, W, fir, input seed) of every oracle comparison below; the CPU sensitivity check runs on the same list
INTERMEDIATE_CASES = [(R, n, R, R, fir, 5 + n) for R in (64, 256) for n in (1, 3) for fir in ("uniform", "per_channel")]
FC_CASES = [(256, 2, 320, 448, "per_channel", 21), (512, 1, 640, 896, "per_channel", 22)]
BIG_CASE = (512, 32, 512, 512, "per_channel", 77)
ODD_CASE = (256, 2, 256, 256, "odd_channel", 31)
RELOAD_CASES = [(256, n, H, W, fir, 40 + n) for fir in ("constructor", "per_channel", "uniform")
                for n, H, W in ((2, 256, 256), (6, 256, 256), (1, 320, 448))]


def state_dict(R, fir):
    """make_state_dict's modes, plus "odd_channel": the uniform taps with the last channel's filter flipped, so only one
    channel differs from the others."""
    if fir != "odd_channel":
        return O.make_state_dict(R, seed=WSEED, fir=fir)
    sd = O.make_state_dict(R, seed=WSEED, fir="uniform")
    for k in sd:
        if k.endswith("filter.weight"):
            sd[k][-1] = sd[k][-1].flip([1, 2])
    return sd


_models = {}
_oracle = {}


def make_model(R, path, fir):
    key = (R, path, fir)
    if key not in _models:
        g = migan_b200.Generator(R, path=path)
        g.load_state_dict(state_dict(R, fir))
        _models[key] = g.to("cuda:0").eval()
    return _models[key]


def release_models():
    _models.clear()
    gc.collect()
    torch.cuda.empty_cache()


def oracle(case, pick=None, taps=None):
    """float64 oracle output of a case (images `pick` only); with `taps`, also fills the intermediates (not cached)."""
    R, n, H, W, fir, seed = case
    key = case + (tuple(pick) if pick is not None else None,)
    if taps is None and key in _oracle:
        return _oracle[key]
    x = FC.make_input_hw(R, n, H, W, seed)
    if pick is not None:
        x = x[pick]
    y = FC.generator_forward_fc(state_dict(R, fir), x, R, taps=taps, dtype=torch.float64)
    if taps is None:
        _oracle[key] = y
    return y


def errs(got, want):
    d = (got.double().cpu() - want.double()).abs()
    return float(d.max()), float(d.mean())


def run(g, x):
    R = g.resolution
    return g(x) if tuple(x.shape[2:]) == (R, R) else g.forward_fc(x)


def plan_labels(g, x):
    """Kernel labels of the plan the forward of x runs (the plain launch sequence: profiling bypasses the graph)."""
    g.set_profiling(True)
    try:
        run(g, x)
        torch.cuda.synchronize()
        return [row[0] for row in g.profile_steps()]
    finally:
        g.set_profiling(False)


def fused_up_levels(R, path, fir):
    """Levels whose conv1 FIR runs in the fused UP prologue rather than in up2_noise_act_skip: {128, 256} at R = 256 on the
    tensor-core path with channel-uniform taps, none at R = 64."""
    if path == "simt" or fir in ("per_channel", "odd_channel"):
        return set()
    return {r for r in O.block_res(R)[1:] if r >= 16 and O.channels(r) < 512}


def check_plan(labels, R, path, fir):
    """conv1's FIR runs where fused_up_levels says, and on the tensor-core path the 128- and 256-channel levels draw their
    image in conv2's epilogue whatever the taps (with an NHWC source when conv1 runs up2), so the fused torgb reads its
    [16][3] table with three different per-colour filters under per_channel taps."""
    fused = fused_up_levels(R, path, fir)
    for r in O.block_res(R)[1:]:
        up2 = "synthesis.b%d.conv1.up2_noise_act_skip" % r in labels
        assert up2 == (r not in fused), (r, path, fir, labels)
        rgb_kernel = "synthesis.b%d.torgb.torgb_img" % r in labels
        if path == "simt":
            assert rgb_kernel, (r, path, fir, labels)
        elif r in (128, 256):
            assert not rgb_kernel, (r, path, fir, labels)


def walk_taps(g, xd, taps, fc):
    """Every intermediate the plan exposes against the oracle's; returns the failures."""
    R = g.resolution
    n, _, H, W = xd.shape
    bad = []
    names = g.tap_names()
    assert len(names) > 20
    for name, (c, h, w) in names:
        if fc:
            _, got = g.forward_fc(xd, tap=name)
        else:
            _, got = g.forward_with_tap(xd, name, (c, h, w))
        assert tuple(got.shape) == (n, c, h * H // R, w * W // R), name
        if name.endswith("out_skip"):
            want = taps[name[: -len("_skip")]] + taps["feat%d" % h]
        else:
            want = taps[name]
        scale = max(float(want.abs().max()), 1.0)
        mx, _ = errs(got, want)
        if not (mx < 2e-4 * scale):
            bad.append((name, mx, scale))
    return bad


# ---- the reference's own outputs ---------------------------------------------------------------------------------------------
def _fixture_cases():
    return list(range(int(np.load(GOLD)["num_cases"])))


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS + ["tc_fast"])
@pytest.mark.parametrize("case", _fixture_cases())
def test_reference_fixture(cuda_device, path, case):
    """Outputs the reference itself computed with asymmetric taps (make_golden_fir.py), on the rows the fixture keeps."""
    z = np.load(GOLD)
    R, N, H, W, wseed, xseed = [int(v) for v in z["case%d_meta" % case]]
    assert wseed == WSEED
    g = make_model(R, path, str(z["case%d_fir" % case]))
    got = run(g, FC.make_input_hw(R, N, H, W, xseed).to(cuda_device))
    assert got.shape == (N, 3, H, W)
    rows = torch.from_numpy(z["case%d_rows" % case]).to(cuda_device)
    mx, mean = errs(got[:, :, rows], torch.from_numpy(z["case%d_y" % case]))
    print("fir fixture %d R=%d %dx%d n=%d %s path=%s max-abs=%.3e mean-abs=%.3e"
          % (case, R, H, W, N, z["case%d_fir" % case], path, mx, mean))
    if path == "tc_fast":
        # Single fp16 pass, stated as ~1e-2 (DESIGN.md).  Measured on an H100 80GB HBM3 at a 400 W power limit: mean-abs
        # 2.5e-3 .. 1.1e-2 on these cases, about 470x the 3-pass path's error on each (fused and unfused levels alike), so
        # the spread is the fp16 pass, not the taps.  Wrong taps in any one group of filters move the output by at least
        # 0.17 max-abs and 0.03 mean-abs (test_oracle_sees_wrong_taps), so this bound still sees them.
        assert mx < 1e-1 and mean < 2e-2
        assert mx > 1e-4   # it really is the single-pass path
    else:
        assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS


# ---- every intermediate, fixed resolution --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("case", INTERMEDIATE_CASES, ids=lambda c: "R%d-n%d-%s" % (c[0], c[1], c[4]))
def test_every_intermediate_matches_oracle(cuda_device, path, case):
    """n = 1 and n = 3 give different stationary-A groups in the tensor-core kernel."""
    R, n, H, W, fir, seed = case
    g = make_model(R, path, fir)
    xd = FC.make_input_hw(R, n, H, W, seed).to(cuda_device)
    check_plan(plan_labels(g, xd), R, path, fir)
    taps = {}
    want = oracle(case, taps=taps)
    mx, mean = errs(g(xd), want)
    print("R=%d n=%d %s path=%s max-abs=%.3e mean-abs=%.3e (|y|max=%.2f)" % (R, n, fir, path, mx, mean, float(want.abs().max())))
    assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS
    bad = walk_taps(g, xd, taps, fc=False)
    assert not bad, "first mismatching stages: %s" % bad[:5]


# ---- the fully convolutional forward: partial tiles under up2 and the down-samplers -------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("case", FC_CASES, ids=lambda c: "R%d-%dx%d" % (c[0], c[2], c[3]))
def test_forward_fc_per_channel(cuda_device, path, case):
    R, n, H, W, fir, seed = case
    g = make_model(R, path, fir)
    xd = FC.make_input_hw(R, n, H, W, seed).to(cuda_device)
    check_plan(plan_labels(g, xd), R, path, fir)
    taps = {}
    want = oracle(case, taps=taps)
    mx, mean = errs(g.forward_fc(xd), want)
    print("fc R=%d %dx%d n=%d %s path=%s max-abs=%.3e mean-abs=%.3e" % (R, H, W, n, fir, path, mx, mean))
    assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS
    bad = walk_taps(g, xd, taps, fc=True)
    assert not bad, "first mismatching stages: %s" % bad[:5]


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_migan512_batch32_per_channel(cuda_device, path):
    release_models()                       # the n = 32 workspace is large
    R, n, H, W, fir, seed = BIG_CASE
    g = make_model(R, path, fir)
    xd = FC.make_input_hw(R, n, H, W, seed).to(cuda_device)
    y = g(xd)
    assert torch.isfinite(y).all()
    mx, mean = errs(y[[0, 31]], oracle(BIG_CASE, pick=[0, 31]))
    print("512/32 per_channel path=%s max-abs=%.3e mean-abs=%.3e" % (path, mx, mean))
    assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS
    check_plan(plan_labels(g, xd), R, path, fir)
    release_models()


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_one_odd_channel_is_not_uniform(cuda_device, path):
    """Taps equal for every channel but the last: the uniformity scan must see the last channel and keep up2."""
    R, n, H, W, fir, seed = ODD_CASE
    g = make_model(R, path, fir)
    xd = FC.make_input_hw(R, n, H, W, seed).to(cuda_device)
    check_plan(plan_labels(g, xd), R, path, fir)
    mx, mean = errs(g(xd), oracle(ODD_CASE))
    print("odd channel path=%s max-abs=%.3e mean-abs=%.3e" % (path, mx, mean))
    assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS


# ---- weight reloads that flip the fusion decision ------------------------------------------------------------------------------
@pytest.mark.gpu
def test_reload_across_the_fusion_decision(cuda_device):
    """One R = 256 Generator with fixed shapes: n = 2 (the captured CUDA graph), n = 6 (the plain launch sequence) and
    forward_fc at 320 x 448.  Loading per-channel taps, then uniform taps, must rebuild every cached plan and graph: each
    call matches the oracle of the weights loaded, and the plan labels and tap names follow the new fusion decision.

    Each round ends with an n = 2 forward that replays the captured graph, and the next round starts with the same call on
    the same workspace, so nothing but the weight load can retire that graph (profiling, taps and other batch sizes all
    do).  A graph kept across the constructor -> per-channel load would replay the fused UP prologue with the old taps,
    which its kernel parameters hold by value, and miss the oracle."""
    R = 256
    g = migan_b200.Generator(R, path="tc").to(cuda_device).eval()
    assert 2 <= g.graph_max_batch < 6
    xs = {}
    for case in RELOAD_CASES:
        _, n, H, W, _, seed = case
        xs[(n, H, W)] = FC.make_input_hw(R, n, H, W, seed).to(cuda_device)
    x2 = xs[(2, 256, 256)]

    def graph_forward(case):
        """Two n = 2 forwards, each against the oracle: the first captures a graph if none is current, the second replays it."""
        ws = None
        for _ in range(2):
            mx, mean = errs(g(x2), oracle(case))
            print("reload %s n=2 graph max-abs=%.3e mean-abs=%.3e" % (case[4], mx, mean))
            assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS, case
            w = g._engine(x2.device).workspaces[(2, "graph")]
            assert ws is None or w.data_ptr() == ws, "the graph workspace moved between the two calls"
            ws = w.data_ptr()
        return ws

    prev_labels = {}
    graph_ws = None
    for fir in ("constructor", "per_channel", "uniform"):
        g.load_state_dict(state_dict(R, fir))
        case2 = [c for c in RELOAD_CASES if c[4] == fir and c[1] == 2][0]
        # first call after the load: the n = 2 graph call on the workspace the previous round's graph was captured for
        ws = graph_forward(case2)
        assert graph_ws is None or ws == graph_ws
        for case in [c for c in RELOAD_CASES if c[4] == fir]:
            _, n, H, W, _, _ = case
            x = xs[(n, H, W)]
            if n != 2:
                for _ in range(2):
                    mx, mean = errs(run(g, x), oracle(case))
                    print("reload %s n=%d %dx%d max-abs=%.3e mean-abs=%.3e" % (fir, n, H, W, mx, mean))
                    assert mx < TOL_MAX_ABS and mean < TOL_MEAN_ABS, (fir, n, H, W)
            labels = plan_labels(g, x)
            check_plan(labels, R, "tc", fir)
            if (n, H, W) in prev_labels:
                assert labels != prev_labels[(n, H, W)], (fir, n, H, W)
            prev_labels[(n, H, W)] = labels
        # the tap list follows the plan: conv1's up-sampled output exists only where up2 runs
        names = dict(g.tap_names())
        unfused = not fused_up_levels(R, "tc", fir)
        assert ("synthesis.b128.conv1.out_skip" in names) == unfused, fir
        taps = {}
        oracle(case2, taps=taps)
        for name in ("synthesis.b128.conv1.out_skip", "synthesis.b128.conv1.pw"):
            if name in names:
                _, got = g.forward_with_tap(x2, name, names[name])
                want = taps[name] if name.endswith("pw") else taps["synthesis.b128.conv1.out"] + taps["feat128"]
                assert errs(got, want)[0] < 2e-4 * max(float(want.abs().max()), 1.0), (fir, name)
        # last calls before the next load: capture a graph for these weights and replay it, with no profiling or tap after
        graph_ws = graph_forward(case2)


# ---- CPU: the inputs above can see the mistakes the constructor's filter hides ------------------------------------------------
FILTER_GROUPS = {"down": "downsample.filter.weight", "up": "conv1.upsample.filter.weight"}
MUTATIONS = {"flip": lambda f: f.flip([2, 3]), "transpose": lambda f: f.transpose(2, 3).contiguous(),
             "channel0": lambda f: f[:1].expand_as(f).contiguous()}
_unmutated = {}


def _sensitivity_cases():
    """Every weight / input pair compared with the oracle above (image 0 of each batch)."""
    cases = INTERMEDIATE_CASES + FC_CASES + [BIG_CASE, ODD_CASE]
    out = []
    for R, n, H, W, fir, seed in cases:
        for group in ("down", "up", "torgb"):
            for m in MUTATIONS:
                if m == "channel0" and fir != "per_channel":
                    continue   # uniform taps: channel 0's filter is every channel's
                out.append(pytest.param((R, n, H, W, fir, seed), group, m, id="R%d-n%d-%dx%d-%s-%s-%s" % (R, n, H, W, fir, group, m)))
    return out


@pytest.mark.parametrize("case,group,mutation", _sensitivity_cases())
def test_oracle_sees_wrong_taps(case, group, mutation):
    """A kernel that convolves instead of correlating (flipped taps), swaps the tap axes, or reads channel 0's taps for
    every channel, in any one group of filters, moves the output by more than 100x the bounds the GPU tests use.  This keeps
    the seeds above able to show such a bug."""
    R, n, H, W, fir, seed = case
    sd = state_dict(R, fir)
    x = FC.make_input_hw(R, n, H, W, seed)[:1]
    if case not in _unmutated:
        _unmutated[case] = FC.generator_forward_fc(sd, x, R)
    want = _unmutated[case]
    bad = dict(sd)
    hit = 0
    for k, v in sd.items():
        if not k.endswith("filter.weight"):
            continue
        is_torgb = k.startswith("synthesis.") and k.split(".")[2] == "upsample"
        if (group == "torgb" and is_torgb) or (group != "torgb" and k.endswith(FILTER_GROUPS[group])):
            bad[k] = MUTATIONS[mutation](v)
            hit += 1
    assert hit > 0
    mx, mean = errs(FC.generator_forward_fc(bad, x, R), want)
    print("%s %s: max-abs %.3f mean-abs %.4f" % (group, mutation, mx, mean))
    assert mx > 100 * TOL_MAX_ABS and mean > 100 * TOL_MEAN_ABS, (mx, mean)
