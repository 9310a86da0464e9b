"""Stationary-A schedule of the fused SeparableConv2d kernel -- needs an H100.

A CTA tile of the tensor-core kernel covers one pixel tile and a group of N tiles: the depthwise prologue runs once
per pixel tile, and torgb is fused into the epilogue wherever the group holds all output channels.  These tests
check the resulting plan and walk every intermediate against the oracle at batch sizes where the group is narrower
than the layer (n = 1) and where it spans every N tile.
"""
import pytest
import torch

import migan_b200
from oracle import migan_oracle as O

pytestmark = pytest.mark.gpu


def make_model(R, path="tc", seed=1):
    sd = O.make_state_dict(R, seed=seed)
    g = migan_b200.Generator(R, path=path)
    g.load_state_dict(sd)
    return g.to("cuda:0").eval(), sd


def test_migan512_plan_fuses_torgb_at_wide_levels(cuda_device):
    R, N = 512, 32
    g, _ = make_model(R)
    x = O.make_input(R, N, seed=3).to(cuda_device)
    g.set_profiling(True)
    g(x)
    torch.cuda.synchronize()
    labels = [row[0] for row in g.profile_steps()]
    g.set_profiling(False)
    # the 128- and 256-channel levels now draw their image in the last conv's epilogue
    for r in (128, 256):
        assert "synthesis.b%d.torgb.torgb_img" % r not in labels
    assert g.last_launch_count() <= 51, labels


@pytest.mark.parametrize("R,N", [(256, 1), (256, 3), (128, 1), (128, 3), (64, 3)])
def test_every_intermediate_matches_oracle(cuda_device, R, N):
    g, sd = make_model(R)
    x = O.make_input(R, N, seed=7)
    taps = {}
    O.generator_forward(sd, x, R, taps=taps)
    xd = x.to(cuda_device)
    bad = []
    names = g.tap_names()
    assert len(names) > 20
    for name, shape in names:
        _, got = g.forward_with_tap(xd, name, shape)
        if name.endswith("out_skip"):
            want = taps[name[: -len("_skip")]] + taps["feat%d" % shape[1]]
        else:
            want = taps[name]
        scale = max(float(want.abs().max()), 1.0)
        mx = float((got.double().cpu() - want.double()).abs().max())
        if not (mx < 2e-4 * scale):
            bad.append((name, mx, scale))
    assert not bad, "first mismatching stages: %s" % bad[:5]
