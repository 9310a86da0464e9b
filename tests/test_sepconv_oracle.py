"""The references of the tensor-core SeparableConv2d kernel (oracle/sepconv_oracle.py) and the schedules its GPU test
reaches -- no GPU needed.

* The float64 operation reproduces the generator oracle's layer taps for every source.
* The exact model of the split arithmetic sees subtly wrong kernels: on every case of the GPU matrix, each wrong variant
  differs from the model by at least 20x the bound the GPU test allows.
* The GPU matrix reaches every schedule `plan_layout` can choose (planned without a device, at 114 and 132 SMs).
"""
import ctypes

import numpy as np
import pytest
import torch

from migan_b200 import _abi
from oracle import migan_oracle as O
from oracle import sepconv_oracle as S


def _layer_case(sd, p, source, x_shape, **kw):
    cin, cout = sd[p + "conv2.weight"].shape[1], sd[p + "conv2.weight"].shape[0]
    n, h, w = x_shape
    case = S.Case(source, n, h, w, cin, cout, **kw)
    t = case.t
    if source != S.SPLIT:
        t["dw_w"], t["dw_b"] = sd[p + "conv1.weight"], sd[p + "conv1.bias"]
    t["pw_w"] = sd[p + "conv2.weight"][:, :, 0, 0]
    return case


def _plane(noise, case):
    """[h][w] -> a [h + 2][noise_pitch] plane (zero padding)."""
    out = torch.zeros(case.h + 2, case.noise_pitch)
    out[: case.h, : case.w] = noise
    return out


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("R", [64, 256])
def test_op_reproduces_generator_layer_taps(R):
    """One STEM, NHWC, SPLIT and UP layer of the generator oracle, recomputed by sepconv_op from its inputs."""
    sd = O.make_state_dict(R, seed=3)
    x = O.make_input(R, 2, seed=5)
    taps = {}
    O.generator_forward(sd, x, R, taps=taps)
    checks = []
    # STEM: encoder.b{R}.conv1 on fromrgb(x)
    p = "encoder.b%d.conv1." % R
    c = _layer_case(sd, p, S.STEM, (2, R, R))
    c.t["x"] = x
    c.t["fromrgb_w"] = sd["encoder.b%d.fromrgb.weight" % R][:, :, 0, 0]
    c.t["fromrgb_b"] = sd["encoder.b%d.fromrgb.bias" % R]
    checks.append((c, taps[p + "out"], None))
    # NHWC: encoder.b4.conv1 on encoder.b8.conv2's output
    p = "encoder.b4.conv1."
    c = _layer_case(sd, p, S.NHWC, (2, 4, 4))
    c.t["in"] = _nhwc(taps["encoder.b8.conv2.out"])
    checks.append((c, taps[p + "out"], None))
    # SPLIT: encoder.b{R/2}.conv2's 1x1 conv on its down-sampled activation, pre-split as the down-sampling kernel does
    r = R // 2
    p = "encoder.b%d.conv2." % r
    down = taps[p + "down"]
    c = _layer_case(sd, p, S.SPLIT, (2, r // 2, r // 2))
    c.t["a_hi"], c.t["a_lo"] = S.split_trunc((_nhwc(down) * S.SPLIT_SCALE).numpy())
    checks.append((c, taps[p + "out"], None))
    # UP: synthesis.b{r}.conv2 rebuilt from conv1's raw 1x1 output, with both noise planes and the fused torgb + image
    r = R // 2
    p, p1 = "synthesis.b%d.conv2." % r, "synthesis.b%d.conv1." % r
    c = _layer_case(sd, p, S.UP, (2, r, r), noise=True, up_noise=True, torgb=True, img_lo=True)
    t = c.t
    t["in"] = _nhwc(taps["feat%d" % r])
    t["up_t"] = _nhwc(taps[p1 + "pw"])
    t["up_fir"] = sd[p1 + "upsample.filter.weight"][0, 0]
    t["up_noise"] = _plane(sd[p1 + "noise_const"] * sd[p1 + "noise_strength"], c)
    t["noise"] = _plane(sd[p + "noise_const"] * sd[p + "noise_strength"], c)
    q = "synthesis.b%d." % r
    t["rgb_w"], t["rgb_b"] = sd[q + "torgb.weight"][:, :, 0, 0], sd[q + "torgb.bias"]
    t["rgb_fir"] = sd[q + "upsample.filter.weight"][:, 0]
    t["img_lo"] = taps["synthesis.b%d.img" % (r // 2)]
    checks.append((c, taps[p + "out"], taps[q + "img"]))
    for case, want, want_img in checks:
        out, img = S.sepconv_op(case)
        scale = max(float(want.abs().max()), 1.0)
        assert float((out.permute(0, 3, 1, 2) - want.double()).abs().max()) < 1e-5 * scale, case.id
        if want_img is not None:
            assert float((img - want_img.double()).abs().max()) < 1e-5 * max(float(want_img.abs().max()), 1.0), case.id


@pytest.mark.parametrize("case", S.CASES, ids=lambda c: c.id)
def test_model_sees_wrong_kernels(case):
    """The exact model agrees with the float64 operation, and every applicable wrong variant differs from the model by
    at least 20x its bound somewhere."""
    m = S.sepconv_model(case)
    assert S.op_error(case, m["out"], m.get("img")) < S.OP_BOUND[case.passes] / 2
    for v in S.VARIANTS:
        if S.variant_applies(case, v):
            mv = S.sepconv_model(case, v)
            assert S.model_ratio(case, mv["out"], mv.get("img"), model=m) >= 20, v


def plan_only(lib, case, sms, candidate=-1):
    io = _abi.SepconvTcIO(source=case.source, n=case.n, h=case.h, w=case.w, cin=case.cin, cout=case.cout, act=case.act,
                          passes=case.passes, noise_pitch=case.noise_pitch, torgb=int(case.torgb),
                          store_out=case.store_out)
    plan = _abi.SepconvTcPlan()
    rc = lib.migan_debug_sepconv_tc(ctypes.byref(io), sms, candidate, ctypes.byref(plan), None)
    return plan.as_dict() if rc == 0 else None


def matrix_plans(lib, sms_list=(114, 132)):
    """Every plan the GPU matrix can launch: the production choice and each candidate that fits, per SM count."""
    recs = []
    for case in S.CASES:
        for sms in sms_list:
            first = plan_only(lib, case, sms)
            assert first is not None, (case.id, sms, lib.migan_last_error())
            recs.append((case, dict(first, sms=sms)))
            for i in range(first["num_candidates"]):
                r = plan_only(lib, case, sms, i)
                if r is not None:
                    recs.append((case, dict(r, sms=sms)))
    return recs


def test_plan_only_needs_no_device_and_refuses_what_does_not_fit(lib):
    case = S.CASES[0]
    first = plan_only(lib, case, 132)
    assert first["num_candidates"] > 0 and first["grid"] == min(first["num_tiles"], 132)
    assert plan_only(lib, case, 0) is None                              # plan-only needs an explicit SM count
    assert plan_only(lib, case, 132, first["num_candidates"]) is None   # past the candidate list
    # 512 input channels: no stationary A fits, so its candidates (listed first) are refused
    big = S.Case(S.NHWC, 4, 64, 64, 512, 512)
    r = plan_only(lib, big, 132)
    assert r["n_group"] == 1 and plan_only(lib, big, 132, 0) is None


def test_matrix_reaches_every_schedule(lib):
    recs = matrix_plans(lib)
    u = lambda key: {r[key] for _, r in recs}
    assert u("n_group") == {1, 2, 4, 8}
    assert u("in_stages") >= {2, 4, 6}
    stationary = {r["a_stages"] for _, r in recs if r["n_group"] > 1}
    plain = {r["a_stages"] for _, r in recs if r["n_group"] == 1}
    assert plain >= {2, 3, 4} and stationary                            # streamed A rings and a resident A
    assert {r["b_stages"] for _, r in recs if not r["b_resident"]} >= {2, 3} and 1 in u("b_resident")
    assert u("dw_global") == {0, 1}
    assert {(r["tile_w"], r["tile_h"], r["tile_n"]) for _, r in recs} >= {(16, 8, 1), (8, 8, 2), (4, 4, 8)}
    assert any(c.source == S.SPLIT and r["tile_h"] * r["tile_w"] == 128 and r["tile_w"] >= 32 for c, r in recs)
    assert u("n_tile") == {64, 128}
    assert any(c.w % r["tile_w"] for c, r in recs) and any(c.h % r["tile_h"] for c, r in recs)
    assert any(c.n % r["tile_n"] for c, r in recs)
    assert any(r["grid"] < r["num_tiles"] for _, r in recs)
