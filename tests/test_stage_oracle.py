"""The references of the CUDA-core stage kernels (oracle/stage_oracle.py) and the launches their GPU test reaches -- no GPU
needed.

* The float64 operations reproduce the generator oracle's intermediate taps.
* The exact model agrees with the float64 operation, and sees subtly wrong kernels: each wrong variant is at least 10x
  outside the model bound on some case of the matrix (a truncated fp16 hi fails the split-form check instead).
* The matrix reaches every (kernel, rows per thread, C / G template) that production forwards launch, at R = 8 .. 512 on
  both paths, at R x R and at the fully convolutional extents of the GPU suite; planned through `migan_debug_stage`
  without a device.
* The down-sampling taps of every filter the suite loads keep m = 0, so the tensor-core feed's tables are the fp32 taps.
"""
import ctypes

import numpy as np
import pytest
import torch

from migan_b200 import _abi
from oracle import migan_oracle as O
from oracle import stage_oracle as S

MODEL_CASES = [c for c in S.CASES if c.kind not in (S.NOISE_TILE, S.ADD)]


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def test_op_reproduces_generator_taps():
    """One launch of every kind, recomputed by stage_op from the generator oracle's own intermediates (R = 64)."""
    R = 64
    sd = O.make_state_dict(R, seed=3, fir="per_channel")
    x = O.make_input(R, 2, seed=5)
    taps = {}
    O.generator_forward(sd, x, R, taps=taps)
    checks = []
    p = "encoder.b64."
    c = S.Case(S.STEM, 2, R, R, 512)
    c.t.update({"in": x, "fromrgb_w": sd[p + "fromrgb.weight"][:, :, 0, 0], "fromrgb_b": sd[p + "fromrgb.bias"]})
    checks.append((c, _nhwc(taps[p + "fromrgb"])))
    c = S.Case(S.DW, 2, R, R, 512)
    c.t.update({"in": _nhwc(taps[p + "fromrgb"]), "dw_w": sd[p + "conv1.conv1.weight"], "dw_b": sd[p + "conv1.conv1.bias"]})
    checks.append((c, _nhwc(taps[p + "conv1.dw_act"])))
    c = S.Case(S.DOWN, 2, R, R, 512)
    c.t.update({"in": _nhwc(taps["feat64"]), "dw_w": sd[p + "conv2.conv1.weight"], "dw_b": sd[p + "conv2.conv1.bias"],
                "fir": sd[p + "conv2.downsample.filter.weight"]})
    checks.append((c, _nhwc(taps[p + "conv2.down"])))
    q = "synthesis.b32.conv1."
    c = S.Case(S.UP2, 2, 16, 16, 512, noise=True, skip=True)
    nz = torch.zeros(32, c.noise_pitch)
    nz[:, :32] = sd[q + "noise_const"] * sd[q + "noise_strength"]
    c.t.update({"in": _nhwc(taps[q + "pw"]), "fir": sd[q + "upsample.filter.weight"], "noise": nz,
                "skip": _nhwc(taps["feat32"])})
    checks.append((c, _nhwc(taps[q + "out"] + taps["feat32"])))
    q = "synthesis.b32."
    c = S.Case(S.TORGB, 2, 32, 32, 512, img_lo=True)
    c.t.update({"in": _nhwc(taps[q + "conv2.out"]), "rgb_w": sd[q + "torgb.weight"][:, :, 0, 0],
                "rgb_b": sd[q + "torgb.bias"], "fir": sd[q + "upsample.filter.weight"], "img_lo": taps["synthesis.b16.img"]})
    checks.append((c, taps[q + "img"]))
    for case, want in checks:
        got = S.stage_op(case)
        assert float((got - want.double()).abs().max()) < 1e-5 * max(float(want.abs().max()), 1.0), case.id


@pytest.mark.parametrize("case", MODEL_CASES, ids=lambda c: c.id)
def test_model_agrees_with_op(case):
    m = S.stage_model(case)
    assert bool(torch.isfinite(m["out"]).all()) and bool((m["bound"] > 0).all())
    assert S.op_error(case, m["out"]) < 1e-6, case.id
    if case.sat:   # the negative-lobe cases saturate both signs of the clamp instead
        want = (True, True) if case.fir != "lobes" else (True, False)
        assert S.saturation(case) == want, "the case must hit the clamp and the negative branch"


def test_model_sees_wrong_kernels():
    """Every wrong variant is >= 10x outside the model bound on some case it applies to."""
    for v in S.VARIANTS:
        cases = [c for c in MODEL_CASES if S.variant_applies(c, v)]
        assert cases, v
        worst = max(S.model_ratio(c, S.stage_model(c, v)["out"], S.stage_model(c)) for c in cases)
        assert worst >= 10, (v, worst)


def test_truncated_hi_fails_the_split_check():
    """A kernel that truncated its fp16 hi instead of rounding it to nearest: hi + lo can still be exact, so the model
    bound does not see it, but |lo| > ulp(hi) / 2 does."""
    seen = False
    for c in MODEL_CASES:
        if c.kind != S.DOWN or c.form == S.F32:
            continue
        s = S.stage_model(c)["out"].numpy().astype(np.float32)
        hi, lo = S.split_f16(s, 1.0)
        assert S.split_is_nearest(hi, lo), c.id
        hi_t = s.astype(np.float16)
        toward = np.abs(hi_t.astype(np.float32)) > np.abs(s)      # rounded away from zero: step back one fp16
        hi_t[toward] = np.nextafter(hi_t[toward], np.float16(0))
        lo_t = (s - hi_t.astype(np.float32)).astype(np.float16)
        seen |= not S.split_is_nearest(hi_t, lo_t)
    assert seen


def test_fir_shift_keeps_every_suite_filter_unscaled():
    """m = 0 -- the tensor-core feed's taps equal the fp32 taps -- for every filter the suite loads; the negative-lobe
    filter (sum |f| = 9) gets m = 3."""
    for R in (8, 64, 256, 512):
        for fir in O.FIR_MODES:
            sd = O.make_state_dict(R, seed=1, fir=fir)
            for k, v in sd.items():
                if k.endswith("downsample.filter.weight"):
                    assert S.fir_shift(v) == 0, (R, fir, k)
    assert S.fir_shift(torch.outer(S.LOBES, S.LOBES)) == 3
    assert S.fir_shift(torch.full((4, 4), 2.0 / 16)) == 0 and S.fir_shift(torch.full((4, 4), 2.01 / 16)) == 1


# ---- coverage of what production forwards launch -----------------------------------------------------------------------
def plan(lib, kind, n, h, w, c, variant=S.AUTO, tc=0, level=0, **kw):
    io = _abi.StageIO(kind=kind, n=n, h=h, w=w, c=c, tc=tc, level=level, **kw)
    rec = _abi.StagePlan()
    rc = lib.migan_debug_stage(ctypes.byref(io), variant, ctypes.byref(rec), None)
    return rec.as_dict() if rc == 0 else None


def _key(rec):
    name = S.KIND_NAMES[rec["kind"]] + ("_" + S.FORM_NAMES[rec["down_form"]] if rec["kind"] == S.DOWN else "")
    return name, rec["rs"], rec["cg"]


# extents of the fully convolutional forwards the GPU suite runs (test_fullconv_gpu.py, test_fir_gpu.py)
FC_EXTENTS = {128: [(160, 224)], 256: [(256, 384), (320, 256), (640, 320), (320, 448)],
              512: [(512, 768), (640, 896), (1024, 1536), (768, 512)]}


def production_launches(lib, R, tc, H, W, n=1, uniform_up=True):
    """The stage launches of one forward, as PlanBuilder emits them (migan_abi.cu), each planned by the hook: the layer
    list is restated here; which kernel, rows per thread and template run is the library's choice."""
    ch = O.channels
    ext = lambda r: (H * r // R, W * r // R)
    steps = []
    if (H, W) != (R, R):
        steps.append((S.NOISE_TILE, dict(n=1, h=H, w=W, c=4, r=R, noise_pitch=(W + 3) // 4 * 4)))
    if not (tc and R >= 16 and ch(R) < 512):
        steps.append((S.STEM, dict(n=n, h=H, w=W, c=ch(R))))
    for r in O.encode_res(R):
        h, w = ext(r)
        if not tc or (ch(r) >= 512 and r >= 64):               # conv1: its own depthwise kernel
            steps.append((S.DW, dict(n=n, h=h, w=w, c=ch(r))))
        if r > 4:                                              # conv2 down-samples
            steps.append((S.DOWN, dict(n=n, h=h, w=w, c=ch(r), tc=int(tc), level=r // 2)))
        elif not tc:
            steps.append((S.DW, dict(n=n, h=h, w=w, c=ch(r))))
    for r in O.block_res(R):
        h, w = ext(r)
        if r == 4:
            if not tc:
                steps.append((S.DW, dict(n=n, h=h, w=w, c=ch(4))))
            steps.append((S.ADD, dict(n=n, h=h, w=w, c=ch(4))))
        else:
            lh, lw = ext(r // 2)
            if not tc:
                steps.append((S.DW, dict(n=n, h=lh, w=lw, c=ch(r // 2))))
            if not (tc and uniform_up and r >= 16 and ch(r) < 512):
                steps.append((S.UP2, dict(n=n, h=lh, w=lw, c=ch(r))))
        if not tc or (ch(r) >= 512 and r >= 64):                # conv2 (torgb is not fused at 512 channels)
            steps.append((S.DW, dict(n=n, h=h, w=w, c=ch(r))))
        if not tc or ch(r) >= 512:
            steps.append((S.TORGB, dict(n=n, h=h, w=w, c=ch(r))))
    recs = []
    for kind, kw in steps:
        rec = plan(lib, kind, **kw)
        assert rec is not None, (R, tc, H, W, kind, kw, lib.migan_last_error())
        recs.append(rec)
    return recs


def matrix_launches(lib):
    out = {}
    for c in S.CASES:
        kw = dict(n=c.n, h=c.h, w=c.w, c=c.c)
        if c.kind == S.NOISE_TILE:
            kw.update(c=4, r=c.r, noise_pitch=c.noise_pitch)
        rec = plan(lib, c.kind, variant=c.form if c.kind == S.DOWN else S.AUTO, **kw)
        assert rec is not None, (c.id, lib.migan_last_error())
        out[c.id] = rec
    return out


def test_plan_only_needs_no_device_and_refuses_what_no_instance_runs(lib):
    rec = plan(lib, S.DOWN, 1, 32, 32, 512, S.TMA)
    assert rec == {"kind": S.DOWN, "down_form": S.TMA, "rs": 8, "cg": 0, "grid": 2 * 1 * 8, "groups": 1, "fir_shift": 0}
    assert plan(lib, S.DOWN, 1, 16, 32, 512, S.TMA)["rs"] == 8
    assert plan(lib, S.DOWN, 1, 14, 32, 512, S.TMA) is None          # H2 < 8 would need 4-row strips: no such instance
    assert plan(lib, S.DOWN, 1, 32, 30, 512, S.TMA) is None          # odd W2
    assert plan(lib, S.DOWN, 1, 16, 16, 256, S.SPLIT) is None        # the split kernel has C = 512 only
    assert plan(lib, S.DOWN, 1, 16, 16, 512, S.SPLIT)["cg"] == 512
    assert plan(lib, S.DOWN, 1, 16, 16, 512, S.AUTO, tc=1, level=8)["down_form"] == S.SPLIT
    assert plan(lib, S.DOWN, 1, 32, 32, 256, S.AUTO, tc=1, level=16)["down_form"] == S.TMA
    assert plan(lib, S.DOWN, 1, 32, 32, 256, S.AUTO, tc=0, level=16)["down_form"] == S.F32
    assert plan(lib, S.DOWN, 1, 16, 16, 512, 3) is None
    assert plan(lib, S.STEM, 1, 5, 7, 64) is None                    # H * W not a multiple of 4
    assert plan(lib, 7, 1, 4, 4, 64) is None


def test_matrix_reaches_every_production_launch(lib):
    prod = {}
    for R in (8, 16, 32, 64, 128, 256, 512):
        for tc in (False, True):
            for H, W in [(R, R)] + FC_EXTENTS.get(R, []):
                for uniform in (True, False):
                    for rec in production_launches(lib, R, tc, H, W, uniform_up=uniform):
                        prod.setdefault(_key(rec), set()).add(rec["groups"])
    mat = {}
    for rec in matrix_launches(lib).values():
        mat.setdefault(_key(rec), set()).add(rec["groups"])
    assert set(prod) == set(mat), ("production only", set(prod) - set(mat), "matrix only", set(mat) - set(prod))
    for k in prod:
        assert prod[k] <= mat[k], k
    # what item the deleted instances were: nothing production launches needs them
    assert not any(k[0] == "down_tma" and k[1] == 4 for k in prod)
    assert {k[2] for k in prod if k[0] == "down_split"} == {512}
