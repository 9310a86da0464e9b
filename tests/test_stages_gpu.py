"""The CUDA-core stage kernels of the forward on their own, one launch at a time -- needs an H100.

Each case of the matrix (oracle/stage_oracle.py CASES) runs through the test hook `migan_debug_stage`:
  a. against the exact model of the kernel's fp32 chain (tight bound) and the float64 operation (contract bound), or
     byte for byte where the arithmetic allows it (noise_tile, add_inplace, the DW split output, hi nearest to hi + lo);
  b. outputs in 64 KB sentinel guard bands; inputs between NaN guard bands and noise planes with NaN in their pitch
     padding, so a read outside a tensor shows up as a non-finite output;
  c. the launched plan equals the plan-only record, two launches give the same bytes, and image i's bytes do not depend on
     the batch it is launched in;
  d. dw3x3_down_split and dw3x3_down_tma give byte-identical hi / lo on every shape both accept.
Then the generator with negative-lobe down-sampling taps on saturated inputs, on both paths.
"""
import ctypes
import time

import numpy as np
import pytest
import torch

import migan_b200
from migan_b200 import _abi
from oracle import fullconv_oracle as FC
from oracle import migan_oracle as O
from oracle import stage_oracle as S

pytestmark = pytest.mark.gpu

GUARD = 16384                      # 4-byte words (64 KB) of guard band before and after each buffer
SENTINEL = 0x7FC0DEAD              # a NaN bit pattern no kernel writes
STATS = {"launches": 0}
T0 = time.time()


def _guarded_out(nbytes):
    words = (nbytes + 3) // 4
    buf = torch.full((GUARD + words + GUARD,), SENTINEL, dtype=torch.int32, device="cuda:0")
    return buf, buf[GUARD: GUARD + words]


def _guarded_in(t):
    """A device copy of t between NaN guard bands."""
    t = torch.as_tensor(t).float().contiguous().reshape(-1)
    buf = torch.full((GUARD + t.numel() + GUARD,), float("nan"), device="cuda:0")
    buf[GUARD: GUARD + t.numel()] = t.to("cuda:0")
    return buf, buf[GUARD: GUARD + t.numel()]


class Launch:
    """Device copies of a case's operands (images [i0, i0 + n) of it); run() launches once."""

    def __init__(self, case, variant=None, images=None):
        self.case = S.make_case(case)
        c, t = self.case, self.case.t
        self.variant = c.form if variant is None else variant
        self.images = images
        n = c.n if images is None else len(images)
        self.n = n
        self.keep = []
        io = _abi.StageIO(kind=c.kind, n=n, h=c.h, w=c.w, c=c.c if c.kind != S.NOISE_TILE else 4, r=c.r,
                          noise_pitch=c.noise_pitch)
        for name, field in (("in", "in_"), ("dw_w", "dw_w"), ("dw_b", "dw_b"), ("fir", "fir"), ("fromrgb_w", "fromrgb_w"),
                            ("fromrgb_b", "fromrgb_b"), ("rgb_w", "rgb_w"), ("rgb_b", "rgb_b"), ("img_lo", "img_lo"),
                            ("noise", "noise"), ("skip", "skip")):
            if name not in t:
                continue
            v = t[name]
            if images is not None and name in ("in", "img_lo", "skip") and c.kind != S.NOISE_TILE:
                v = v[images]
            if name == "noise":
                v = v.clone()
                v[:, 2 * c.w:] = float("nan")
            buf, d = _guarded_in(v)
            self.keep.append(buf)
            setattr(io, field, d.data_ptr())
        self.io = io

    def out_bytes(self):
        c = self.case
        shape = list(c.out_shape())
        if c.kind not in (S.NOISE_TILE,):
            shape[0] = self.n
        return int(np.prod(shape)), shape

    def run(self, lib):
        c = self.case
        numel, shape = self.out_bytes()
        split = c.kind == S.DOWN and self.variant != S.F32
        bufs = {}
        if not split:
            bufs["out"] = _guarded_out(4 * numel)
            if c.kind == S.ADD:    # added to in place
                src = c.t["out"] if self.images is None else c.t["out"][self.images]
                bufs["out"][1].copy_(src.reshape(-1).view(torch.int32).to("cuda:0"))
            self.io.out = bufs["out"][1].data_ptr()
        if split or (c.kind == S.DW and c.form == S.SPLIT):
            bufs["hi"], bufs["lo"] = _guarded_out(2 * numel), _guarded_out(2 * numel)
            self.io.out_hi, self.io.out_lo = bufs["hi"][1].data_ptr(), bufs["lo"][1].data_ptr()
        rec = _abi.StagePlan()
        rc = lib.migan_debug_stage(ctypes.byref(self.io), self.variant, ctypes.byref(rec),
                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc == _abi.ERR_INVALID and split:
            return None
        assert rc == 0, (c.id, lib.migan_last_error())
        STATS["launches"] += 1
        torch.cuda.synchronize()
        res = {"plan": rec.as_dict()}
        for k, (buf, body) in bufs.items():
            s = buf.cpu()
            assert bool((s[:GUARD] == SENTINEL).all()) and bool((s[-GUARD:] == SENTINEL).all()), (c.id, k, "guard band written")
            raw = body.cpu()
            if k == "out":
                res[k] = raw.view(torch.float32)[:numel].reshape(shape)
            else:
                res[k] = raw.view(torch.int16)[:numel].numpy().view(np.float16).reshape(shape)
        return res


def _bytes(res):
    return {k: (v.numpy().tobytes() if isinstance(v, torch.Tensor) else v.tobytes()) for k, v in res.items() if k != "plan"}


def _plan_only(lib, L):
    io = _abi.StageIO(**{f: getattr(L.io, f) for f, _ in _abi.StageIO._fields_ if f in ("kind", "n", "h", "w", "c", "r",
                                                                                    "noise_pitch")})
    rec = _abi.StagePlan()
    _abi.check(lib.migan_debug_stage(ctypes.byref(io), L.variant, ctypes.byref(rec), None))
    return rec.as_dict()


def check_values(case, res):
    """Bounds and bitwise properties of one launch; returns (model ratio, contract error) or None (bitwise kinds)."""
    if case.kind == S.NOISE_TILE:
        assert res["out"].numpy().tobytes() == S.tile_noise(case).tobytes(), case.id
        return None
    if case.kind == S.ADD:
        want = (case.t["out"].numpy() + case.t["in"].numpy()).astype(np.float32)
        assert res["out"].numpy().tobytes() == want.tobytes(), case.id
        return None
    split = case.kind == S.DOWN and case.form != S.F32
    if split:
        assert np.isfinite(res["hi"]).all() and np.isfinite(res["lo"]).all(), (case.id, "non-finite split operand")
        assert S.split_is_nearest(res["hi"], res["lo"]), case.id
        got = S.kernel_value(case, hi=res["hi"], lo=res["lo"])
    else:
        assert bool(torch.isfinite(res["out"]).all()), (case.id, "non-finite output: NaN padding read?")
        got = res["out"]
        if case.kind == S.DW and case.form == S.SPLIT:   # the split is numpy's split of the fp32 output, byte for byte
            hi, lo = S.split_f16(res["out"].numpy(), S.SPLIT_SCALE)
            assert hi.tobytes() == res["hi"].tobytes() and lo.tobytes() == res["lo"].tobytes(), case.id
    r, e = S.model_ratio(case, got), S.op_error(case, got)
    key = case.name
    m, o = STATS.setdefault("model", {}), STATS.setdefault("op", {})
    m[key], o[key] = max(m.get(key, 0.0), r), max(o.get(key, 0.0), e)
    assert r <= 1.0, (case.id, "outside the model bound", r)
    assert e < S.OP_BOUND[key], (case.id, "outside the contract bound", e)
    return r, e


@pytest.mark.parametrize("case", S.CASES, ids=lambda c: c.id)
def test_launch(lib, cuda_device, case):
    L = Launch(case)
    res = L.run(lib)
    assert res is not None, case.id
    dry = _plan_only(lib, L)
    assert dict(res["plan"], fir_shift=0) == dry, case.id    # a plan-only call has no taps to derive the shift from
    out = check_values(case, res)
    if case.kind == S.DOWN:
        assert res["plan"]["fir_shift"] == S.fir_shift(case.t["fir"]), case.id
    print("\n%s: %s%s" % (case.id, res["plan"], "" if out is None else ", model ratio %.3f, float64 error %.2e" % out))
    # two launches, and each image launched on its own: the same bytes
    assert _bytes(L.run(lib)) == _bytes(res), case.id
    if case.n > 1 and case.kind != S.NOISE_TILE:
        for i in range(case.n):
            one = Launch(case, images=[i]).run(lib)
            for k, v in _bytes(one).items():
                whole = res[k][i]
                assert v == (whole.numpy().tobytes() if isinstance(whole, torch.Tensor) else whole.tobytes()), (case.id, i, k)


@pytest.mark.parametrize("case", [c for c in S.CASES if c.kind == S.DOWN and c.form != S.F32], ids=lambda c: c.id)
def test_split_and_tma_agree(lib, cuda_device, case):
    """The two tensor-core feed kernels do the same per-output arithmetic: byte-identical hi / lo where both run."""
    other = S.TMA if case.form == S.SPLIT else S.SPLIT
    a = Launch(case).run(lib)
    b = Launch(case, variant=other).run(lib)
    accepts = (case.c == 512) if other == S.SPLIT else (case.w // 2 >= 16 and case.w % 4 == 0 and case.h // 2 >= 8)
    assert (b is not None) == accepts, case.id
    if b is not None:
        assert _bytes(a) == _bytes(b), case.id


@pytest.mark.parametrize("path", ["simt", "tc"])
def test_generator_negative_lobe_down_taps(cuda_device, path):
    """migan-64 with outer([-1,2,2,-1]/2) (sum |f| = 9) in every downsample.filter.weight, on inputs scaled into the clamp:
    finite and within 1e-4 |y|max of the float64 oracle."""
    R, N = 64, 2
    sd = O.make_state_dict(R, seed=1)
    for k in sd:
        if k.endswith("downsample.filter.weight"):
            sd[k] = torch.outer(S.LOBES, S.LOBES).expand_as(sd[k]).contiguous()
    x = O.make_input(R, N, seed=3) * 3000.0
    want = FC.generator_forward_fc(sd, x, R, dtype=torch.float64)
    g = migan_b200.Generator(R, path=path)
    g.load_state_dict(sd)
    g = g.to(cuda_device).eval()
    got = g(x.to(cuda_device)).cpu().double()
    mx = float((got - want).abs().max())
    print("\nnegative-lobe down taps, %s: finite %s, max-abs %.3e (|y|max %.3e)"
          % (path, bool(torch.isfinite(got).all()), mx, float(want.abs().max())))
    assert bool(torch.isfinite(got).all())
    assert mx < 1e-4 * float(want.abs().max())


def test_report():
    """Measured bounds and launch count of this file (printed with -s)."""
    print("\nstages: max model ratio %s, max float64 error %s, %d launches, %.0f s"
          % ({k: round(v, 3) for k, v in sorted(STATS.get("model", {}).items())},
             {k: float("%.2e" % v) for k, v in sorted(STATS.get("op", {}).items())}, STATS["launches"], time.time() - T0))
