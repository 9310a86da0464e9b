"""The tensor-core SeparableConv2d kernel on its own, one launch at a time -- needs an H100.

Each case of the matrix (oracle/sepconv_oracle.py CASES) runs through the test hook `migan_debug_sepconv_tc`:
  a. the production plan, against the exact model of the split arithmetic (tight bound) and the float64 operation
     (contract bound);
  b. every candidate layout of the planner that fits, and grids of 1, 2, half and all SMs: byte-identical to (a)
     whenever the N tile width is the same, and each launched plan equal to its plan-only record;
  c. in every launch, 64 KB guard bands before and after the output and the image stay untouched (the whole feature map
     too when it is not stored), and NaN in the noise planes' padding never reaches the output.
Then the SM budget at the generator level: MIGAN_TC_RESERVE_SMS changes plans, never results.
"""
import ctypes
import time

import pytest
import torch

import migan_b200
from migan_b200 import _abi
from oracle import migan_oracle as O
from oracle import sepconv_oracle as S

pytestmark = pytest.mark.gpu

GUARD = 16384                      # floats (64 KB) of sentinel before and after each output buffer
SENTINEL = 0x7FC0DEAD              # a NaN bit pattern no kernel writes
STATS = {"launches": 0, "candidate_launches": 0, "sms_launches": 0, "model": {1: 0.0, 3: 0.0}, "op": {1: 0.0, 3: 0.0}}
T0 = time.time()


def _dev(t):
    return torch.as_tensor(t).contiguous().to("cuda:0")


def _guarded(numel):
    buf = torch.full((GUARD + numel + GUARD,), SENTINEL, dtype=torch.int32, device="cuda:0")
    return buf, buf[GUARD: GUARD + numel].view(torch.float32)


def _nan_padded(plane, case):
    p = plane.clone()
    p[:, case.w:] = float("nan")
    p[case.h:, :] = float("nan")
    return p


class Launch:
    """Device copies of a case's operands; run() launches once and returns (out, img, plan)."""

    def __init__(self, case):
        self.case = S.make_case(case)
        c, t = self.case, self.case.t
        self.keep = {}
        io = _abi.SepconvTcIO(source=c.source, n=c.n, h=c.h, w=c.w, cin=c.cin, cout=c.cout, act=c.act, passes=c.passes,
                              noise_pitch=c.noise_pitch, torgb=int(c.torgb), store_out=c.store_out)
        for name, field in (("in", "in_"), ("up_t", "up_t"), ("up_fir", "up_fir"), ("x", "x"), ("fromrgb_w", "fromrgb_w"),
                            ("fromrgb_b", "fromrgb_b"), ("dw_w", "dw_w"), ("dw_b", "dw_b"), ("pw_w", "pw_w"),
                            ("rgb_w", "rgb_w"), ("rgb_b", "rgb_b"), ("rgb_fir", "rgb_fir"), ("img_lo", "img_lo"),
                            ("a_hi", "a_hi"), ("a_lo", "a_lo"), ("noise", "noise"), ("up_noise", "up_noise")):
            if name in t:
                v = t[name]
                if name in ("noise", "up_noise"):
                    v = _nan_padded(v, c)
                d = _dev(torch.from_numpy(v) if not isinstance(v, torch.Tensor) else v)
                self.keep[name] = d
                setattr(io, field, d.data_ptr())
        self.io = io

    def run(self, lib, sms=0, candidate=-1):
        c = self.case
        out_buf, out = _guarded(c.n * c.h * c.w * c.cout)
        img_buf, img = _guarded(c.n * 3 * c.h * c.w)
        self.io.out = out.data_ptr()
        self.io.img_out = img.data_ptr() if c.torgb else None
        plan = _abi.SepconvTcPlan()
        rc = lib.migan_debug_sepconv_tc(ctypes.byref(self.io), sms, candidate, ctypes.byref(plan),
                                        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc == _abi.ERR_INVALID and candidate >= 0:
            return None                                    # this candidate layout does not fit: refused, not launched
        assert rc == 0, (c.id, sms, candidate, lib.migan_last_error(), lib.migan_debug_tc_timeout(0))
        STATS["launches"] += 1
        torch.cuda.synchronize()
        # guard bands (and, with nothing stored, the whole feature map) hold the sentinel
        for buf, used in ((out_buf, c.store_out or not c.torgb), (img_buf, c.torgb)):
            s = buf.cpu()
            body = s[GUARD:-GUARD]
            assert bool((s[:GUARD] == SENTINEL).all()) and bool((s[-GUARD:] == SENTINEL).all()), (c.id, "guard band written")
            if not used:
                assert bool((body == SENTINEL).all()), (c.id, "unused output written")
        out_h = out.cpu().reshape(c.n, c.h, c.w, c.cout) if (c.store_out or not c.torgb) else None
        img_h = img.cpu().reshape(c.n, 3, c.h, c.w) if c.torgb else None
        for v in (out_h, img_h):
            if v is not None:
                assert bool(torch.isfinite(v).all()), (c.id, "non-finite output: NaN padding read?")
        return out_h, img_h, plan.as_dict()


def _plan_only(lib, case, sms, candidate):
    io = _abi.SepconvTcIO(source=case.source, n=case.n, h=case.h, w=case.w, cin=case.cin, cout=case.cout, act=case.act,
                          passes=case.passes, noise_pitch=case.noise_pitch, torgb=int(case.torgb), store_out=case.store_out)
    plan = _abi.SepconvTcPlan()
    _abi.check(lib.migan_debug_sepconv_tc(ctypes.byref(io), sms, candidate, ctypes.byref(plan), None))
    return plan.as_dict()


def _same(a, b):
    return (a is None and b is None) or torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("case", S.CASES, ids=lambda c: c.id)
def test_launch_matches_model_and_op_on_every_schedule(lib, cuda_device, case):
    dev_sms = torch.cuda.get_device_properties(0).multi_processor_count
    L = Launch(case)
    out, img, plan = L.run(lib)
    # a. production plan: exact model (tight) and float64 operation (contract)
    r = S.model_ratio(case, out, img)
    e = S.op_error(case, out, img)
    print("\n%s: %s, model ratio %.3f, float64 error %.2e" % (case.id, plan, r, e))
    STATS["model"][case.passes] = max(STATS["model"][case.passes], r)
    STATS["op"][case.passes] = max(STATS["op"][case.passes], e)
    assert r <= 1.0, ("outside the model bound", r)
    assert e < S.OP_BOUND[case.passes], ("outside the contract bound", e)
    # b. every candidate that fits, and other grids: the sums do not depend on the schedule
    runs = [(0, i) for i in range(plan["num_candidates"])] + [(s, -1) for s in sorted({1, 2, dev_sms // 2, dev_sms})]
    launched = 0
    for sms, cand in runs:
        res = L.run(lib, sms, cand)
        if res is None:
            continue
        launched += 1
        STATS["candidate_launches" if cand >= 0 else "sms_launches"] += 1
        o2, i2, p2 = res
        assert p2 == _plan_only(lib, case, sms or dev_sms, cand), (sms, cand)
        if p2["n_tile"] == plan["n_tile"]:
            assert _same(o2, out) and _same(i2, img), ("schedule changed the result", sms, cand, p2)
        else:
            assert S.model_ratio(case, o2, i2) <= 1.0 and S.op_error(case, o2, i2) < S.OP_BOUND[case.passes]
    assert launched > 4


def _fresh_outputs(R, n, monkeypatch, reserve, hw=None):
    monkeypatch.setenv("MIGAN_TC_RESERVE_SMS", str(reserve))
    sd = O.make_state_dict(R, seed=2)
    g = migan_b200.Generator(R)
    g.load_state_dict(sd)
    g = g.to("cuda:0").eval()
    g.set_profiling(True)
    x = O.make_input(R, n, seed=9).to("cuda:0")
    res = [g(x)]
    labels = [row[0] for row in g.profile_steps()]
    if hw is not None:
        xf = torch.nn.functional.interpolate(x, size=hw, mode="nearest")
        res.append(g.forward_fc(xf))
        labels += [row[0] for row in g.profile_steps()]
    torch.cuda.synchronize()
    return [t.cpu() for t in res], labels


@pytest.mark.parametrize("R,n,hw", [(512, 4, (640, 896)), (256, 1, None)])
def test_sm_reserve_changes_plans_not_results(lib, cuda_device, monkeypatch, R, n, hw):
    want, want_labels = _fresh_outputs(R, n, monkeypatch, 0, hw)
    for reserve in (8, 12, 66):
        got, labels = _fresh_outputs(R, n, monkeypatch, reserve, hw)
        assert labels == want_labels, reserve
        for a, b in zip(got, want):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), reserve
    # the reserve does change plans: synthesis.b128.conv2 of migan-512 at n = 4 (UP source, 256 -> 256, torgb fused)
    dev_sms = torch.cuda.get_device_properties(0).multi_processor_count
    layer = S.Case(S.UP, 4, 128, 128, 256, 256, torgb=True, img_lo=True)
    plans = {_plan_only(lib, layer, dev_sms - min(r, dev_sms // 2), -1)["grid"] for r in (0, 8, 12, 66)}
    assert len(plans) == 4


def test_report():
    """Measured bounds and launch counts of this file (printed with -s)."""
    print("\nsepconv_tc: max model ratio %s, max float64 error %s, %d launches (%d candidate, %d grid), %.0f s"
          % (STATS["model"], STATS["op"], STATS["launches"], STATS["candidate_launches"], STATS["sms_launches"],
             time.time() - T0))
