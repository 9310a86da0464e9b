"""The epilogue window ring of the tensor-core SeparableConv2d kernel, as its planner places it -- no GPU needed.

The producer brings each CTA tile's noise and low-resolution image window into a ring of shared-memory stages, so that
the epilogue reads no global memory.  The ring is planned for 3-pass launches with noise or an image to up-sample, after
the layout the planner picks without it: it never changes the schedule, and it stays out of every other area.
"""
import ctypes

import pytest

from migan_b200 import _abi
from oracle import sepconv_oracle as S

SMEM_LIMIT, STATIC_SMEM = 232448, 4096      # per-block opt-in limit and the kernel's static shared memory (rounded up)
LAYOUT_KEYS = ("n_group", "in_stages", "a_stages", "b_stages", "b_resident", "dw_global", "tile_w", "tile_h", "tile_n",
               "n_tile", "grid", "num_tiles", "num_candidates")
FAKE = 0x10000                               # plan-only reads the operand pointers as flags only


def plan(lib, case, sms, candidate=-1, noise=None, img_lo=None, passes=None):
    io = _abi.SepconvTcIO(source=case.source, n=case.n, h=case.h, w=case.w, cin=case.cin, cout=case.cout, act=case.act,
                          passes=passes or case.passes, noise_pitch=case.noise_pitch, torgb=int(case.torgb),
                          store_out=case.store_out)
    io.noise = FAKE if (case.noise if noise is None else noise) else None
    io.img_lo = FAKE if (case.img_lo if img_lo is None else img_lo) else None
    rec = _abi.SepconvTcPlan()
    rc = lib.migan_debug_sepconv_tc(ctypes.byref(io), sms, candidate, ctypes.byref(rec), None)
    return dict(rec.as_dict(), **rec.ring()) if rc == 0 else None


def generator_like_cases():
    """The matrix plus the migan-512 fused synthesis layers at 32 images (UP source, noise, torgb, image)."""
    extra = [S.Case(S.UP, 32, r, r, c, c, 3, noise=True, up_noise=True, torgb=True, img_lo=True)
             for r, c in ((512, 64), (256, 128), (128, 256))]
    return list(S.CASES) + extra


@pytest.mark.parametrize("sms", [114, 132])
def test_ring_is_planned_exactly_where_it_has_work(lib, sms):
    for case in generator_like_cases():
        for passes in (1, 3):
            for noise in (False, True):
                for img in (False, True) if case.torgb else (False,):
                    r = plan(lib, case, sms, noise=noise, img_lo=img, passes=passes)
                    if r is None:
                        continue
                    if passes == 1 or not (noise or img):
                        assert r["ep_stages"] == 0, (case.id, passes, noise, img)
                    else:
                        assert r["ep_stages"] in (0, 2, 4), (case.id, noise, img)


@pytest.mark.parametrize("sms", [114, 132])
def test_ring_keeps_the_layout_and_its_own_area(lib, sms):
    for case in generator_like_cases():
        base = plan(lib, case, sms, noise=False, img_lo=False)
        assert base is not None and base["ep_stages"] == 0
        for i in [-1] + list(range(base["num_candidates"])):
            bare = plan(lib, case, sms, i, noise=False, img_lo=False)
            full = plan(lib, case, sms, i, noise=True, img_lo=case.torgb)
            assert (bare is None) == (full is None), (case.id, i)
            if full is None:
                continue
            assert {k: full[k] for k in LAYOUT_KEYS} == {k: bare[k] for k in LAYOUT_KEYS}, (case.id, i)
            if full["ep_stages"] == 0:
                assert full["smem_bytes"] == bare["smem_bytes"]
                continue
            layout_end = bare["smem_bytes"] - 1024
            assert full["ep_offset"] >= layout_end and full["ep_offset"] % 128 == 0 and full["ep_stage_bytes"] % 128 == 0
            end = full["ep_offset"] + full["ep_stages"] * full["ep_stage_bytes"]
            assert full["smem_bytes"] == end + 1024 <= SMEM_LIMIT - STATIC_SMEM, (case.id, i)


def test_migan512_synthesis_rings(lib):
    """Where the ring lands at migan-512 / 32 images: the 512- and 256-pixel fused layers get one; the 128-pixel layer's
    layout (a resident A at cin = 256) fills the budget to the byte and keeps its global reads."""
    got = {}
    for r, c in ((512, 64), (256, 128), (128, 256)):
        case = S.Case(S.UP, 32, r, r, c, c, 3, noise=True, up_noise=True, torgb=True, img_lo=True)
        got[r] = plan(lib, case, 132)["ep_stages"]
    assert got[512] > 0 and got[256] > 0 and got[128] == 0, got
