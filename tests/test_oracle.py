"""The oracle against the committed golden fixtures (produced from the REAL reference by
tests/golden/make_golden.py).  CPU only."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import fullconv_oracle as FC
from oracle import migan_oracle as O

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _checksum(t):
    return float(t.double().abs().sum())


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "migan_R*.npz"))))
def test_forward_matches_reference_golden(path):
    z = np.load(path)
    R, N = int(z["resolution"]), int(z["n"])
    if R > 256 and os.environ.get("MIGAN_FAST_TESTS"):
        pytest.skip("fast mode")
    sd = O.make_state_dict(R, seed=int(z["wseed"]))
    x = O.make_input(R, N, seed=int(z["xseed"]))
    # the seeded generators must reproduce what the fixture was made from
    assert _checksum(x) == pytest.approx(float(z["x_checksum"]), rel=1e-12)
    assert sum(_checksum(v) for v in sd.values()) == pytest.approx(float(z["w_checksum"]), rel=1e-12)
    taps = {}
    y = O.generator_forward(sd, x, R, taps=taps)
    want = torch.from_numpy(z["y"])
    if "y_rows" in z.files:                              # large outputs are stored on a row sample (shrink_golden.py)
        y = y[:, :, z["y_rows"]]
    # same torch build => bit exact; allow fp32 reassociation noise across CPUs (different oneDNN kernels)
    assert float((y - want).abs().max()) <= 2e-4
    for name, (cs, mx) in zip(z["tap_names"], z["tap_stats"]):
        t = taps[str(name)]
        assert _checksum(t) == pytest.approx(cs, rel=1e-4)
        assert float(t.abs().max()) == pytest.approx(mx, rel=1e-4)


def test_fp64_noise_floor():
    """fp32 vs fp64 evaluation of the same network: sets the floor of any tolerance (~1e-5)."""
    R = 64
    sd = O.make_state_dict(R, seed=1)
    x = O.make_input(R, 2)
    y32 = O.generator_forward(sd, x, R)
    y64 = O.generator_forward(sd, x, R, dtype=torch.float64)
    assert float((y32.double() - y64).abs().max()) < 1e-4


def test_state_dict_spec_counts():
    assert len(O.state_dict_spec(256)) == 154   # SURVEY.md 8b
    assert len(O.state_dict_spec(512)) == 177
    n512 = sum(int(np.prod(s)) for k, s in O.state_dict_spec(512).items()
               if not k.endswith(("filter_const", "noise_const")))
    assert n512 == 5973366                      # parameter count of the reference @512


def test_resolution_validation():
    with pytest.raises(ValueError):
        O.encode_res(96)


def _polyphase_up(x, f):
    """The polyphase form of Upsample2d the kernels implement, for any 4x4 filter f [C,1,4,4]:
    out[2i + a][2j + b] = sum_{u,v in {0,1}} f[a + 2u][b + 2v] * x[i - 1 + a + u][j - 1 + b + v]   (x = 0 outside)."""
    n, c, h, w = x.shape
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1))
    out = torch.zeros(n, c, 2 * h, 2 * w, dtype=x.dtype)
    for a in (0, 1):
        for b in (0, 1):
            for u in (0, 1):
                for v in (0, 1):
                    tap = f[:, 0, a + 2 * u, b + 2 * v].view(1, c, 1, 1)
                    out[:, :, a::2, b::2] += tap * xp[:, :, a + u:a + u + h, b + v:b + v + w]
    return out


def test_polyphase_identity():
    """Upsample2d == the 2-tap polyphase form the kernels use (SURVEY.md 7.4(4)), for the constructor's filter and for
    asymmetric per-channel filters (a checkpoint may carry trained taps)."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 2, 5, 5, generator=g)
    f = O.setup_filter([1, 3, 3, 1], gain=4).repeat(2, 1, 1, 1)
    fc = torch.tensor([[1.0, 0.0], [0.0, 0.0]]).repeat(1, 1, 5, 5)
    ref = O.upsample2d(x, f, fc)
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1))
    rows_e = 0.25 * xp[:, :, 0:5] + 0.75 * xp[:, :, 1:6]
    rows_o = 0.75 * xp[:, :, 1:6] + 0.25 * xp[:, :, 2:7]
    rows = torch.stack([rows_e, rows_o], 3).reshape(1, 2, 10, 7)
    cols_e = 0.25 * rows[..., 0:5] + 0.75 * rows[..., 1:6]
    cols_o = 0.75 * rows[..., 1:6] + 0.25 * rows[..., 2:7]
    out = torch.stack([cols_e, cols_o], 4).reshape(1, 2, 10, 10)
    assert float((out - ref).abs().max()) < 1e-6
    assert float((_polyphase_up(x, f) - ref).abs().max()) < 1e-6
    # asymmetric taps, different per channel, on a non-square input
    x = torch.randn(2, 3, 5, 7, generator=g, dtype=torch.float64)
    f = O.random_fir(3, 4.0, g).double()
    assert not torch.equal(f, f.flip([2, 3])) and not torch.equal(f, f.transpose(2, 3)) and not torch.equal(f[0], f[1])
    ref = O.upsample2d(x, f, FC.zero_insertion(10, 14).double())
    assert float((_polyphase_up(x, f) - ref).abs().max()) < 1e-12
    for wrong in (f.flip([2, 3]), f.transpose(2, 3), f[:1].expand_as(f)):   # the oracle tells each mistake apart
        assert float((_polyphase_up(x, wrong) - ref).abs().max()) > 1e-2


def test_make_state_dict_fir_modes():
    """fir= changes the FIR taps only; the constructor mode is the default, and random taps keep their gain."""
    base = O.make_state_dict(64, seed=1)
    assert all(torch.equal(a, b) for a, b in zip(base.values(), O.make_state_dict(64, seed=1, fir="constructor").values()))
    for mode in ("uniform", "per_channel"):
        sd = O.make_state_dict(64, seed=1, fir=mode)
        assert list(sd.keys()) == list(base.keys())
        for k, v in sd.items():
            if not k.endswith("filter.weight"):
                assert torch.equal(v, base[k]), k
                continue
            assert v.shape == base[k].shape and v.is_contiguous()
            gain = 1.0 if "downsample" in k else 4.0
            assert torch.allclose(v.sum(dim=(2, 3)), torch.full(v.shape[:2], gain), atol=1e-5), k
            assert (v > 0).all() and not torch.equal(v, v.flip([2, 3])) and not torch.equal(v, v.transpose(2, 3)), k
            assert torch.equal(v, v[:1].expand_as(v)) == (mode == "uniform"), k
    with pytest.raises(ValueError):
        O.make_state_dict(64, fir="symmetric")


def _fir_cases():
    return list(range(int(np.load(os.path.join(GOLDEN, "fir.npz"))["num_cases"])))


@pytest.mark.parametrize("case", _fir_cases())
def test_oracle_reproduces_fir_fixture(case):
    """The oracle with asymmetric FIR taps against outputs of the reference itself (make_golden_fir.py)."""
    z = np.load(os.path.join(GOLDEN, "fir.npz"))
    R, N, H, W, wseed, xseed = [int(v) for v in z["case%d_meta" % case]]
    sd = O.make_state_dict(R, seed=wseed, fir=str(z["case%d_fir" % case]))
    x = FC.make_input_hw(R, N, H, W, seed=xseed)
    assert sum(_checksum(v) for v in sd.values()) == pytest.approx(float(z["case%d_w_checksum" % case]), rel=1e-12)
    assert _checksum(x) == pytest.approx(float(z["case%d_x_checksum" % case]), rel=1e-12)
    y = FC.generator_forward_fc(sd, x, R)
    if (H, W) == (R, R):
        assert torch.equal(y, O.generator_forward(sd, x, R))
    rows = z["case%d_rows" % case]
    assert np.array_equal(rows, np.arange(H) if R == 64 else FC.fixture_rows(H, period=16).numpy())
    assert float((y[:, :, rows] - torch.from_numpy(z["case%d_y" % case])).abs().max()) <= 1e-5


def test_op_oracles_match_golden():
    z = np.load(os.path.join(GOLDEN, "ops.npz"))
    x = torch.from_numpy(z["x"])
    bvec = torch.from_numpy(z["bvec"])
    f2 = O.setup_filter([1, 3, 3, 1])
    f1 = torch.from_numpy(z["f1"])
    cases = [(f2, 1, 1, (1, 2, 2, 1), False, 1.0), (f2, 2, 1, (2, 1, 2, 1), False, 4.0),
             (f2, 1, 2, (1, 1, 1, 1), False, 1.0), (f2, 2, 2, (3, 0, 1, 2), True, 2.0),
             (f1, 1, 1, (4, 3, 4, 3), False, 1.0), (f1, 2, 1, (5, 4, 5, 4), True, 4.0),
             (None, 1, 1, (0, 0, 0, 0), False, 1.0), (f2, 1, 1, (-1, 2, 3, -1), False, 1.0)]
    for i, (f, up, down, pad, flip, gain) in enumerate(cases):
        got = O.upfirdn2d_ref(x, f, up=up, down=down, padding=pad, flip_filter=flip, gain=gain)
        assert np.allclose(got.numpy().ravel(), z["up%d" % i], atol=1e-6)
    i = 0
    for act in O._ACT:
        for clamp in (None, 0.7):
            got = O.bias_act_ref(x, bvec, dim=1, act=act, clamp=clamp)
            assert np.allclose(got.numpy().ravel(), z["ba%d" % i], atol=1e-6), act
            i += 1


# --------------------------------------------------------------------------- #
# Co-Mod-GAN oracle (oracle/comodgan_oracle.py) against the fixtures the real reference produced
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("name", ["comodgan_R16_n2_w1", "comodgan_R32_n2_w3", "comodgan_R64_n1_w1"])
def test_comodgan_oracle_reproduces_reference_fixture(name):
    from oracle import comodgan_oracle as C
    from oracle import migan_oracle as O
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz"))
    R, N = int(g["resolution"]), int(g["n"])
    sd = C.make_state_dict(R, seed=int(g["wseed"]))
    x = O.make_input(R, N, seed=int(g["xseed"]))
    z = C.make_latent(N, seed=int(g["xseed"]) + 1)
    assert abs(float(x.double().abs().sum()) - float(g["x_checksum"])) < 1e-6 * float(g["x_checksum"])
    cutoff = None if int(g["cutoff"]) < 0 else int(g["cutoff"])
    y = C.generator_forward(sd, x, z, R, truncation_psi=float(g["psi"]), truncation_cutoff=cutoff)
    assert float((y - torch.from_numpy(g["y"])).abs().max()) <= 1e-4   # same primitives; allows a different BLAS build
    y0 = C.generator_forward(sd, x, z, R, truncation_psi=float(g["psi"]), truncation_cutoff=cutoff, noise_mode="none")
    assert float((y0 - torch.from_numpy(g["y_noise_none"])).abs().max()) <= 1e-4


def test_comodgan_state_dict_spec_counts():
    from oracle import comodgan_oracle as C
    spec = C.state_dict_spec(256)
    assert len(spec) == 180                                          # SURVEY: reference state_dict @256
    assert sum(int(np.prod(s)) for s in spec.values()) == 79353026   # 79 M parameters + buffers
    assert C.num_ws(256) == 14 and C.num_ws(512) == 16               # comodgan.py:371-374


def _c2r_cases(g):
    """(name, x, w, f or None, kwargs) of every vector in tests/golden/conv2d_resample.npz."""
    from oracle import migan_oracle as O
    f44 = O.setup_filter([1, 3, 3, 1])
    for name in sorted({k.rsplit(".", 1)[0] for k in g.files}):
        a = [int(v) for v in g[name + ".args"]]
        f = f44
        if name + ".f" in g.files:
            f = None if g[name + ".f"].size == 0 else torch.from_numpy(g[name + ".f"])
        yield name, torch.from_numpy(g[name + ".x"]), torch.from_numpy(g[name + ".w"]), f, dict(
            up=a[0], down=a[1], groups=a[2], flip_weight=bool(a[3]), padding=a[4:8], flip_filter=bool(a[8]) if len(a) > 8 else False)


def _c2r_stored_rows(g, name, y):
    """y (computed, full) on the rows the fixture stores: large outputs are kept as a row sample (shrink_golden.py)."""
    if name + ".yrows" not in g.files:
        assert tuple(y.shape) == g[name + ".y"].shape, name
        return y
    assert tuple(y.shape) == tuple(int(v) for v in g[name + ".yshape"]), name
    return y[:, :, g[name + ".yrows"]]


def test_conv2d_resample_oracle_reproduces_reference_vectors():
    from oracle import comodgan_oracle as C
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "conv2d_resample.npz"))
    cases = list(_c2r_cases(g))
    assert len(cases) == 15
    for name, x, w, f, kw in cases:
        y = _c2r_stored_rows(g, name, C.conv2d_resample_ref(x, w, f=f, **kw))
        assert float((y - torch.from_numpy(g[name + ".y"])).abs().max()) <= 1e-4, name
