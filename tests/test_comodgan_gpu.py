"""Co-Mod-GAN generator (BASELINE.json config 5) and conv2d_resample on the H100, through the C ABI, against the CPU
oracle (oracle/comodgan_oracle.py, pinned bit-exact to the reference) and the fixtures the REAL reference produced
(tests/golden/comodgan_*.npz, conv2d_resample.npz).  Tolerance: max-abs < 1e-3 at output scale ~10 (north_star); the
arithmetic is exact fp32 FMA, so the observed error is the summation-order noise floor (~1e-5)."""
import os

import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from migan_b200 import comodgan, ops
from oracle import comodgan_oracle as C
from oracle import migan_oracle as O

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-3


def make_generator(R, sd, device):
    g = comodgan.Generator(comodgan.Mapping(num_ws=C.num_ws(R)), comodgan.Encoder(resolution=R),
                           comodgan.Synthesis(resolution=R))
    g.load_state_dict(sd, strict=True)
    return g.to(device).eval()


@pytest.fixture(scope="module")
def gen16(cuda_device):
    sd = C.make_state_dict(16, seed=1)
    return make_generator(16, sd, cuda_device), sd


def test_r16_matches_oracle_and_reference_fixture(gen16, cuda_device):
    g, sd = gen16
    x, z = O.make_input(16, 2, seed=1234), C.make_latent(2, seed=1235)
    y = g(x.to(cuda_device), z=z.to(cuda_device), noise_mode="const").cpu()
    assert y.shape == (2, 3, 16, 16) and y.dtype == torch.float32
    y_or = C.generator_forward(sd, x, z, 16)
    gold = np.load(os.path.join(GOLDEN, "comodgan_R16_n2_w1.npz"))
    err = float((y - y_or).abs().max())
    print("comodgan R=16 max-abs vs oracle %.3e  mean-abs %.3e" % (err, float((y - y_or).abs().mean())))
    assert err < TOL
    assert float((y - torch.from_numpy(gold["y"])).abs().max()) < TOL
    y0 = g(x.to(cuda_device), z=z.to(cuda_device), noise_mode="none").cpu()
    assert float((y0 - torch.from_numpy(gold["y_noise_none"])).abs().max()) < TOL
    assert g.last_launch_count() > 50


@pytest.mark.parametrize("tap", ["mapping.w", "encoder.b16.fromrgb.out", "encoder.b16.conv1.out", "encoder.b4.fc.out",
                                 "synthesis.b4.conv.out", "synthesis.b8.conv0.out", "synthesis.b8.img",
                                 "synthesis.b16.torgb.out"])
def test_r16_intermediates(gen16, cuda_device, tap):
    g, sd = gen16
    x, z = O.make_input(16, 2, seed=5), C.make_latent(2, seed=6)
    taps = {}
    C.generator_forward(sd, x, z, 16, taps=taps)
    if tap == "mapping.w":
        want = taps["mapping.ws"][:, 0].reshape(2, 512, 1, 1)
    elif tap == "encoder.b4.fc.out":
        want = taps[tap].reshape(2, 1024, 1, 1)
    elif tap == "synthesis.b8.conv0.out":    # the epilogue also adds the encoder feature (comodgan.py:324)
        want = taps[tap] + taps["encoder.b8.conv0.out"]
    else:
        want = taps[tap]
    _, got = g(x.to(cuda_device), z=z.to(cuda_device), noise_mode="const", _tap=(tap, tuple(want.shape[1:])))
    assert float((got.cpu() - want).abs().max()) < 1e-4 * max(1.0, float(want.abs().max())), tap


def test_r16_truncation_and_random_noise(gen16, cuda_device):
    g, sd = gen16
    x, z = O.make_input(16, 3, seed=8), C.make_latent(3, seed=9)
    for psi, cutoff in ((0.6, None), (0.7, 3)):
        y = g(x.to(cuda_device), z=z.to(cuda_device), truncation_psi=psi, truncation_cutoff=cutoff, noise_mode="const").cpu()
        y_or = C.generator_forward(sd, x, z, 16, truncation_psi=psi, truncation_cutoff=cutoff)
        assert float((y - y_or).abs().max()) < TOL
    gen = torch.Generator().manual_seed(3)
    planes, noise = [], {}
    for (key, r), shape in zip(C.noise_keys(16), g.noise_plane_shapes(3)):
        assert shape == (3, r, r)
        p = torch.randn(3, 1, r, r, generator=gen)
        noise[key] = p
        planes.append(p.reshape(-1))
    y = g(x.to(cuda_device), z=z.to(cuda_device), noise_mode="random", noise=torch.cat(planes)).cpu()
    y_or = C.generator_forward(sd, x, z, 16, noise_mode="random", noise=noise)
    assert float((y - y_or).abs().max()) < TOL
    # default call of scripts/demo.py:134 (z and noise drawn by the module): runs, finite, not the const-noise image
    y_rand = g(x.to(cuda_device))
    assert torch.isfinite(y_rand).all()


@pytest.mark.parametrize("name", ["comodgan_R32_n2_w3", "comodgan_R64_n1_w1", "comodgan_R256_n1_w1"])
def test_reference_fixtures(cuda_device, name, monkeypatch):
    gold = np.load(os.path.join(GOLDEN, name + ".npz"))
    R, N = int(gold["resolution"]), int(gold["n"])
    if R == 32:
        monkeypatch.setenv("COMOD_COL_CAP_MB", "1")      # one-image chunks: exercises the chunk loop on the device
    sd = C.make_state_dict(R, seed=int(gold["wseed"]))
    assert abs(sum(float(v.double().abs().sum()) for v in sd.values()) - float(gold["w_checksum"])) < 1e-6 * float(gold["w_checksum"])
    g = make_generator(R, sd, cuda_device)
    x, z = O.make_input(R, N, seed=int(gold["xseed"])), C.make_latent(N, seed=int(gold["xseed"]) + 1)
    cutoff = None if int(gold["cutoff"]) < 0 else int(gold["cutoff"])
    y = g(x.to(cuda_device), z=z.to(cuda_device), truncation_psi=float(gold["psi"]), truncation_cutoff=cutoff,
          noise_mode="const").cpu()
    err = (y - torch.from_numpy(gold["y"])).abs()
    print("%s: max-abs %.3e mean-abs %.3e (|y|max %.2f)" % (name, float(err.max()), float(err.mean()), float(y.abs().max())))
    assert float(err.max()) < TOL


def test_demo_batch_256(cuda_device):
    """BASELINE.json config 5 shape: comodgan-256, batch 16.  Against the oracle on 2 of the 16 images would be wrong
    (the style normalisation of stylegan.py:146 couples the batch), so check the whole batch against the oracle."""
    sd = C.make_state_dict(256, seed=1)
    g = make_generator(256, sd, cuda_device)
    x, z = O.make_input(256, 4, seed=21), C.make_latent(4, seed=22)
    y = g(x.to(cuda_device), z=z.to(cuda_device), noise_mode="const").cpu()
    y_or = C.generator_forward(sd, x, z, 256)
    err = (y - y_or).abs()
    print("comodgan-256 n=4: max-abs %.3e mean-abs %.3e" % (float(err.max()), float(err.mean())))
    assert float(err.max()) < TOL
    # the configuration's own batch size: all 16 images against the oracle run on the same 16 (about 15 s of CPU)
    x16, z16 = O.make_input(256, 16, seed=23), C.make_latent(16, seed=24)
    y16 = g(x16.to(cuda_device), z=z16.to(cuda_device), noise_mode="const").cpu()
    assert y16.shape == (16, 3, 256, 256) and torch.isfinite(y16).all()
    err16 = (y16 - C.generator_forward(sd, x16, z16, 256)).abs()
    print("comodgan-256 n=16: max-abs %.3e mean-abs %.3e" % (float(err16.max()), float(err16.mean())))
    assert float(err16.max()) < TOL


def test_conv2d_resample_reference_vectors(cuda_device):
    from test_oracle import _c2r_cases, _c2r_stored_rows
    gold = np.load(os.path.join(GOLDEN, "conv2d_resample.npz"))
    cases = list(_c2r_cases(gold))
    assert len(cases) == 15
    for name, x, w, f, kw in cases:
        y = ops.conv2d_resample(x.to(cuda_device), w.to(cuda_device), None if f is None else f.to(cuda_device), **kw)
        y = _c2r_stored_rows(gold, name, y.cpu())
        assert float((y - torch.from_numpy(gold[name + ".y"])).abs().max()) < 1e-4, name


def test_conv2d_resample_odd_shapes(cuda_device):
    gen = torch.Generator().manual_seed(2)
    fa = torch.tensor([[1., 2., 0.5], [0.25, 3., 1.], [2., 1., 0.125]]) / 10.875
    f1 = torch.tensor([1., 3., 3., 1.]) / 8
    for (cin, cout, k, up, down, pad, groups, flipw, f, flipf) in [
        (3, 5, 3, 1, 1, 1, 1, True, None, False), (6, 10, 3, 2, 1, 1, 2, False, fa, False),
        (3, 7, 1, 1, 2, 0, 1, True, fa, True), (5, 3, 3, 1, 2, 1, 1, False, fa, False),
        (3, 6, 3, 1, 1, [1, 0, 2, 0], 3, True, None, False), (16, 64, 3, 2, 1, 1, 1, False, f1, False),
    ]:
        x = torch.randn(2, cin, 9, 7, generator=gen)
        w = torch.randn(cout, cin // groups, k, k, generator=gen)
        want = C.conv2d_resample_ref(x, w, f=f, up=up, down=down, padding=pad, groups=groups, flip_weight=flipw, flip_filter=flipf)
        got = ops.conv2d_resample(x.to(cuda_device), w.to(cuda_device), None if f is None else f.to(cuda_device), up=up,
                                  down=down, padding=pad, groups=groups, flip_weight=flipw, flip_filter=flipf)
        assert tuple(got.shape) == tuple(want.shape)
        assert float((got.cpu() - want).abs().max()) < 1e-4


def test_comodgan_512_matches_oracle(cuda_device):
    """scripts/demo.py:101-106 (comodgan-512, num_ws=16): adds the 64-channel levels.  The oracle is pinned bit-exact to
    the reference at this size by make_golden_comodgan.py (no fixture committed: 3 MB)."""
    sd = C.make_state_dict(512, seed=2)
    g = make_generator(512, sd, cuda_device)
    assert g.num_ws == 16
    x, z = O.make_input(512, 1, seed=3), C.make_latent(1, seed=4)
    y = g(x.to(cuda_device), z=z.to(cuda_device), noise_mode="const").cpu()
    err = (y - C.generator_forward(sd, x, z, 512)).abs()
    print("comodgan-512 n=1: max-abs %.3e mean-abs %.3e" % (float(err.max()), float(err.mean())))
    assert float(err.max()) < TOL
