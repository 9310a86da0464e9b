"""Pin the Co-Mod-GAN oracle against the REAL reference and write the committed fixtures.

Needs a checkout of the reference (MIGAN_REF):   python tests/golden/make_golden_comodgan.py

For each case it builds ``lib.model_zoo.comodgan.Generator(Mapping, Encoder, Synthesis)`` the way
``scripts/demo.py:95-100`` does, loads the oracle's seeded state_dict with ``strict=True`` (key names, order and shapes
are thereby checked against the reference), runs both on the same (x, z) with ``noise_mode='const'`` and asserts that
they agree (bit-exact is expected: same torch primitives in the same order), then stores the reference output in
``tests/golden/comodgan_R{R}_n{N}_w{seed}.npz``.  It also pins ``conv2d_resample_ref`` against the reference's
``conv2d_resample`` for every branch and stores small vectors in ``tests/golden/conv2d_resample.npz``.
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("MIGAN_REF", "../MI-GAN")   # a checkout of the reference project
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)
warnings.filterwarnings("ignore")

from oracle import comodgan_oracle as C  # noqa: E402
from oracle import migan_oracle as O  # noqa: E402


def checksum(t: torch.Tensor) -> float:
    return float(t.double().abs().sum())


def build_reference(R: int):
    from lib.model_zoo.comodgan import Encoder, Generator, Mapping, Synthesis
    syn = Synthesis(resolution=R)
    if not hasattr(syn, "num_ws"):          # the reference only sets num_ws for 256 / 512 (comodgan.py:371-374)
        syn.num_ws = C.num_ws(R)
    return Generator(Mapping(num_ws=C.num_ws(R)), Encoder(resolution=R), syn).eval()


def main():
    from torch_utils.ops import conv2d_resample as ref_c2r
    from torch_utils.ops import upfirdn2d as ref_upfirdn2d

    cases = [(16, 2, 1, 1234, 1.0, None), (32, 2, 3, 77, 0.7, 4), (64, 1, 1, 1234, 1.0, None),
             (256, 1, 1, 1234, 1.0, None)]
    for R, N, wseed, xseed, psi, cutoff in cases:
        ref = build_reference(R)
        sd = C.make_state_dict(R, seed=wseed)
        assert list(ref.state_dict().keys()) == list(sd.keys()), "state_dict key order differs"
        for k, v in ref.state_dict().items():
            assert tuple(v.shape) == tuple(sd[k].shape), k
        ref.load_state_dict(sd, strict=True)
        x = O.make_input(R, N, seed=xseed)
        z = C.make_latent(N, seed=xseed + 1)
        with torch.no_grad():
            y_ref = ref(x.clone(), z=z.clone(), truncation_psi=psi, truncation_cutoff=cutoff, noise_mode="const")
        taps = {}
        y_or = C.generator_forward(sd, x, z, R, truncation_psi=psi, truncation_cutoff=cutoff, taps=taps)
        err = float((y_ref - y_or).abs().max())
        print("R=%d N=%d  ref-vs-oracle max-abs = %.3e   |y|max=%.3f  |y|mean=%.3f"
              % (R, N, err, float(y_ref.abs().max()), float(y_ref.abs().mean())))
        assert err == 0.0, "oracle does not reproduce the reference"
        with torch.no_grad():
            y_none = ref(x.clone(), z=z.clone(), truncation_psi=psi, truncation_cutoff=cutoff, noise_mode="none")
        assert float((y_none - C.generator_forward(sd, x, z, R, truncation_psi=psi, truncation_cutoff=cutoff,
                                                   noise_mode="none")).abs().max()) == 0.0
        f64err = -1.0
        if R <= 64:
            y64 = C.generator_forward(sd, x, z, R, truncation_psi=psi, truncation_cutoff=cutoff, dtype=torch.float64)
            f64err = float((y_ref.double() - y64).abs().max())
            print("    fp32 reference vs fp64 oracle max-abs = %.3e" % f64err)
        names = ["mapping.ws", "encoder.b%d.fromrgb.out" % R, "encoder.b%d.conv1.out" % R, "encoder.b4.fc.out",
                 "synthesis.b4.conv.out", "synthesis.b%d.conv0.out" % R, "synthesis.b%d.torgb.out" % R]
        stats = np.stack([np.array([checksum(taps[k]), float(taps[k].abs().max())]) for k in names])
        np.savez_compressed(
            os.path.join(HERE, "comodgan_R%d_n%d_w%d.npz" % (R, N, wseed)),
            y=y_ref.numpy(), y_noise_none=(y_none.numpy() if R <= 64 else np.zeros(0, np.float32)),
            resolution=R, n=N, wseed=wseed, xseed=xseed, psi=psi, cutoff=(-1 if cutoff is None else cutoff),
            x_checksum=checksum(x), z_checksum=checksum(z), w_checksum=sum(checksum(v) for v in sd.values()),
            fp64_maxabs=f64err, tap_names=np.array(names), tap_stats=stats)

    # comodgan-512 (scripts/demo.py:101-106, num_ws=16): pin only, no fixture (3 MB)
    ref = build_reference(512)
    sd = C.make_state_dict(512, seed=2)
    ref.load_state_dict(sd, strict=True)
    x, z = O.make_input(512, 1, seed=3), C.make_latent(1, seed=4)
    with torch.no_grad():
        y_ref = ref(x.clone(), z=z.clone(), noise_mode="const")
    err = float((y_ref - C.generator_forward(sd, x, z, 512)).abs().max())
    print("R=512 N=1  ref-vs-oracle max-abs = %.3e" % err)
    assert err == 0.0

    # conv2d_resample: every branch, against the reference op (impl falls back to its own ref path on CPU) -------
    g = torch.Generator().manual_seed(11)
    f = ref_upfirdn2d.setup_filter([1, 3, 3, 1])
    out = {}
    specs = [  # name, cin, cout, k, up, down, padding, groups, flip_weight
        ("k1_down", 16, 64, 1, 1, 2, 0, 1, True), ("k1_up", 16, 64, 1, 2, 1, 0, 1, True),
        ("k3_down", 16, 64, 3, 1, 2, 1, 1, True), ("k3_up", 16, 64, 3, 2, 1, 1, 1, False),
        ("k3_up_groups", 32, 128, 3, 2, 1, 1, 2, False), ("k3_plain", 16, 64, 3, 1, 1, 1, 1, True),
        ("k3_plain_groups_noflip", 32, 128, 3, 1, 1, 1, 2, False), ("k3_asym_pad", 16, 64, 3, 1, 1, [2, 0, 1, 0], 1, True),
        ("k3_updown", 16, 64, 3, 2, 2, 1, 1, True),
    ]
    for name, cin, cout, k, up, down, pad, groups, flipw in specs:
        x = torch.randn(2, cin, 10, 12, generator=g)
        w = torch.randn(cout, cin // groups, k, k, generator=g)
        y_ref = ref_c2r.conv2d_resample(x, w, f=f, up=up, down=down, padding=pad, groups=groups, flip_weight=flipw)
        y_or = C.conv2d_resample_ref(x, w, f=f, up=up, down=down, padding=pad, groups=groups, flip_weight=flipw)
        assert y_ref.shape == y_or.shape and float((y_ref - y_or).abs().max()) == 0.0, name
        out[name + ".x"], out[name + ".w"], out[name + ".y"] = x.numpy(), w.numpy(), y_ref.numpy()
        out[name + ".args"] = np.array([up, down, groups, int(flipw)] + (pad if isinstance(pad, list) else [pad] * 4))
        print("conv2d_resample %-24s -> %s pinned" % (name, tuple(y_ref.shape)))
    # filters other than the 4x4 binomial: none at all with up/down > 1 (negative padding adjustments), non-square 2-D,
    # non-square kernel, flip_filter.  The filter travels with the vector ("<name>.f", empty = None).
    fns = torch.rand(3, 5, generator=g)
    extra = [  # name, cin, cout, kh, kw, up, down, pad, groups, flipw, f, flipf
        ("x_fnone_up3", 4, 6, 3, 3, 3, 1, 1, 1, True, None, False), ("x_fnone_down3", 4, 6, 2, 2, 1, 3, 0, 2, False, None, False),
        ("x_fnone_updown", 4, 6, 3, 3, 2, 3, [0, 1, 2, 0], 1, True, None, False),
        ("x_nonsquare_f_up2", 4, 6, 3, 3, 2, 1, 1, 1, False, fns, False), ("x_nonsquare_f_down2_flip", 6, 4, 1, 1, 1, 2, 1, 1, True, fns, True),
        ("x_nonsquare_k", 4, 8, 2, 4, 2, 2, [1, 0, 0, 2], 2, False, f, False),
    ]
    for name, cin, cout, kh, kw, up, down, pad, groups, flipw, ff, flipf in extra:
        x = torch.randn(2, cin, 7, 9, generator=g)
        w = torch.randn(cout, cin // groups, kh, kw, generator=g)
        y_ref = ref_c2r.conv2d_resample(x, w, f=ff, up=up, down=down, padding=pad, groups=groups, flip_weight=flipw, flip_filter=flipf)
        y_or = C.conv2d_resample_ref(x, w, f=ff, up=up, down=down, padding=pad, groups=groups, flip_weight=flipw, flip_filter=flipf)
        assert y_ref.shape == y_or.shape and float((y_ref - y_or).abs().max()) == 0.0, name
        out[name + ".x"], out[name + ".w"], out[name + ".y"] = x.numpy(), w.numpy(), y_ref.numpy()
        out[name + ".f"] = np.zeros((0, 0), np.float32) if ff is None else ff.numpy()
        out[name + ".args"] = np.array([up, down, groups, int(flipw)] + (pad if isinstance(pad, list) else [pad] * 4) + [int(flipf)])
        print("conv2d_resample %-24s -> %s pinned" % (name, tuple(y_ref.shape)))
    np.savez_compressed(os.path.join(HERE, "conv2d_resample.npz"), **out)


if __name__ == "__main__":
    main()
