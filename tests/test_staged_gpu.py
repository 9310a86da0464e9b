"""Opt-in code paths (off by default).

  COMOD_GEMM=tc   Co-Mod-GAN plain / strided / 1x1 convolutions on the wgmma GEMM of the MI-GAN path (sepconv_tc.cu in its
                  A_TMA configuration, K up to 4608) fed by an fp16 hi/lo split im2col.  Operand packing is covered on the
                  CPU by tests/test_comodgan_emul.py::test_staged_tcgen05_route_operands.
"""
import os

import numpy as np
import pytest
import torch

from oracle import comodgan_oracle as C
from oracle import migan_oracle as O

pytestmark = [pytest.mark.gpu]
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("name", ["comodgan_R16_n2_w1", "comodgan_R64_n1_w1", "comodgan_R256_n1_w1"])
def test_comodgan_tcgen05_route(cuda_device, name, monkeypatch):
    from migan_b200 import comodgan
    monkeypatch.setenv("COMOD_GEMM", "tc")
    gold = np.load(os.path.join(GOLDEN, name + ".npz"))
    R, N = int(gold["resolution"]), int(gold["n"])
    sd = C.make_state_dict(R, seed=int(gold["wseed"]))
    g = comodgan.Generator(comodgan.Mapping(num_ws=C.num_ws(R)), comodgan.Encoder(resolution=R), comodgan.Synthesis(resolution=R))
    g.load_state_dict(sd)
    g = g.to(cuda_device).eval()
    x, z = O.make_input(R, N, seed=int(gold["xseed"])), C.make_latent(N, seed=int(gold["xseed"]) + 1)
    y = g(x.to(cuda_device), z=z.to(cuda_device), noise_mode="const").cpu()
    err = (y - torch.from_numpy(gold["y"])).abs()
    print("%s [wgmma route]: max-abs %.3e mean-abs %.3e" % (name, float(err.max()), float(err.mean())))
    assert float(err.max()) < 1e-3
