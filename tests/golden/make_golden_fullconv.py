"""Generate tests/golden/fullconv.npz by running the REAL reference fully convolutionally.

Run where a checkout of the reference exists (MIGAN_REF; not on the GPU box):
    python tests/golden/make_golden_fullconv.py

The reference README ("Quick Test") says the network is fully convolutional once `filter_const` and `noise_const` are
made dynamic.  For each case this
  1. builds the reference ``lib.model_zoo.migan_inference.Generator(R)`` and loads the oracle's seeded state_dict
     (strict, so names / order / shapes are checked),
  2. replaces every ``Upsample2d.filter_const`` by the zero-insertion pattern at its block's output extent and every
     ``noise_const`` by its r x r plane tiled over the layer's extent (noise[i, j] = noise_const[i mod r, j mod r]),
  3. runs the reference forward on a seeded [N, 4, H, W] input, checks the oracle's fully convolutional form
     (oracle/fullconv_oracle.py) gives the same output, and stores y on a fixed row sample (`fixture_rows`: r % 8 in
     {0, 1} and the last two rows, which keeps the file below 1 MB) with the seeds, shapes and a weight checksum.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("MIGAN_REF", "../MI-GAN")   # a checkout of the reference project
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

from oracle import fullconv_oracle as FC  # noqa: E402
from oracle import migan_oracle as O  # noqa: E402

# (R, N, H, W, weight seed, input seed)
CASES = [(64, 2, 64, 96, 1, 1234), (64, 1, 112, 80, 3, 77), (128, 1, 160, 224, 1, 5), (256, 1, 256, 320, 1, 1234)]


def make_fullconv(ref, R, H, W):
    """Step 2 above, on the reference module tree."""
    for m in ref.modules():
        if "filter_const" in m._buffers:
            r = m.filter_const.shape[-1]
            m.filter_const = FC.zero_insertion(H * r // R, W * r // R)
        if "noise_const" in m._buffers:
            r = m.noise_const.shape[-1]
            m.noise_const = FC.tiled_noise(m.noise_const, H * r // R, W * r // R)


def main():
    from lib.model_zoo.migan_inference import Generator as RefGenerator

    out = {}
    for i, (R, N, H, W, wseed, xseed) in enumerate(CASES):
        ref = RefGenerator(resolution=R).eval()
        sd = O.make_state_dict(R, seed=wseed)
        assert list(ref.state_dict().keys()) == list(sd.keys()), "state_dict key order differs"
        ref.load_state_dict(sd, strict=True)
        make_fullconv(ref, R, H, W)
        x = FC.make_input_hw(R, N, H, W, seed=xseed)
        with torch.no_grad():
            y = ref(x.clone())
        y_or = FC.generator_forward_fc(sd, x, R)
        err = float((y - y_or).abs().max())
        print("R=%d N=%d %dx%d  ref-vs-oracle max-abs = %.3e  |y|max=%.3f" % (R, N, H, W, err, float(y.abs().max())))
        assert tuple(y.shape) == (N, 3, H, W)
        assert err <= 1e-5, "the oracle's fully convolutional form does not reproduce the reference"
        rows = FC.fixture_rows(H)
        out["case%d_y" % i] = np.ascontiguousarray(y[:, :, rows].numpy().astype(np.float32))
        out["case%d_rows" % i] = rows.numpy()
        out["case%d_meta" % i] = np.array([R, N, H, W, wseed, xseed], np.int64)
        out["case%d_w_checksum" % i] = np.float64(sum(float(v.double().abs().sum()) for v in sd.values()))
        out["case%d_x_checksum" % i] = np.float64(float(x.double().abs().sum()))
    out["num_cases"] = np.int64(len(CASES))
    path = os.path.join(HERE, "fullconv.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))
    assert os.path.getsize(path) < 1000000, "fixtures stay below 1 MB"


if __name__ == "__main__":
    main()
