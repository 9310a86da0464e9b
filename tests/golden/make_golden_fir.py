"""Generate tests/golden/fir.npz: the REAL reference with random asymmetric FIR taps.

Run where a checkout of the reference exists (MIGAN_REF; not on the GPU box):
    python tests/golden/make_golden_fir.py

The `*.filter.weight` taps of the reference are parameters (migan_inference.py:72, :96), so a trained checkpoint may
carry any values there.  Every other fixture uses the constructor's [1,3,3,1] filter, which is symmetric, separable and
the same for every channel: a kernel that flips the taps, swaps their axes or reads one channel's taps for all channels
still matches it.  For each case this
  1. builds the reference ``lib.model_zoo.migan_inference.Generator(R)`` and loads the oracle's seeded state_dict with
     asymmetric taps (`make_state_dict(..., fir=...)`) with ``strict=True``,
  2. for the fully convolutional case, applies make_golden_fullconv.py's two buffer replacements to the module tree,
  3. runs the reference forward, asserts the oracle gives exactly the same output, and stores y (in full at R = 64,
     otherwise on the rows `fixture_rows(H, period=16)` keeps) with the seeds, shapes and weight / input checksums.
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
sys.path.insert(0, HERE)

from make_golden_fullconv import make_fullconv  # noqa: E402
from oracle import fullconv_oracle as FC  # noqa: E402
from oracle import migan_oracle as O  # noqa: E402

# (R, N, H, W, fir, weight seed, input seed, full output?)
CASES = [(64, 2, 64, 64, "per_channel", 1, 1234, True),
         (256, 1, 256, 256, "per_channel", 1, 1234, False),
         (256, 1, 256, 256, "uniform", 1, 1234, False),
         (256, 1, 320, 448, "per_channel", 1, 5, False)]


def main():
    from lib.model_zoo.migan_inference import Generator as RefGenerator

    out = {}
    for i, (R, N, H, W, fir, wseed, xseed, full) in enumerate(CASES):
        ref = RefGenerator(resolution=R).eval()
        sd = O.make_state_dict(R, seed=wseed, fir=fir)
        assert list(ref.state_dict().keys()) == list(sd.keys()), "state_dict key order differs"
        ref.load_state_dict(sd, strict=True)
        if (H, W) != (R, R):
            make_fullconv(ref, R, H, W)
        x = FC.make_input_hw(R, N, H, W, seed=xseed)
        with torch.no_grad():
            y = ref(x.clone())
        y_or = FC.generator_forward_fc(sd, x, R)
        err = float((y - y_or).abs().max())
        print("R=%d N=%d %dx%d fir=%s  ref-vs-oracle max-abs = %.3e  |y|max=%.3f" % (R, N, H, W, fir, err, float(y.abs().max())))
        assert tuple(y.shape) == (N, 3, H, W)
        assert err == 0.0, "the oracle does not reproduce the reference"
        rows = np.arange(H) if full else FC.fixture_rows(H, period=16).numpy()
        out["case%d_y" % i] = np.ascontiguousarray(y[:, :, rows].numpy().astype(np.float32))
        out["case%d_rows" % i] = rows
        out["case%d_meta" % i] = np.array([R, N, H, W, wseed, xseed], np.int64)
        out["case%d_fir" % i] = np.array(fir)
        out["case%d_w_checksum" % i] = np.float64(sum(float(v.double().abs().sum()) for v in sd.values()))
        out["case%d_x_checksum" % i] = np.float64(float(x.double().abs().sum()))
    out["num_cases"] = np.int64(len(CASES))
    path = os.path.join(HERE, "fir.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))
    assert os.path.getsize(path) < 550000, "this fixture stays near 500 KB"


if __name__ == "__main__":
    main()
