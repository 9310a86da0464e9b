"""Generate the committed golden fixtures by running the REAL reference.

Run in the build container only (needs a checkout of the reference, MIGAN_REF, which does not exist on the
GPU box):   python tests/golden/make_golden.py

For each case it
  1. builds the reference ``lib.model_zoo.migan_inference.Generator(R)``,
  2. loads the oracle's seeded state_dict with ``strict=True`` (so key names, order
     and shapes are checked against the reference),
  3. runs the reference forward and the oracle forward on the same input and
     asserts they agree exactly (this is what pins the oracle),
  4. stores the reference output + a few intermediate statistics in
     ``tests/golden/migan_R{R}_n{N}.npz`` (float32; weights/inputs are regenerated
     from seeds, their checksums are stored to detect RNG drift).
It also pins the op-level oracles (upfirdn2d / bias_act) against the reference's own
``impl='ref'`` functions and stores small vectors for them.
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

from oracle import migan_oracle as O  # noqa: E402


def checksum(t: torch.Tensor) -> float:
    return float(t.double().abs().sum())


def main():
    from lib.model_zoo.migan_inference import Generator as RefGenerator
    from torch_utils.ops import upfirdn2d as ref_upfirdn2d
    from torch_utils.ops import bias_act as ref_bias_act

    torch.manual_seed(0)
    cases = [(64, 2, 1, 1234), (256, 1, 1, 1234), (512, 1, 1, 1234), (256, 2, 7, 99)]
    for R, N, wseed, xseed in cases:
        ref = RefGenerator(resolution=R).eval()
        sd = O.make_state_dict(R, seed=wseed)
        assert list(ref.state_dict().keys()) == list(sd.keys()), "state_dict key order differs"
        ref.load_state_dict(sd, strict=True)
        x = O.make_input(R, N, seed=xseed)
        with torch.no_grad():
            y_ref = ref(x.clone())
        taps = {}
        y_or = O.generator_forward(sd, x, R, taps=taps)
        err = float((y_ref - y_or).abs().max())
        print("R=%d N=%d  ref-vs-oracle max-abs = %.3e   |y|max=%.3f  |y|mean=%.3f"
              % (R, N, err, float(y_ref.abs().max()), float(y_ref.abs().mean())))
        assert err == 0.0, "oracle does not reproduce the reference"
        y64 = O.generator_forward(sd, x, R, dtype=torch.float64)
        f64err = float((y_ref.double() - y64).abs().max())
        print("    fp32 reference vs fp64 oracle max-abs = %.3e" % f64err)
        tap_stats = {}
        for k in ("encoder.b%d.conv1.out" % R, "encoder.b%d.conv2.out" % R, "encoder.b4.conv2.out",
                  "synthesis.b4.conv2.out", "synthesis.b%d.conv1.out" % R, "synthesis.b%d.conv2.out" % R):
            tap_stats[k] = np.array([checksum(taps[k]), float(taps[k].abs().max())])
        np.savez_compressed(
            os.path.join(HERE, "migan_R%d_n%d_w%d.npz" % (R, N, wseed)),
            y=y_ref.numpy(), resolution=R, n=N, wseed=wseed, xseed=xseed,
            x_checksum=checksum(x), w_checksum=sum(checksum(v) for v in sd.values()),
            fp64_maxabs=f64err, tap_names=np.array(list(tap_stats.keys())),
            tap_stats=np.stack(list(tap_stats.values())))

    # op-level pins ---------------------------------------------------------
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 5, 9, 12, generator=g)
    f2 = ref_upfirdn2d.setup_filter([1, 3, 3, 1])
    assert torch.equal(f2, O.setup_filter([1, 3, 3, 1]))
    f1 = torch.tensor([1., 2., 4., 2., 1., .5, .25, .125]) / 10.875
    up_cases = []
    for (f, up, down, pad, flip, gain) in [
        (f2, 1, 1, (1, 2, 2, 1), False, 1.0), (f2, 2, 1, (2, 1, 2, 1), False, 4.0),
        (f2, 1, 2, (1, 1, 1, 1), False, 1.0), (f2, 2, 2, (3, 0, 1, 2), True, 2.0),
        (f1, 1, 1, (4, 3, 4, 3), False, 1.0), (f1, 2, 1, (5, 4, 5, 4), True, 4.0),
        (None, 1, 1, (0, 0, 0, 0), False, 1.0), (f2, 1, 1, (-1, 2, 3, -1), False, 1.0),
    ]:
        a = ref_upfirdn2d.upfirdn2d(x, f, up=up, down=down, padding=list(pad), flip_filter=flip, gain=gain, impl="ref")
        b = O.upfirdn2d_ref(x, f, up=up, down=down, padding=pad, flip_filter=flip, gain=gain)
        assert torch.equal(a, b), "upfirdn2d oracle mismatch"
        up_cases.append(a.numpy().ravel())
    acts = list(O._ACT.keys())
    ba_cases = []
    bvec = torch.randn(5, generator=g)
    for act in acts:
        for clamp in (None, 0.7):
            a = ref_bias_act.bias_act(x, bvec, dim=1, act=act, clamp=clamp, impl="ref")
            b = O.bias_act_ref(x, bvec, dim=1, act=act, clamp=clamp)
            assert torch.equal(a, b), "bias_act oracle mismatch " + act
            ba_cases.append(a.numpy().ravel())
    np.savez_compressed(os.path.join(HERE, "ops.npz"), x=x.numpy(), bvec=bvec.numpy(), f1=f1.numpy(),
                        **{"up%d" % i: v for i, v in enumerate(up_cases)},
                        **{"ba%d" % i: v for i, v in enumerate(ba_cases)})
    # Upsample2d / Downsample2d modules == upfirdn2d ref (SURVEY 8c pin 2)
    from lib.model_zoo.migan_inference import Upsample2d, Downsample2d
    xx = torch.randn(1, 3, 8, 8, generator=g)
    a = Upsample2d(3, resolution=16)(xx)
    b = O.upfirdn2d_ref(xx, f2, up=2, padding=(2, 1, 2, 1), gain=4.0)
    print("Upsample2d vs upfirdn2d_ref max-abs", float((a - b).abs().max()))
    a = Downsample2d(3)(xx)
    b = O.upfirdn2d_ref(xx, f2, down=2, padding=(1, 1, 1, 1))
    print("Downsample2d vs upfirdn2d_ref max-abs", float((a - b).abs().max()))
    print("golden fixtures written to", HERE)


if __name__ == "__main__":
    main()
