"""Pin oracle/prepost_oracle.preprocess against the reference's own scripts/demo.py:preprocess (build container only)."""
import os
import sys

import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("MIGAN_REF", "../MI-GAN")   # a checkout of the reference project
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

from oracle import prepost_oracle as P  # noqa: E402


def main():
    from scripts.demo import preprocess as ref_preprocess
    rng = np.random.RandomState(3)
    for R in (64, 256):
        img = rng.randint(0, 256, size=(R, R, 3), dtype=np.uint8)
        mask = (rng.rand(R, R) > 0.4).astype(np.uint8) * 255
        mask[0, :5] = [0, 1, 127, 254, 255]                     # only 255 counts as known (`// 255`)
        x_ref = ref_preprocess(Image.fromarray(img), Image.fromarray(mask).convert("L"), R)
        x_or = P.preprocess(img[None], mask[None])
        assert x_ref.shape == x_or.shape and torch.equal(x_ref, x_or), R
        print("preprocess R=%d pinned bit-exact" % R)
    # post-processing vector (restatement only; see the oracle header)
    g = torch.Generator().manual_seed(5)
    y = torch.randn(2, 3, 32, 32, generator=g) * 1.5
    y[0, 0, 0, :6] = torch.tensor([-1.0, 1.0, 0.0, 0.99999994, -1.0000001, 0.00392157 * 2 - 1])
    img = rng.randint(0, 256, size=(2, 32, 32, 3), dtype=np.uint8)
    mask = (rng.rand(2, 32, 32) > 0.5).astype(np.uint8) * 255
    np.savez_compressed(os.path.join(HERE, "prepost.npz"), y=y.numpy(), img=img, mask=mask,
                        x=P.preprocess(img, mask).numpy(), out=P.postprocess(y, img, mask))


def pin_feather():
    """oracle feather_composite == MIGAN_Pipeline.postprocess of scripts/create_onnx_pipeline.py (its cv2 / onnxruntime imports are
    not needed by the class and are stubbed).  Writes tests/golden/feather.npz."""
    import types
    import importlib.machinery
    for name in ("cv2", "onnxruntime"):
        if name not in sys.modules:
            stub = types.ModuleType(name)
            stub.__spec__ = importlib.machinery.ModuleSpec(name, None)
            sys.modules[name] = stub
    from scripts import create_onnx_pipeline as cop

    class _Pipe:   # the two attributes postprocess uses
        gaussian_blur = cop.GaussianSmoothing(channels=1, kernel_size=5, sigma=1.0, dim=2)
    assert torch.equal(_Pipe.gaussian_blur.weight[0, 0], P.gaussian_kernel_5x5())
    rng = np.random.RandomState(21)
    g = torch.Generator().manual_seed(22)
    cases = {}
    for tag, (H, W) in (("a", (48, 64)), ("b", (40, 40))):
        image = torch.from_numpy(rng.randint(0, 256, size=(1, 3, H, W), dtype=np.uint8))
        mask = torch.full((1, 1, H, W), 255, dtype=torch.uint8)
        mask[:, :, H // 4: H // 2, W // 3: W - 5] = 0            # a hole away from the border
        mask[:, :, :3, :7] = 0                                    # and one touching it (reflect padding matters)
        mask[:, :, H - 2:, W - 9:] = 0
        y = torch.randn(1, 3, H, W, generator=g) * 0.8
        ref = cop.MIGAN_Pipeline.postprocess(_Pipe, image, mask, y)
        mine = P.feather_composite(image, mask, y)
        assert torch.equal(ref, mine), tag
        cases.update({"image_" + tag: image.numpy(), "mask_" + tag: mask.numpy(), "y_" + tag: y.numpy(), "out_" + tag: ref.numpy()})
        print("feather composite %dx%d pinned bit-exact against MIGAN_Pipeline.postprocess" % (H, W))
    np.savez_compressed(os.path.join(HERE, "feather.npz"), **cases)


if __name__ == "__main__":
    main()
    pin_feather()
