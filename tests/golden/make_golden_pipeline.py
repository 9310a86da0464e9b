"""Pin oracle/pipeline_oracle.py against the reference's own ``MIGAN_Pipeline`` (scripts/create_onnx_pipeline.py:121-264) and
write tests/golden/pipeline.npz.  Needs a checkout of the reference (MIGAN_REF) and torchvision; the class does not use its
module's cv2 / onnxruntime imports, which are stubbed.

Every case records the inputs' SEED (the tests regenerate image / mask with ``case_inputs`` below), the crop window, the
model input x, the reference generator's output y and the final image -- all produced by the reference; the oracle must
reproduce each of them bit for bit before the file is written.
"""
import importlib.machinery
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("MIGAN_REF", "../MI-GAN")   # a checkout of the reference project
sys.path.insert(0, ROOT)

# (tag, res, padding, H, W, mask H, mask W, hole rows, hole cols, extra)
CASES = [
    ("down", 64, 16, 150, 210, 150, 210, (40, 110), (60, 190), "gray"),     # crop = whole image, both axes shrink (420 -> 256 style)
    ("corner", 64, 16, 200, 260, 200, 260, (0, 9), (250, 260), ""),         # small hole in a corner: 64-pixel crop clipped to the border, identity resize
    ("up", 64, 16, 50, 45, 50, 45, (10, 30), (5, 40), ""),                   # image smaller than the model resolution: up-sampling both ways
    ("mixed", 64, 16, 64, 300, 64, 300, (20, 40), (100, 240), ""),          # height already at the model resolution (that pass is skipped)
    ("maskres", 64, 16, 120, 100, 60, 50, (10, 40), (10, 30), "gray"),      # mask at half the image size (nearest resize first)
    ("nohole", 64, 16, 90, 130, 90, 130, None, None, ""),                   # nothing to fill
    ("r256", 256, 128, 300, 420, 300, 420, (100, 180), (150, 330), ""),     # the deployed configuration (resolution 256, padding 128)
]


def case_inputs(case):
    tag, res, pad, H, W, MH, MW, rows, cols, extra = case
    rng = np.random.RandomState(sum(map(ord, tag)))
    image = rng.randint(0, 256, size=(1, 3, H, W), dtype=np.uint8)
    mask = np.full((1, 1, MH, MW), 255, dtype=np.uint8)
    if rows is not None:
        mask[:, :, rows[0]:rows[1], cols[0]:cols[1]] = 0
    if extra == "gray":      # values other than 0 / 255 count as hole for the box and blend partially
        mask[:, :, MH // 2, : MW // 3] = 128
        mask[:, :, 3, 5] = 254
    return torch.from_numpy(image), torch.from_numpy(mask)


def load_fixture():
    """pipeline.npz + pipeline_r256.npz (the r256 request, stored apart by shrink_golden.py) as one dict."""
    here = os.path.dirname(os.path.abspath(__file__))
    gold = {}
    for name in ("pipeline.npz", "pipeline_r256.npz"):
        z = np.load(os.path.join(here, name))
        gold.update({k: z[k] for k in z.files})
    return gold


def on_stored_rows(gold, key, tag, a):
    """`a` (a full x or final image of request `tag`) restricted to the rows the fixture stores for it."""
    rows = gold.get(("rows_" if key == "x" else "frows_") + tag)
    return a if rows is None else a[:, :, rows]


def main():
    for name in ("cv2", "onnxruntime"):
        if name not in sys.modules:
            stub = types.ModuleType(name)
            stub.__spec__ = importlib.machinery.ModuleSpec(name, None)
            sys.modules[name] = stub
    sys.path.insert(0, REF)
    from scripts import create_onnx_pipeline as cop
    from oracle import pipeline_oracle as PO
    import migan_b200
    from migan_b200 import synthetic

    out = {}
    pipes = {}
    for case in CASES:
        tag, res, pad = case[0], case[1], case[2]
        if res not in pipes:
            sd = synthetic.export_style_state_dict(res, seed=11)
            with tempfile.NamedTemporaryFile(suffix=".pt") as f:
                torch.save(sd, f.name)
                pipes[res] = cop.MIGAN_Pipeline(f.name, res, padding=pad)
        pipe = pipes[res]
        pipe.padding = torch.tensor(pad)
        image, mask = case_inputs(case)
        with torch.no_grad():
            # the reference, stage by stage (the same calls as MIGAN_Pipeline.forward, :250-264) ...
            import torchvision.transforms.functional as tvF
            from PIL import Image
            m = tvF.resize(mask, (image.size(2), image.size(3)), interpolation=Image.NEAREST)
            x0, x1, y0, y1 = [int(v) for v in pipe.get_masked_bbox(m)]
            ci, cm = image[:, :, y0:y1, x0:x1], m[:, :, y0:y1, x0:x1]
            x_ref = pipe.preprocess(ci, cm)
            y_ref = pipe.model(x_ref)
            post_ref = pipe.postprocess(ci, cm, y_ref)
            final_ref = pipe(image.clone(), mask)
            # ... and the oracle
            taps = {}
            final_or = PO.forward(pipe.model, image.clone(), mask, res, pad, taps)
        assert taps["box"] == (x0, x1, y0, y1), (tag, taps["box"], (x0, x1, y0, y1))
        assert torch.equal(taps["x"], x_ref), tag
        assert torch.equal(taps["post"], post_ref), tag
        assert torch.equal(final_or, final_ref), tag
        assert torch.equal(final_ref[:, :, y0:y1, x0:x1], post_ref), tag
        print("pipeline case %-8s %dx%d -> box x[%d,%d) y[%d,%d)  pinned bit-exact (box, x, composite, final image)" % (tag, image.size(2), image.size(3), x0, x1, y0, y1))
        out["box_" + tag] = np.array([x0, x1, y0, y1], np.int32)
        out["x_" + tag] = x_ref.numpy()
        out["y_" + tag] = y_ref.numpy()
        out["final_" + tag] = final_ref.numpy()
    # the bounding-box arithmetic alone on random masks (cheap, many shapes)
    rng = np.random.RandomState(5)
    boxes = []
    pipe = pipes[64]
    for t in range(300):
        H, W = int(rng.randint(8, 400)), int(rng.randint(8, 400))
        mask = np.full((H, W), 255, np.uint8)
        for _ in range(int(rng.randint(0, 3))):
            a, b = sorted(rng.randint(0, H, 2)); c, d = sorted(rng.randint(0, W, 2))
            mask[a:b + 1, c:d + 1] = rng.choice([0, 0, 128, 254])
        pad = int(rng.choice([0, 5, 16, 128]))
        pipe.padding = torch.tensor(pad)
        ref = tuple(int(v) for v in pipe.get_masked_bbox(torch.from_numpy(mask)[None, None]))
        assert PO.masked_bbox(mask, 64, pad) == ref, (t, ref)
        boxes.append([H, W, pad, *ref])
    out["bbox_cases"] = np.array(boxes, np.int32)      # the masks are regenerated from seed 5 by the test
    print("masked_bbox pinned on 300 random masks")
    # the weight table against the weights torch applies (impulse responses)
    import torch.nn.functional as F
    for (L, O) in [(256, 420), (420, 256), (300, 256), (257, 256), (1920, 512), (50, 64), (64, 50)]:
        eye = torch.eye(L).view(1, L, 1, L)
        wt = F.interpolate(eye, size=(1, O), mode="bilinear", align_corners=False, antialias=True)[0, :, 0, :].numpy()
        xmin, xsize, w = PO.aa_weights(L, O)
        mine = np.zeros((L, O), np.float32)
        for i in range(O):
            mine[xmin[i]:xmin[i] + xsize[i], i] = w[i, :xsize[i]]
        assert np.array_equal(wt, mine), (L, O)
    print("aa_weights equals the weights torch applies (7 size pairs)")
    np.savez_compressed(os.path.join(HERE, "pipeline.npz"), **out)
    print("wrote", os.path.join(HERE, "pipeline.npz"), os.path.getsize(os.path.join(HERE, "pipeline.npz")), "bytes")


if __name__ == "__main__":
    main()
