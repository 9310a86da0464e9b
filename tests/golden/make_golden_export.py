"""Pin the reference's training-snapshot -> inference-weights export (scripts/export_inference_model.py:17-85) and its
module layout, and write tests/golden/export.npz.  Needs a checkout of the reference (MIGAN_REF, default ../MI-GAN):

    MIGAN_REF=/path/to/MI-GAN python tests/golden/make_golden_export.py

Stored, for a seeded re-parameterised migan-64 training Generator (lib/model_zoo/migan.py) exported with the reference's
own `copy_weights` into its inference Generator:
  <conv>.ws    the k re-parameterisation tensors of a sample of output filters   [k, rows, cin/groups, kh, kw]
  <conv>.want  the same filters of the exported state_dict                       [rows, cin/groups, kh, kw]
Every depthwise / fromrgb convolution keeps 8 filters, four 1x1 / torgb convolutions keep one (a filter is normalised on
its own, so a sample of filters is exact).  Also the state_dict keys of the reference's Co-Mod-GAN Generator
(`dropin_comodgan_keys`, demo construction num_ws=14 at 256) that the drop-in launcher has to reproduce.
"""
import importlib
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("MIGAN_REF", os.path.join(HERE, "..", "..", "..", "MI-GAN"))
LARGE = ("encoder.b64.conv1.conv2", "encoder.b8.conv2.conv2", "synthesis.b16.conv1.conv2", "synthesis.b64.torgb")


def main():
    sys.path.insert(0, REF)
    warnings.filterwarnings("ignore")
    M = importlib.import_module("lib.model_zoo.migan")
    ref_inf = importlib.import_module("lib.model_zoo.migan_inference")
    ref_cm = importlib.import_module("lib.model_zoo.comodgan")
    exp = importlib.import_module("scripts.export_inference_model")
    R = 64
    torch.manual_seed(1)
    src = M.Generator(M.Encoder(resolution=R, ic_n=4, depthwise=True, reparametrize=True, num_reparam_tensors=9),
                      M.Synthesis(resolution=R, depthwise=True, reparametrize=True, num_reparam_tensors=9)).eval()
    ref = ref_inf.Generator(resolution=R).eval()
    exp.copy_weights(src, ref, resolution=R)
    sd = ref.state_dict()
    out = {}
    g = torch.Generator().manual_seed(5)
    for side in ("encoder", "synthesis"):
        for res in (4, 8, 16, 32, 64):
            blk = getattr(getattr(src, side), "b%d" % res)
            convs = [("conv1.conv1", blk.conv1.conv1), ("conv1.conv2", blk.conv1.conv2), ("conv2.conv1", blk.conv2.conv1),
                     ("conv2.conv2", blk.conv2.conv2)]
            head = "fromrgb" if side == "encoder" else "torgb"
            if "%s.b%d.%s.weight" % (side, res, head) in sd:
                convs.append((head, getattr(blk, head)))
            for name, conv in convs:
                key = "%s.b%d.%s" % (side, res, name)
                ws = [getattr(conv, "w%d" % i).detach() for i in range(conv.num_reparam_tensors)] if conv.reparametrize else [conv.weight.detach()]
                want = sd[key + ".weight"]
                small = ws[0][0].numel() <= 64
                if not small and key not in LARGE:
                    continue
                rows = torch.randperm(want.shape[0], generator=g)[:8 if small else 1].sort().values
                out[key + ".ws"] = torch.stack([w[rows] for w in ws]).numpy()
                out[key + ".want"] = want[rows].numpy()
    cm = ref_cm.Generator(ref_cm.Mapping(num_ws=14), ref_cm.Encoder(resolution=256), ref_cm.Synthesis(resolution=256))
    out["dropin_comodgan_keys"] = np.array(list(cm.state_dict().keys()))
    path = os.path.join(HERE, "export.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "-", sum(1 for k in out if k.endswith(".want")), "convolutions,", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
