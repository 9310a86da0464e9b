"""Run an UNMODIFIED reference script with the H100 generator swapped in.

    PYTHONPATH=/path/to/MI-GAN:/path/to/this/repo python -m migan_b200.dropin scripts.demo \
        --model-name migan-512 --model-path models/migan_512_places2.pt \
        --images-dir examples/places2_512_object/images --masks-dir examples/places2_512_object/masks \
        --output-dir out --device cuda

The reference scripts import the generator as
`from lib.model_zoo.migan_inference import Generator as MIGAN` (scripts/demo.py:15,
scripts/evaluate_fid_lpips.py:21).  This launcher imports that module from the reference checkout,
rebinds its `Generator` attribute to `migan_b200.Generator` and then runs the requested script as
`__main__` -- no file of the reference is edited.
"""
from __future__ import annotations

import importlib
import runpy
import sys


def install() -> None:
    """Patch `lib.model_zoo.migan_inference.Generator` (the reference must be importable), the Co-Mod-GAN modules,
    when pytorch_fid is importable its InceptionV3 and calculate_frechet_distance, and when lpips is importable its
    LPIPS."""
    import migan_b200

    ref_mod = importlib.import_module("lib.model_zoo.migan_inference")
    ref_mod.ReferenceGenerator = ref_mod.Generator   # keep the original reachable for A/B comparisons
    ref_mod.Generator = migan_b200.Generator
    # Co-Mod-GAN (scripts/demo.py:16-21 imports Generator / Mapping / Encoder / Synthesis from lib.model_zoo.comodgan)
    from migan_b200 import comodgan

    ref_cm = importlib.import_module("lib.model_zoo.comodgan")
    for name in ("Generator", "Mapping", "Encoder", "Synthesis"):
        setattr(ref_cm, "Reference" + name, getattr(ref_cm, name))
        setattr(ref_cm, name, getattr(comodgan, name))
    _install_fid()
    _install_lpips()


def _install_fid() -> None:
    """FID: scripts/evaluate_fid_lpips.py imports InceptionV3 and calculate_frechet_distance from pytorch_fid."""
    try:
        fid_inception = importlib.import_module("pytorch_fid.inception")
        fid_score = importlib.import_module("pytorch_fid.fid_score")
    except ImportError:
        return
    from migan_b200 import fid

    fid_inception.ReferenceInceptionV3 = fid_inception.InceptionV3
    fid_inception.InceptionV3 = fid.InceptionV3
    fid_score.ReferenceInceptionV3 = fid_score.InceptionV3
    fid_score.InceptionV3 = fid.InceptionV3
    fid_score.calculate_frechet_distance = fid.calculate_frechet_distance


def _install_lpips() -> None:
    """LPIPS: scripts/evaluate_fid_lpips.py does `import lpips` and calls `lpips.LPIPS(net="alex")`."""
    try:
        ref_lpips = importlib.import_module("lpips")
    except ImportError:
        return
    from migan_b200 import lpips

    ref_lpips.ReferenceLPIPS = ref_lpips.LPIPS
    ref_lpips.LPIPS = lpips.LPIPS


def main(argv=None) -> None:
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        raise SystemExit("usage: python -m migan_b200.dropin <reference module, e.g. scripts.demo> [script args...]")
    install()
    sys.argv = [argv[0]] + argv[1:]
    runpy.run_module(argv[0], run_name="__main__", alter_sys=True)


if __name__ == "__main__":
    main()
