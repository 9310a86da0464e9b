"""Host-side logic and the C-ABI surface, no GPU needed."""
import ctypes
import os
import re
import sys

import pytest
import torch

import migan_b200
from migan_b200 import _abi, arch
from oracle import migan_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol(lib):
    header = open(os.path.join(ROOT, "include", "migan_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b((?:migan|b200)_[a-z0-9_]+)\s*\(", header))
    bound = {name for name, _, _ in _abi.SYMBOLS}
    assert declared == bound, declared ^ bound
    for name in declared:
        assert hasattr(lib, name)
    assert b"sm_90a" in lib.migan_version()


@pytest.mark.parametrize("R", [8, 64, 256, 512])
def test_state_dict_layout_matches_reference_order(lib, R):
    """Python module, C registry and the oracle spec (checked against the real reference by
    make_golden.py with strict=True) all agree on names, order and shapes."""
    spec = O.state_dict_spec(R)
    g = migan_b200.Generator(R)
    sd = g.state_dict()
    assert list(sd.keys()) == list(spec.keys())
    assert all(tuple(sd[k].shape) == tuple(spec[k]) for k in spec)
    h = ctypes.c_void_p()
    _abi.check(lib.migan_create(R, -1, ctypes.byref(h)))
    try:
        assert lib.migan_num_weights(h) == len(spec)
        for i, (k, shape) in enumerate(spec.items()):
            nm, nd, sh = ctypes.c_char_p(), ctypes.c_int(), (ctypes.c_int64 * 4)()
            _abi.check(lib.migan_weight_info(h, i, ctypes.byref(nm), ctypes.byref(nd), sh))
            assert nm.value.decode() == k and tuple(sh[: nd.value]) == tuple(shape)
        assert lib.migan_workspace_bytes(h, 2) > lib.migan_workspace_bytes(h, 1) > 0
    finally:
        lib.migan_destroy(h)


def test_param_vs_buffer_split_and_attribute_paths():
    g = migan_b200.Generator(256)
    assert sum(p.numel() for p in g.parameters()) == 5943617      # SURVEY.md section 6
    bufs = dict(g.named_buffers())
    assert "synthesis.b64.conv1.noise_const" in bufs and "synthesis.b64.upsample.filter_const" in bufs
    assert g.encoder.b256.fromrgb.weight.shape == (128, 4, 1, 1)
    assert g.synthesis.b8.conv1.use_noise and not g.synthesis.b4.conv2.use_noise
    assert g.encoder.b64.conv2.downsample.filter.weight.shape == (512, 1, 4, 4)
    # a reference state_dict (seeded stand-in) loads strictly
    g.load_state_dict(O.make_state_dict(256), strict=True)


def test_constructor_and_cpu_errors(lib):
    with pytest.raises(ValueError):
        migan_b200.Generator(96)          # reference raises ValueError (migan_inference.py:215-216)
    g = migan_b200.Generator(64)
    with pytest.raises(RuntimeError, match="no CPU"):
        g(torch.zeros(1, 4, 64, 64))
    h = ctypes.c_void_p()
    assert lib.migan_create(96, -1, ctypes.byref(h)) == _abi.ERR_INVALID
    assert b"power of two" in lib.migan_last_error()
    _abi.check(lib.migan_create(64, -1, ctypes.byref(h)))
    w = torch.zeros(7)
    assert lib.migan_set_weight(h, b"no.such.key", w.data_ptr(), 7) == _abi.ERR_INVALID
    assert lib.migan_set_weight(h, b"encoder.b64.fromrgb.bias", w.data_ptr(), 7) == _abi.ERR_INVALID
    assert lib.migan_finalize_weights(h) == _abi.ERR_CUDA        # description-only context cannot compute
    lib.migan_destroy(h)


def test_no_cuda_device_fails_loudly(lib):
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    h = ctypes.c_void_p()
    assert lib.migan_create(64, 0, ctypes.byref(h)) == _abi.ERR_CUDA
    assert b"no CPU path" in lib.migan_last_error()


def test_product_does_not_import_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py's checker / CPU legs may touch oracle/: not the package, not tools/."""
    for top in ("mi-gan_b200", "tools", "include"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, top)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".h", ".sh")):
                    src = open(os.path.join(dirpath, f)).read()
                    assert "import oracle" not in src and "from oracle" not in src, f


def test_arch_helpers():
    assert arch.encoder_resolutions(256) == [256, 128, 64, 32, 16, 8, 4]
    assert arch.synthesis_resolutions(64) == [4, 8, 16, 32, 64]
    assert [arch.nf(r) for r in (512, 256, 128, 64, 4)] == [64, 128, 256, 512, 512]


# --------------------------------------------------------------------------- #
# Co-Mod-GAN boundary (include/comodgan_b200.h, migan_b200.comodgan)
# --------------------------------------------------------------------------- #
def test_library_exports_every_comodgan_symbol(lib):
    header = open(os.path.join(ROOT, "include", "comodgan_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b((?:comodgan|b200)_[a-z0-9_]+)\s*\(", header))
    bound = {name for name, _, _ in _abi.COMOD_SYMBOLS}
    assert declared == bound, declared ^ bound
    for name in declared:
        assert hasattr(lib, name)


@pytest.mark.parametrize("R", [16, 256, 512])
def test_comodgan_state_dict_layout_matches_reference_order(lib, R):
    """Python modules, C registry and the oracle spec (checked against the real reference by
    make_golden_comodgan.py with strict=True) agree on names, order and shapes."""
    from migan_b200 import comodgan
    from oracle import comodgan_oracle as C
    spec = C.state_dict_spec(R)
    g = comodgan.Generator(comodgan.Mapping(num_ws=C.num_ws(R)), comodgan.Encoder(resolution=R),
                           comodgan.Synthesis(resolution=R))
    sd = g.state_dict()
    assert list(sd.keys()) == list(spec.keys())
    for k, shape in spec.items():
        assert tuple(sd[k].shape) == tuple(shape), k
    params = {k for k, _ in g.named_parameters()}
    assert "mapping.w_avg" not in params and "synthesis.b4.conv.noise_const" not in params
    assert "synthesis.b4.conv.noise_strength" in params and "encoder.b4.fc.weight" in params
    g.load_state_dict(C.make_state_dict(R) if R == 16 else sd, strict=True)
    assert g.num_ws == C.num_ws(R) and g.img_resolution == R and g.z_dim == 512


def test_comodgan_constructor_and_cpu_errors(lib):
    from migan_b200 import comodgan
    with pytest.raises(ValueError):
        comodgan.Encoder(resolution=48)
    with pytest.raises(ValueError):     # num_ws mismatch (stylegan.py:580-581)
        comodgan.Generator(comodgan.Mapping(num_ws=16), comodgan.Encoder(resolution=256), comodgan.Synthesis(resolution=256))
    g = comodgan.Generator(comodgan.Mapping(num_ws=6), comodgan.Encoder(resolution=16), comodgan.Synthesis(resolution=16))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        g(torch.zeros(1, 4, 16, 16))
    with pytest.raises(RuntimeError, match="shape"):
        g(torch.zeros(1, 3, 16, 16))
    h = ctypes.c_void_p()
    assert lib.comodgan_create(16, -1, ctypes.byref(h)) == 0
    assert lib.comodgan_finalize_weights(h) != 0        # no device, no weights: fails loudly
    lib.comodgan_destroy(h)


EXPORT_GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "export.npz")   # tests/golden/make_golden_export.py


def test_dropin_rebinds_reference_modules(lib, monkeypatch, tmp_path):
    """python -m migan_b200.dropin scripts.demo ...: the reference's import sites (scripts/demo.py:15-21) resolve to the
    H100 classes without editing any reference file.  The reference's modules are stood in for by stubs with the same
    names; the model built through the patched names has the reference's Co-Mod-GAN state_dict keys (stored)."""
    import importlib
    import numpy as np
    pkg = tmp_path / "lib" / "model_zoo"
    pkg.mkdir(parents=True)
    (tmp_path / "lib" / "__init__.py").write_text("")
    (pkg / "__init__.py").write_text("")
    (pkg / "migan_inference.py").write_text("class Generator:\n    pass\n")
    (pkg / "comodgan.py").write_text("".join("class %s:\n    pass\n" % c for c in ("Generator", "Mapping", "Encoder", "Synthesis")))
    for name in [m for m in sys.modules if m == "lib" or m.startswith("lib.")]:
        monkeypatch.delitem(sys.modules, name)
    monkeypatch.syspath_prepend(str(tmp_path))
    from migan_b200 import comodgan, dropin
    ref_mi = importlib.import_module("lib.model_zoo.migan_inference")
    ref_cm = importlib.import_module("lib.model_zoo.comodgan")
    saved = (ref_mi.Generator, ref_cm.Generator)
    dropin.install()
    assert ref_mi.Generator is migan_b200.Generator and ref_mi.ReferenceGenerator is saved[0]
    assert ref_cm.Generator is comodgan.Generator and ref_cm.ReferenceGenerator is saved[1]
    # the construction of scripts/demo.py:95-100, through the patched names
    model = ref_cm.Generator(ref_cm.Mapping(num_ws=14), ref_cm.Encoder(resolution=256), ref_cm.Synthesis(resolution=256))
    assert list(model.state_dict().keys()) == [str(k) for k in np.load(EXPORT_GOLD)["dropin_comodgan_keys"]]


def test_resolutions_above_512_are_rejected_up_front(lib):
    """min(32768 // R, 512) drops below 64 channels for R > 512: not built (no released model); fail at create, not mid-forward.
    A description-only context (device -1: names and shapes) is still available."""
    h = ctypes.c_void_p()
    assert lib.migan_create(1024, 0, ctypes.byref(h)) == 1 and b"64 channels" in lib.migan_last_error()
    assert lib.migan_create(1024, -1, ctypes.byref(h)) == 0
    lib.migan_destroy(h)


def _emul_reparam(ws):
    """The export kernel's functor compiled for the host (tests/emul), on numpy copies of the tensors."""
    import numpy as np
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul"))
    import build_emul
    emul = ctypes.CDLL(build_emul.build())
    emul.b200_reparam_filter.restype = ctypes.c_int
    emul.b200_reparam_filter.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]
    arrs = [np.ascontiguousarray(w.detach().numpy(), dtype=np.float32) for w in ws]
    out = np.empty_like(arrs[0])
    ptrs = (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    assert emul.b200_reparam_filter(ctypes.cast(ptrs, ctypes.c_void_p), len(arrs), arrs[0].shape[0], arrs[0][0].size,
                                    out.ctypes.data_as(ctypes.c_void_p), None) == 0
    return torch.from_numpy(out)


def test_export_kernel_matches_oracle_in_emulation():
    """csrc/reparam.cu (host-emulation build) against oracle/export_oracle.merged_filter: depthwise 3x3, 1x1 and k = 1 / 9 tensors.
    Bar: relative error < 1e-6 of the filter's largest tap (the sum of squares is accumulated in fp64 instead of torch's fp32 tree)."""
    from oracle import export_oracle as E
    g = torch.Generator().manual_seed(3)
    for shape, k in (((64, 1, 3, 3), 9), ((128, 64, 1, 1), 9), ((3, 512, 1, 1), 1), ((512, 512, 1, 1), 4), ((64, 4, 1, 1), 1)):
        ws = [torch.randn(shape, generator=g) * (0.5 + i) for i in range(k)]
        got, want = _emul_reparam(ws), E.merged_filter(ws)
        assert got.shape == want.shape
        err = (got - want).abs().amax(dim=(1, 2, 3)) / want.abs().amax(dim=(1, 2, 3))
        assert float(err.max()) < 1e-6, (shape, k, float(err.max()))
        assert torch.allclose(got.flatten(1).square().sum(1), torch.ones(shape[0]), atol=1e-5)   # unit L2 filters


def test_export_matches_reference_copy_weights():
    """oracle/export_oracle.merged_filter == the reference's `get_source_w` (through its effect: `copy_weights` of a seeded
    re-parameterised migan-64 training Generator into the reference's inference Generator), and the export kernel
    (emulation) reproduces those filters.  Stored vectors: a sample of filters of 25 of its 46 convolutions, every kind."""
    import numpy as np
    from oracle import export_oracle as E
    gold = np.load(EXPORT_GOLD)
    names = sorted(k[:-len(".want")] for k in gold.files if k.endswith(".want"))
    for name in names:
        ws = list(torch.from_numpy(gold[name + ".ws"]))
        want = torch.from_numpy(gold[name + ".want"])
        assert torch.equal(E.merged_filter(ws), want), name             # the oracle IS the reference expression
        got = _emul_reparam(ws)
        assert float(((got - want).abs().amax(dim=(1, 2, 3)) / want.abs().amax(dim=(1, 2, 3))).max()) < 1e-6, name
    kinds = {n.rsplit(".", 1)[-1] if n.endswith(("fromrgb", "torgb")) else n.rsplit(".", 1)[-1] + str(gold[n + ".want"].shape[2:]) for n in names}
    assert len(names) == 25 and kinds == {"fromrgb", "torgb", "conv1(3, 3)", "conv2(1, 1)"}
