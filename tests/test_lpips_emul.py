"""LPIPS without a GPU: the oracle's key layout against torchvision's AlexNet, the library's host runtime in the
emulation build (weight registry, launch plan, the whole forward against the float64 oracle), the weight-file contract
and the drop-in rebinding of `lpips.LPIPS`."""
import ctypes
import os
import sys
import types
import urllib.request

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

import build_emul  # noqa: E402
import migan_b200  # noqa: E402
from migan_b200 import _abi, lpips  # noqa: E402
from oracle import lpips_oracle as O  # noqa: E402
from torchvision.models import alexnet  # noqa: E402


@pytest.fixture(scope="module")
def emul():
    path = build_emul._compile("lpips_emul", [os.path.join(build_emul.CSRC, s) for s in ("lpips_abi.cu", "abi_error.cu")])
    L = lpips.lib(ctypes.CDLL(path))
    L.migan_last_error.restype = ctypes.c_char_p
    return L


@pytest.fixture(scope="module")
def sd():
    return O.seeded_state_dict(0)


def _spec(sd):
    return [(k, tuple(v.shape)) for k, v in sd.items()]


def test_oracle_keys_map_onto_torchvision_features(sd):
    tv = {k: tuple(v.shape) for k, v in alexnet(weights=None).state_dict().items() if k.startswith("features.")}
    mapped = {}
    for k, shape in _spec(sd):
        if k.startswith("net."):
            prefix, leaf = k.rsplit(".", 1)
            mapped[O.LPIPS_TO_TORCHVISION[prefix] + "." + leaf] = shape
    assert mapped == tv   # one to one: every torchvision key once, with its shape
    assert sorted(O.LPIPS_TO_TORCHVISION.values()) == sorted("features.%d" % i for i in (0, 3, 6, 8, 10))
    assert lpips.TORCHVISION_KEYS == O.LPIPS_TO_TORCHVISION


def test_library_spec_matches_oracle(emul, sd):
    assert lpips.weight_spec(emul) == _spec(sd)
    assert len(_spec(sd)) == 17


def _ctx(L, device=0):
    h = ctypes.c_void_p()
    _abi.check(L.lpips_create(device, ctypes.byref(h)), L)
    return h


def _set(L, h, key, t):
    t = t.detach().float().contiguous()
    return L.lpips_set_weight(h, key.encode(), t.data_ptr(), t.numel())


def test_registry_refuses_bad_keys_by_name(emul, sd):
    h = _ctx(emul)
    try:
        assert _set(emul, h, "net.slice6.12.weight", torch.zeros(4)) == _abi.ERR_INVALID
        assert "net.slice6.12.weight" in emul.migan_last_error().decode()
        assert _set(emul, h, "lin2.model.1.weight", torch.zeros(1, 383, 1, 1)) == _abi.ERR_INVALID
        assert "lin2.model.1.weight" in emul.migan_last_error().decode()
        for k, v in sd.items():
            if k != "net.slice4.8.bias":
                assert _set(emul, h, k, v) == 0, emul.migan_last_error()
        assert emul.lpips_finalize_weights(h) == _abi.ERR_INVALID
        assert "net.slice4.8.bias" in emul.migan_last_error().decode()
    finally:
        emul.lpips_destroy(h)


def _hook_shapes(sd, H, W):
    """Output shape of every convolution and pool of features[:12] at H x W, by torchvision index."""
    m = O.model(sd)
    shapes = {}
    hooks = [mod.register_forward_hook(lambda mm, i, o, idx=idx: shapes.__setitem__(idx, tuple(o.shape[1:])))
             for idx, mod in enumerate(m) if isinstance(mod, (torch.nn.Conv2d, torch.nn.MaxPool2d))]
    with torch.no_grad():
        m(torch.zeros(1, 3, H, W, dtype=torch.float64))
    for h in hooks:
        h.remove()
    return shapes


@pytest.mark.parametrize("size", [(97, 131), (31, 31)])
def test_launch_plan_shapes(emul, sd, size):
    H, W = size
    plan = lpips.launch_plan(3, H, W, emul)
    assert plan[0] == "input in=2x3x3x%dx%d normalize=0 out=6x%dx%dx4" % (H, W, H, W)
    kinds = [line.split()[0] for line in plan]
    assert kinds == ["input", "conv", "distance", "pool", "conv", "distance", "pool", "conv", "distance", "conv",
                     "distance", "conv", "distance", "reduce"]
    shapes = _hook_shapes(sd, H, W)
    seen, hw = set(), []
    for line in plan:
        if line.startswith(("conv ", "pool ")):
            name = line.split()[1] if line.startswith("conv ") else line.split()[2]
            kv = dict(tok.split("=") for tok in line.split() if "=" in tok)
            oh, ow, co = map(int, kv["out"].split("x"))
            idx = int(name.rsplit(".", 1)[1])
            assert (co, oh, ow) == shapes[idx], line
            seen.add(idx)
            if line.startswith("conv "):
                hw.append(oh * ow)
    assert seen == set(shapes)
    assert plan[-1] == "reduce pairs=3 hw=%s" % ",".join(map(str, hw))


def test_sizes_below_the_minimum_are_refused(emul):
    for H, W in ((30, 31), (31, 30)):
        with pytest.raises(_abi.MiganError, match="31"):
            lpips.launch_plan(1, H, W, emul)
        h = _ctx(emul, -1)
        try:
            assert emul.lpips_workspace_bytes(h, 1, H, W) == 0
        finally:
            emul.lpips_destroy(h)


def _emul_lpips(L, sd, a, b, normalize):
    h = _ctx(L)
    try:
        for k, v in sd.items():
            _abi.check(_set(L, h, k, v), L)
        _abi.check(L.lpips_finalize_weights(h), L)
        n, _, H, W = a.shape
        nbytes = L.lpips_workspace_bytes(h, n, H, W)
        ws = (ctypes.c_uint8 * (nbytes + 256))()
        base = (ctypes.addressof(ws) + 255) // 256 * 256
        a, b = a.float().contiguous(), b.float().contiguous()
        out = torch.empty(n, dtype=torch.float32)
        per = torch.empty(5, n, dtype=torch.float32)
        _abi.check(L.lpips_forward(h, a.data_ptr(), b.data_ptr(), n, H, W, int(normalize), out.data_ptr(), per.data_ptr(),
                                   base, nbytes, None), L)
        assert L.lpips_last_launch_count(h) == 14
        return per, out
    finally:
        L.lpips_destroy(h)


@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("pair", ["hole", "unrelated"])
def test_whole_forward_matches_oracle(emul, sd, normalize, pair):
    a = O.make_images(2, 97, 131, seed=5)
    b = O.composed(a, seed=6) if pair == "hole" else O.make_images(2, 97, 131, seed=7)
    if not normalize:
        a, b = 2 * a - 1, 2 * b - 1
    want_per, want = O.distance(sd, a, b, normalize)
    per, out = _emul_lpips(emul, sd, a, b, normalize)
    err_per = float(((per.double() - want_per).abs() / want_per).max())
    err = float(((out.double() - want).abs() / want).max())
    print("emulated LPIPS %s normalize=%s: per-layer rel err %.3e, total %.3e" % (pair, normalize, err_per, err))
    assert (want_per > 0).all()
    assert err_per < 1e-5 and err < 1e-5
    # the same pairs swapped: the same arithmetic with the roles exchanged
    per_ba, out_ba = _emul_lpips(emul, sd, b, a, normalize)
    assert torch.equal(out_ba, out) and torch.equal(per_ba, per)


def test_identical_images_give_zero(emul, sd):
    a = O.make_images(2, 40, 33, seed=9)
    per, out = _emul_lpips(emul, sd, a, a.clone(), True)
    assert (out == 0).all() and (per == 0).all()


# ---- the weight files -------------------------------------------------------------------------------------------------
@pytest.fixture
def offline(tmp_path, monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("network access attempted")

    hub = tmp_path / "hub"
    hub.mkdir()
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(hub))
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(urllib.request, "urlopen", refuse)
    monkeypatch.setattr(urllib.request, "urlretrieve", refuse)
    lin_path = tmp_path / "lpips_pkg" / "lpips" / "weights" / "v0.1" / "alex.pth"
    monkeypatch.setattr(lpips, "default_lin_path", lambda: str(lin_path))
    return hub, lin_path


def _write_files(sd, hub, lin_path):
    alex = {}
    for ours, tv in O.LPIPS_TO_TORCHVISION.items():
        for leaf in ("weight", "bias"):
            alex[tv + "." + leaf] = sd[ours + "." + leaf]
    alex["classifier.1.weight"] = torch.zeros(8, 9216)   # torchvision's classifier: ignored
    (hub / "checkpoints").mkdir(parents=True, exist_ok=True)
    torch.save(alex, str(hub / "checkpoints" / lpips.ALEXNET_FILE))
    lin_path.parent.mkdir(parents=True, exist_ok=True)
    torch.save({k: v for k, v in sd.items() if k.startswith("lin")}, str(lin_path))


def test_missing_files_are_named_and_never_downloaded(offline):
    hub, lin_path = offline
    with pytest.raises(FileNotFoundError) as e:
        lpips.LPIPS(net="alex")
    assert lpips.ALEXNET_FILE in str(e.value) and os.path.join(str(hub), "checkpoints") in str(e.value)
    assert str(lin_path) in str(e.value)


def test_default_files_give_the_weights_spec(offline, sd, monkeypatch):
    hub, lin_path = offline
    _write_files(sd, hub, lin_path)
    m = lpips.LPIPS(net="alex")
    assert [(k, tuple(v.shape)) for k, v in m._state.items()] == lpips.weight_spec()
    for k, v in sd.items():
        assert torch.equal(m._state[k], v), k
    # model_path takes the place of the lpips package's file
    other = lin_path.parent / "mine.pth"
    os.replace(lin_path, other)
    with pytest.raises(FileNotFoundError, match="alex.pth"):
        lpips.LPIPS()
    assert torch.equal(lpips.LPIPS(model_path=str(other))._state["lin4.model.1.weight"], sd["lin4.model.1.weight"])


def test_lpips_package_weights_are_found_by_spec(tmp_path, monkeypatch):
    pkg = tmp_path / "site" / "lpips"
    pkg.mkdir(parents=True)
    (pkg / "__init__.py").write_text("")
    monkeypatch.syspath_prepend(str(tmp_path / "site"))
    monkeypatch.delitem(sys.modules, "lpips", raising=False)
    assert lpips.default_lin_path() == os.path.join(str(pkg), "weights", "v0.1", "alex.pth")


def test_lins_aliases(sd):
    with_alias = dict(sd)
    for k in range(5):
        with_alias["lins.%d.model.1.weight" % k] = sd["lin%d.model.1.weight" % k].clone()
    m = lpips.LPIPS(weights=with_alias)
    assert sorted(m._state) == sorted(sd)
    bad = dict(with_alias)
    bad["lins.3.model.1.weight"] = bad["lins.3.model.1.weight"] * 2
    with pytest.raises(ValueError, match="lins.3.model.1.weight"):
        lpips.LPIPS(weights=bad)


def test_constructor_contract(sd, tmp_path):
    for kw, arg in ((dict(net="vgg"), "net"), (dict(net="squeeze"), "net"), (dict(version="0.0"), "version"),
                    (dict(lpips=False), "lpips"), (dict(spatial=True), "spatial"), (dict(pnet_rand=True), "pnet_rand"),
                    (dict(pnet_tune=True), "pnet_tune")):
        with pytest.raises(NotImplementedError, match=arg):
            lpips.LPIPS(weights=sd, **kw)
    missing = {k: v for k, v in sd.items() if k != "lin1.model.1.weight"}
    with pytest.raises(_abi.MiganError, match="lin1.model.1.weight"):
        lpips.LPIPS(weights=missing)
    path = tmp_path / "sd.pth"
    torch.save(sd, str(path))
    m = lpips.LPIPS(weights=str(path), use_dropout=False, eval_mode=True, verbose=False)
    assert m.to("cpu") is m   # a module without parameters: .to() as the script calls it
    with pytest.raises(RuntimeError, match="no CPU path"):
        m(torch.rand(1, 3, 64, 64), torch.rand(1, 3, 64, 64))


def test_dropin_rebinds_lpips(tmp_path, monkeypatch):
    """python -m migan_b200.dropin scripts.evaluate_fid_lpips ...: the script's `lpips.LPIPS(net="alex")` (a module
    attribute looked up at call time) builds this package's LPIPS.  The reference and lpips are stood in for by stubs."""
    pkg = tmp_path / "lib" / "model_zoo"
    pkg.mkdir(parents=True)
    (tmp_path / "lib" / "__init__.py").write_text("")
    (pkg / "__init__.py").write_text("")
    (pkg / "migan_inference.py").write_text("class Generator:\n    pass\n")
    (pkg / "comodgan.py").write_text("".join("class %s:\n    pass\n" % c for c in ("Generator", "Mapping", "Encoder", "Synthesis")))
    for name in [m for m in sys.modules if m == "lib" or m.startswith("lib.")]:
        monkeypatch.delitem(sys.modules, name)
    monkeypatch.syspath_prepend(str(tmp_path))
    stub = types.ModuleType("lpips")

    class StubLPIPS:
        pass

    stub.LPIPS = StubLPIPS
    monkeypatch.setitem(sys.modules, "lpips", stub)
    from migan_b200 import dropin
    dropin.install()
    assert stub.LPIPS is migan_b200.lpips.LPIPS and stub.ReferenceLPIPS is StubLPIPS
    import lpips as script_lpips   # what evaluate_fid_lpips.py's `import lpips` binds
    assert script_lpips.LPIPS is migan_b200.lpips.LPIPS
