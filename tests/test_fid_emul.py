"""FID InceptionV3 without a GPU: the oracle against torchvision, the Frechet distance's closed form, and the library's
host runtime in the emulation build (weight registry, launch plan, the whole forward against the float64 oracle)."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

import build_emul  # noqa: E402
import migan_b200  # noqa: E402
from migan_b200 import _abi, fid  # noqa: E402
from oracle import fid_oracle as O  # noqa: E402
from torchvision.models import inception as tvi  # noqa: E402


@pytest.fixture(scope="module")
def emul():
    path = build_emul._compile("inception_emul", [os.path.join(build_emul.CSRC, s) for s in ("inception_abi.cu", "abi_error.cu")])
    return fid.lib(ctypes.CDLL(path))


@pytest.fixture(scope="module")
def sd():
    return O.seeded_state_dict(0)


def _spec_of(module):
    return [(k, tuple(v.shape)) for k, v in module.state_dict().items() if not k.endswith("num_batches_tracked")]


def test_oracle_keys_match_torchvision():
    stock = tvi.inception_v3(weights=None, aux_logits=False, init_weights=False, num_classes=1008)
    want = _spec_of(stock)
    assert len(want) == 472
    assert _spec_of(O.fid_inception()) == want
    assert sum(k.endswith("conv.weight") for k, _ in want) == 94


def test_library_spec_matches_torchvision(emul):
    stock = tvi.inception_v3(weights=None, aux_logits=False, init_weights=False, num_classes=1008)
    assert fid.weight_spec(emul) == _spec_of(stock)


@pytest.mark.parametrize("block", ["A", "C", "E_avg", "E_max"])
def test_pool_variants_differ_only_at_borders(block):
    torch.manual_seed(0)
    if block == "A":
        stock, ours, cin = tvi.InceptionA(64, pool_features=32), O.FIDInceptionA(64, pool_features=32), 64
    elif block == "C":
        stock, ours, cin = tvi.InceptionC(64, channels_7x7=32), O.FIDInceptionC(64, channels_7x7=32), 64
    else:
        stock, ours, cin = tvi.InceptionE(64), O.FIDInceptionE(64, block[2:]), 64
    ours.load_state_dict(stock.state_dict())
    stock, ours = stock.double().eval(), ours.double().eval()
    x = torch.randn(2, cin, 9, 11, dtype=torch.float64) + 0.5
    with torch.no_grad():
        a, b = stock(x), ours(x)
    pool_c = 192 if block != "A" else 32
    # every channel but the branch_pool ones agrees everywhere; those agree inside and differ on the border
    torch.testing.assert_close(a[:, :-pool_c], b[:, :-pool_c], rtol=0, atol=0)
    if block == "E_max":   # Mixed_7c max-pools: unlike the stock average everywhere, equal to the max-pooled branch
        assert (a[:, -pool_c:, 1:-1, 1:-1] - b[:, -pool_c:, 1:-1, 1:-1]).abs().max() > 1e-3
        with torch.no_grad():
            torch.testing.assert_close(b[:, -pool_c:], ours.branch_pool(F.max_pool2d(x, 3, 1, 1)), rtol=0, atol=0)
        return
    torch.testing.assert_close(a[:, -pool_c:, 1:-1, 1:-1], b[:, -pool_c:, 1:-1, 1:-1], rtol=1e-12, atol=1e-12)
    border = torch.ones(9, 11, dtype=torch.bool)
    border[1:-1, 1:-1] = False
    assert (a[:, -pool_c:][..., border] - b[:, -pool_c:][..., border]).abs().max() > 1e-6


def test_frechet_distance_closed_form_on_diagonal_covariances():
    rng = np.random.default_rng(0)
    d = 64
    mu1, mu2 = rng.normal(size=d), rng.normal(size=d)
    s1, s2 = rng.uniform(0.1, 2.0, d), rng.uniform(0.1, 2.0, d)
    want = np.sum((mu1 - mu2) ** 2) + np.sum(s1) + np.sum(s2) - 2 * np.sum(np.sqrt(s1 * s2))
    got = fid.calculate_frechet_distance(mu1, np.diag(s1), mu2, np.diag(s2))
    assert got == pytest.approx(want, rel=1e-10)
    assert O.frechet_distance(mu1, np.diag(s1), mu2, np.diag(s2)) == pytest.approx(want, rel=1e-10)
    # singular product: the eps offset path
    s1[:3] = 0.0
    want = np.sum((mu1 - mu2) ** 2) + np.sum(s1) + np.sum(s2) - 2 * np.sum(np.sqrt(s1 * s2))
    assert fid.calculate_frechet_distance(mu1, np.diag(s1), mu2, np.diag(s2)) == pytest.approx(want, rel=1e-4)


def _ctx(lib, device=0):
    h = ctypes.c_void_p()
    _abi.check(lib.inception_create(device, ctypes.byref(h)), lib)
    return h


def _set(lib, h, key, t):
    t = t.detach().float().contiguous()
    return lib.inception_set_weight(h, key.encode(), t.data_ptr(), t.numel())


def _last_error(lib):
    return lib.migan_last_error().decode()


def test_registry_refuses_bad_keys_by_name(emul, sd):
    emul.migan_last_error.restype = ctypes.c_char_p
    h = _ctx(emul)
    try:
        assert _set(emul, h, "Mixed_5b.branch1x1.bn.num_batches_tracked", torch.zeros(1)) == 0
        assert _set(emul, h, "Mixed_5b.branch9x9.conv.weight", torch.zeros(4)) == _abi.ERR_INVALID
        assert "Mixed_5b.branch9x9.conv.weight" in _last_error(emul)
        assert _set(emul, h, "Conv2d_1a_3x3.conv.weight", torch.zeros(32, 3, 3, 2)) == _abi.ERR_INVALID
        assert "Conv2d_1a_3x3.conv.weight" in _last_error(emul)
        for k, v in sd.items():
            if k != "Mixed_6c.branch7x7_2.bn.running_var":
                assert _set(emul, h, k, v) == 0, _last_error(emul)
        assert emul.inception_finalize_weights(h) == _abi.ERR_INVALID
        assert "Mixed_6c.branch7x7_2.bn.running_var" in _last_error(emul)
    finally:
        emul.inception_destroy(h)


def _hook_shapes(sd):
    """Output shape of every BasicConv2d of the oracle at 299 x 299, by torchvision module name."""
    m = O.model(sd)
    shapes = {}
    hooks = [mod.register_forward_hook(lambda mm, i, o, name=name: shapes.__setitem__(name, tuple(o.shape[1:])))
             for name, mod in m.named_modules() if isinstance(mod, tvi.BasicConv2d)]
    with torch.no_grad():
        O.blocks(m, torch.zeros(1, 3, 299, 299, dtype=torch.float64))
    for h in hooks:
        h.remove()
    return shapes


def test_launch_plan_shapes_offsets(emul, sd):
    plan = fid.launch_plan(2, 97, 131, emul)
    assert plan[0] == "resize in=97x131x3 out=299x299x4"
    assert plan[-1] == "avgpool in=8x8x2048 out=2048"
    convs = [line for line in plan if line.startswith("conv ")]
    pools = [line for line in plan if line.startswith("pool ")]
    assert len(convs) == 94 and len(pools) == 13 and len(plan) == 109
    shapes = _hook_shapes(sd)
    slices = {}
    for line in convs:
        name = line.split()[1]
        kv = dict(tok.split("=") for tok in line.split()[2:])
        oh, ow, co = map(int, kv["out"].split("x"))
        assert (co, oh, ow) == shapes[name], line
        slices.setdefault((name.split(".")[0], int(kv["ct"])), []).append((int(kv["c0"]), co))
    for line in pools:
        kind, name = line.split()[1:3]
        kv = dict(tok.split("=") for tok in line.split()[3:])
        if kind == "max_s2" and name.endswith("branch_pool"):
            slices.setdefault((name.split(".")[0], int(kv["ct"])), []).append((int(kv["c0"]), int(kv["in"].split("x")[2])))
        if name == "Mixed_7c.branch_pool":
            assert kind == "max_s1"
        elif name.endswith("branch_pool") and not name.startswith(("Mixed_6a", "Mixed_7a")):
            assert kind == "avg_s1"
    # each block's slices tile its concatenated output exactly, in torchvision's cat order
    concat = {"Mixed_5b": 256, "Mixed_5c": 288, "Mixed_5d": 288, "Mixed_6a": 768, "Mixed_6b": 768, "Mixed_6c": 768,
              "Mixed_6d": 768, "Mixed_6e": 768, "Mixed_7a": 1280, "Mixed_7b": 2048, "Mixed_7c": 2048}
    for block, ct in concat.items():
        s = sorted(slices[(block, ct)])
        assert s[0][0] == 0 and sum(c for _, c in s) == ct
        assert all(a + b == c for (a, b), (c, _) in zip(s, s[1:])), (block, s)


def _emul_features(lib, sd, x):
    h = _ctx(lib)
    try:
        for k, v in sd.items():
            _abi.check(_set(lib, h, k, v), lib)
        _abi.check(lib.inception_finalize_weights(h), lib)
        n, _, H, W = x.shape
        nbytes = lib.inception_workspace_bytes(h, n, H, W)
        ws = (ctypes.c_uint8 * (nbytes + 256))()
        base = (ctypes.addressof(ws) + 255) // 256 * 256
        xc = x.float().contiguous()
        out = torch.empty((n, 2048), dtype=torch.float32)
        _abi.check(lib.inception_features(h, xc.data_ptr(), n, H, W, out.data_ptr(), base, nbytes, None), lib)
        assert lib.inception_last_launch_count(h) == 109
        return out
    finally:
        lib.inception_destroy(h)


def test_whole_forward_matches_oracle(emul, sd):
    x = O.make_images(1, 97, 131, seed=5)
    want = O.features(sd, x)
    got = _emul_features(emul, sd, x).double()
    scale = max(float(want.abs().max()), 1.0)
    err = float((got - want).abs().max()) / scale
    # the same network in plain fp32 (torch CPU): the rounding this seeded network amplifies over its depth
    m = O.fid_inception()
    m.load_state_dict(sd)
    with torch.no_grad():
        f32 = O.blocks(m.float().eval(), O.input_stage(x)).flatten(1).double()
    err32 = float((f32 - want).abs().max()) / scale
    print("emulated forward: max-abs err %.3e, fp32 torch %.3e (over %.3f)" % (err, err32, scale))
    assert err < 4e-4 and err < 3 * err32
    # the BatchNorm fold matters: without it (running_var = 1, running_mean = 0) the features are far off
    assert any(float((v - 1).abs().max()) > 0.1 for k, v in sd.items() if k.endswith("running_var"))


def test_emulated_resize_and_pools(emul):
    torch.manual_seed(1)
    x = torch.rand(2, 3, 13, 7)
    y = torch.empty(2, 299, 299, 4)
    _abi.check(emul.inception_resize(x.data_ptr(), 2, 13, 7, y.data_ptr(), None), emul)
    want = 2 * F.interpolate(x.double(), size=(299, 299), mode="bilinear", align_corners=False) - 1
    torch.testing.assert_close(y[..., :3].permute(0, 3, 1, 2).double(), want, rtol=0, atol=2e-6)
    assert (y[..., 3] == 0).all()
    a = torch.randn(2, 6, 5, 8)
    nchw = a.permute(0, 3, 1, 2).double()
    for kind, ref, (oh, ow) in ((0, F.max_pool2d(nchw, 3, 2), (2, 2)),
                                (1, F.avg_pool2d(nchw, 3, 1, 1, count_include_pad=False), (6, 5)),
                                (2, F.max_pool2d(nchw, 3, 1, 1), (6, 5))):
        out = torch.full((2, oh, ow, 16), 7.0)
        _abi.check(emul.inception_pool(kind, a.data_ptr(), 2, 6, 5, 8, out.data_ptr(), 16, 4, None), emul)
        torch.testing.assert_close(out[..., 4:12].permute(0, 3, 1, 2).double(), ref, rtol=1e-6, atol=1e-6)
        assert (out[..., :4] == 7).all() and (out[..., 12:] == 7).all()


def test_emulated_statistics_match_numpy(emul):
    rng = np.random.default_rng(3)
    feats = (rng.normal(size=(300, 48)) * 2 + 1000).astype(np.float32)
    shift, s1, s2 = np.zeros(48), np.zeros(48), np.zeros((48, 48))
    for i, chunk in enumerate(np.array_split(feats, 7)):
        c = np.ascontiguousarray(chunk)
        _abi.check(emul.fid_stats_update(c.ctypes.data, c.shape[0], 48, shift.ctypes.data, s1.ctypes.data, s2.ctypes.data,
                                         int(i == 0), None), emul)
    n = feats.shape[0]
    mu, cov = O.statistics(feats)
    np.testing.assert_allclose(shift + s1 / n, mu, rtol=1e-13)
    np.testing.assert_allclose((s2 - np.outer(s1, s1) / n) / (n - 1), cov, rtol=1e-11, atol=1e-12 * np.abs(cov).max())


def test_inception_constructor_contract(tmp_path, monkeypatch):
    with pytest.raises(NotImplementedError, match="output_blocks"):
        fid.InceptionV3([0, 3], weights={})
    with pytest.raises(NotImplementedError, match="use_fid_inception"):
        fid.InceptionV3(use_fid_inception=False, weights={})
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    with pytest.raises(FileNotFoundError, match=re.escape(fid.WEIGHTS_FILE)):
        fid.InceptionV3()
