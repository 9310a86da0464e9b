"""FID InceptionV3 and the feature statistics on the H100: each kernel on its own, the whole forward against the
float64 oracle, batch invariance, the statistics against np.cov, the evaluation step end to end, launch accounting."""
import ctypes
import os
import sys
import urllib.request

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import migan_b200  # noqa: E402
from migan_b200 import _abi, fid  # noqa: E402
from oracle import fid_oracle as O  # noqa: E402
from oracle import migan_oracle as MO  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# Feature error over max(|f|max, 1) against the float64 oracle on the seeded weights, measured on an H100 over the 12
# cases of test_features_match_oracle: max-abs 1.3e-4 to 5.3e-4, mean-abs 1e-5 to 5e-5.  Plain fp32 (torch CPU) on the
# same network measures 1.1e-4 on the 97 x 131 case: the seeded 94-layer network amplifies fp32 rounding.  Bounds: ~3x.
FEATURE_TOL, FEATURE_MEAN_TOL = 1.5e-3, 1.5e-4
GUARD = 16384   # floats = 64 KB guard bands


@pytest.fixture(scope="module")
def sd():
    return O.seeded_state_dict(0)


@pytest.fixture(scope="module")
def oracle_model(sd):
    return O.model(sd)


@pytest.fixture(scope="module")
def net(sd):
    return fid.InceptionV3(weights=sd)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def test_resize_against_torch():
    torch.manual_seed(0)
    for (h, w) in ((256, 256), (97, 131), (1, 1), (512, 300)):
        x = torch.rand(2, 3, h, w)
        y = torch.empty(2, 299, 299, 4, device=DEV)
        _abi.check(fid.lib().inception_resize(x.to(DEV).data_ptr(), 2, h, w, y.data_ptr(), _stream()))
        want = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False) * 2 - 1
        got = y.cpu()
        torch.testing.assert_close(got[..., :3].permute(0, 3, 1, 2), want, rtol=0, atol=2e-6)
        assert (got[..., 3] == 0).all()


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_pools_against_torch(kind):
    torch.manual_seed(kind)
    n, H, W, C, ct, c0 = 3, 17, 10, 48, 96, 16
    x = torch.randn(n, H, W, C)
    nchw = x.permute(0, 3, 1, 2)
    want = (F.max_pool2d(nchw, 3, 2), F.avg_pool2d(nchw, 3, 1, 1, count_include_pad=False), F.max_pool2d(nchw, 3, 1, 1))[kind]
    oh, ow = want.shape[2:]
    y = torch.full((n, oh, ow, ct), 3.25, device=DEV)
    _abi.check(fid.lib().inception_pool(kind, x.to(DEV).data_ptr(), n, H, W, C, y.data_ptr(), ct, c0, _stream()))
    got = y.cpu()
    torch.testing.assert_close(got[..., c0:c0 + C].permute(0, 3, 1, 2), want, rtol=1e-6, atol=1e-6)
    assert (got[..., :c0] == 3.25).all() and (got[..., c0 + C:] == 3.25).all()


# the 9 (kh, kw, stride, pad) forms of the network, each with a cin / cout it has
FORMS = [(1, 1, 1, 0, 0, 192, 64), (3, 3, 1, 0, 0, 32, 32), (3, 3, 1, 1, 1, 64, 96), (3, 3, 2, 0, 0, 288, 384),
         (5, 5, 1, 2, 2, 48, 64), (1, 7, 1, 0, 3, 128, 128), (7, 1, 1, 3, 0, 160, 192), (1, 3, 1, 0, 1, 384, 384),
         (3, 1, 1, 1, 0, 384, 384)]


@pytest.mark.parametrize("form", FORMS, ids=["%dx%d_s%d_p%d,%d" % f[:5] for f in FORMS])
def test_conv_forms_write_their_slice(form):
    kh, kw, s, ph, pw, cin, cout = form
    torch.manual_seed(kh * 10 + kw)
    n, H, W = 3, 19, 23
    x = torch.randn(n, H, W, cin)
    w = torch.randn(cout, cin, kh, kw) * (2.0 / (cin * kh * kw)) ** 0.5
    b = torch.randn(cout) * 0.1
    want = F.relu(F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), stride=s, padding=(ph, pw)))
    oh, ow = want.shape[2:]
    c0, ct = 32, cout + 48
    total = n * oh * ow * ct
    buf = torch.full((GUARD + total + GUARD,), -7.5, device=DEV)
    y = buf[GUARD:GUARD + total]
    L = fid.lib()
    need_c = ctypes.c_size_t()
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)   # held: the workspace below must not reuse their memory
    args = [xd.data_ptr(), n, H, W, cin, wd.data_ptr(), bd.data_ptr(), cout, kh, kw, s, ph, pw, y.data_ptr(), ct, c0]
    _abi.check(L.inception_conv2d(*args, None, 0, ctypes.byref(need_c), _stream()))
    ws = torch.empty(need_c.value, dtype=torch.uint8, device=DEV)
    _abi.check(L.inception_conv2d(*args, ws.data_ptr(), ws.numel(), None, _stream()))
    got = buf.cpu()
    assert (got[:GUARD] == -7.5).all() and (got[GUARD + total:] == -7.5).all()
    out = got[GUARD:GUARD + total].view(n, oh, ow, ct)
    assert (out[..., :c0] == -7.5).all() and (out[..., c0 + cout:] == -7.5).all()
    err = float((out[..., c0:c0 + cout].permute(0, 3, 1, 2).double() - want).abs().max())
    scale = max(float(want.abs().max()), 1.0)
    print("conv %s: max-abs err %.3e over %.3f" % (form, err, scale))
    assert err / scale < 2e-5   # measured <= 6.8e-6 on an H100 (fp32-faithful); one TF32 pass would be ~1e-3


@pytest.mark.parametrize("size", [(256, 256), (512, 512), (299, 299), (97, 131)])
@pytest.mark.parametrize("n", [1, 3, 33])
def test_features_match_oracle(net, oracle_model, size, n):
    h, w = size
    x = O.make_images(n, h, w, seed=100 + n)
    got = net(x.to(DEV))[0]
    assert got.shape == (n, 2048, 1, 1) and got.dtype == torch.float32 and got.is_cuda
    got = got.view(n, 2048).cpu().double()
    want = torch.cat([O.features(oracle_model, x[i:i + 8]) for i in range(0, n, 8)])
    scale = max(float(want.abs().max()), 1.0)
    err = (got - want).abs()
    print("features %dx%d n=%d: max-abs %.3e mean-abs %.3e over %.3f" % (h, w, n, float(err.max()) / scale,
                                                                         float(err.mean()) / scale, scale))
    assert float(err.max()) / scale < FEATURE_TOL and float(err.mean()) / scale < FEATURE_MEAN_TOL


def test_batch_invariance(net):
    x = O.make_images(5, 160, 200, seed=7).to(DEV)
    full = net(x)[0].view(5, 2048)
    for i in range(5):
        alone = net(x[i:i + 1])[0].view(1, 2048)
        assert torch.equal(alone[0], full[i])
    pair = net(torch.cat([x[3:4], x[1:2]]))[0].view(2, 2048)
    assert torch.equal(pair[0], full[3]) and torch.equal(pair[1], full[1])


@pytest.mark.parametrize("offset", [0.0, 1e4])
def test_feature_statistics_match_numpy(offset):
    rng = np.random.default_rng(11)
    base = rng.normal(size=(4096, 64)) @ rng.normal(size=(64, 2048)) * 0.1
    feats = (np.abs(base) + offset).astype(np.float32)
    st = fid.FeatureStatistics(2048, device=DEV)
    for chunk in np.array_split(feats, 13):
        st.add(torch.from_numpy(np.ascontiguousarray(chunk)).to(DEV))
    assert st.count == 4096
    mu, sigma = st.mean_cov()
    mu_ref, sigma_ref = O.statistics(feats)
    assert np.max(np.abs(mu - mu_ref)) <= 1e-12 * np.max(np.abs(mu_ref))
    assert np.max(np.abs(sigma - sigma_ref)) <= 1e-12 * np.max(np.abs(sigma_ref))
    assert np.array_equal(sigma, sigma.T)


def test_evaluation_step_end_to_end(net):
    R, n = 256, 8
    gen_sd = MO.make_state_dict(R, seed=3)
    pipe = migan_b200.EvalPipeline(gen_sd, resolution=R, device=DEV, seed=0)
    rng = np.random.default_rng(5)
    imgs = [rng.integers(0, 256, size=(R, R, 3), dtype=np.uint8) for _ in range(n)]
    real, composed = pipe.forward_batch(imgs)
    fr, fc = net(real)[0].view(n, 2048), net(composed)[0].view(n, 2048)
    s_r, s_c = fid.FeatureStatistics(device=DEV), fid.FeatureStatistics(device=DEV)
    s_r.add(fr)
    s_c.add(fc)
    ref_r, ref_c = O.statistics(fr.cpu().numpy()), O.statistics(fc.cpu().numpy())
    for (mu, sigma), (mu_ref, sigma_ref) in ((s_r.mean_cov(), ref_r), (s_c.mean_cov(), ref_c)):
        np.testing.assert_allclose(mu, mu_ref, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(sigma, sigma_ref, rtol=1e-9, atol=1e-12 * np.abs(sigma_ref).max())
    want = O.frechet_distance(*ref_r, *ref_c)
    assert fid.calculate_frechet_distance(*ref_r, *ref_c) == pytest.approx(want, rel=1e-9)
    # the statistics differ from numpy's in the last bits; sqrtm of these rank-deficient products is ill-conditioned
    assert fid.calculate_frechet_distance(*s_r.mean_cov(), *s_c.mean_cov()) == pytest.approx(want, rel=1e-3)


def test_launch_count_matches_profiler(net):
    x = O.make_images(2, 128, 128, seed=9).to(DEV)
    net(x)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        # a tracer started after an earlier session in the process can miss its first few kernel records: lead with
        # torch kernels that are not counted
        pad = torch.zeros(1, device=DEV)
        for _ in range(256):
            pad.add_(1)
        torch.cuda.synchronize()
        net(x)
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and "memset" not in e.name.lower() and "memcpy" not in e.name.lower()]
    ours = [e for e in kernels if "incep" in e.name or "ck_items_kernel" in e.name]
    assert net.last_launch_count() == 109
    assert len(ours) == net.last_launch_count(), sorted({e.name for e in kernels})


def test_no_download_without_weights(tmp_path, monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("network access attempted")

    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(urllib.request, "urlopen", refuse)
    monkeypatch.setattr(urllib.request, "urlretrieve", refuse)
    with pytest.raises(FileNotFoundError, match="checkpoints"):
        fid.InceptionV3()
