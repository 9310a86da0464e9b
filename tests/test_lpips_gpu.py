"""LPIPS on the H100: the input stage and AlexNet's convolution forms on their own, the whole distance against the
float64 oracle, bitwise batch invariance and symmetry, the evaluation step end to end, launch accounting."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import migan_b200  # noqa: E402
from migan_b200 import _abi, fid, lpips  # noqa: E402
from oracle import lpips_oracle as O  # noqa: E402
from oracle import migan_oracle as MO  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# Relative error of each layer term and of the total against the float64 oracle on the seeded weights, over the 12
# cases of test_lpips_matches_oracle (hole and unrelated pairs), measured on an H100: per layer at most 8.4e-6 (31 x 31,
# n = 33), total at most 5.4e-7 (97 x 131, n = 33).  One TF32 pass measures ~1.7e-4 per layer.  Bounds: ~3x.
LAYER_TOL, TOTAL_TOL = 2.5e-5, 1.6e-6
GUARD = 16384   # floats = 64 KB guard bands


@pytest.fixture(scope="module")
def sd():
    return O.seeded_state_dict(0)


@pytest.fixture(scope="module")
def oracle_model(sd):
    return O.model(sd).to(DEV)


@pytest.fixture(scope="module")
def net(sd):
    return lpips.LPIPS(net="alex", weights=sd).to(DEV)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _pairs(n, h, w, seed):
    """n pairs in [0, 1]: a composed copy of the first image (a replaced rectangle), every third pair unrelated."""
    a = O.make_images(n, h, w, seed=seed)
    b = O.composed(a, seed=seed + 1)
    b[2::3] = O.make_images(n, h, w, seed=seed + 2)[2::3]
    return a, b


@pytest.mark.parametrize("normalize", [False, True])
def test_input_stage_against_torch(normalize):
    torch.manual_seed(0)
    n, H, W = 3, 37, 45
    a, b = torch.rand(n, 3, H, W), torch.rand(n, 3, H, W)
    shift, scale = (ctypes.c_float * 3)(*O.SHIFT), (ctypes.c_float * 3)(*O.SCALE)
    y = torch.empty(2 * n, H, W, 4, device=DEV)
    ad, bd = a.to(DEV), b.to(DEV)
    _abi.check(lpips.lib().lpips_input(ad.data_ptr(), bd.data_ptr(), n, H, W, int(normalize), shift, scale, y.data_ptr(),
                                       _stream()))
    x = torch.cat([a, b])
    if normalize:
        x = 2 * x - 1
    want = (x - torch.tensor(O.SHIFT).view(1, 3, 1, 1)) / torch.tensor(O.SCALE).view(1, 3, 1, 1)
    got = y.cpu()
    torch.testing.assert_close(got[..., :3].permute(0, 3, 1, 2), want, rtol=0, atol=0)
    assert (got[..., 3] == 0).all()


# AlexNet features.{0, 3, 6, 8, 10}: (kh, kw, stride, ph, pw, cin, cout); the first at cin = 4 with a zero 4th channel
FORMS = [(11, 11, 4, 2, 2, 4, 64), (5, 5, 1, 2, 2, 64, 192), (3, 3, 1, 1, 1, 192, 384), (3, 3, 1, 1, 1, 384, 256),
         (3, 3, 1, 1, 1, 256, 256)]


@pytest.mark.parametrize("form", FORMS, ids=["%dx%d_s%d_p%d,%d_cin%d" % f[:6] for f in FORMS])
def test_alexnet_conv_forms_write_their_slice(form):
    kh, kw, s, ph, pw, cin, cout = form
    torch.manual_seed(kh * 10 + cin)
    n, H, W = 3, 47, 53
    x = torch.randn(n, H, W, cin)
    if cin == 4:
        x[..., 3] = 0
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
    assert err / scale < 2e-5   # the bound of the FID network's forms; one TF32 pass would be ~1e-3


@pytest.mark.parametrize("size", [(256, 256), (512, 512), (97, 131), (31, 31)])
@pytest.mark.parametrize("n", [1, 3, 33])
def test_lpips_matches_oracle(net, sd, oracle_model, size, n):
    h, w = size
    a, b = _pairs(n, h, w, seed=100 + n)
    val, per = net(a.to(DEV), b.to(DEV), retPerLayer=True, normalize=True)
    assert val.shape == (n, 1, 1, 1) and val.dtype == torch.float32 and val.is_cuda
    assert len(per) == 5 and all(p.shape == (n, 1, 1, 1) for p in per)
    want_per, want = O.distance(sd, a.to(DEV), b.to(DEV), normalize=True, m=oracle_model)
    got_per = torch.stack([p.view(n) for p in per]).double()
    assert (want_per > 0).all()
    err_per = float(((got_per - want_per).abs() / want_per).max())
    err = float(((val.view(n).double() - want).abs() / want).max())
    print("lpips %dx%d n=%d: per-layer rel err %.3e, total %.3e" % (h, w, n, err_per, err))
    assert err_per < LAYER_TOL and err < TOTAL_TOL
    assert torch.equal(net(a.to(DEV), b.to(DEV), normalize=True), val)   # retPerLayer does not change the value


def test_batch_invariance_and_symmetry(net):
    a, b = _pairs(5, 160, 200, seed=7)
    a, b = a.to(DEV), b.to(DEV)
    full = net(a, b).view(5)
    for i in range(5):
        assert torch.equal(net(a[i:i + 1], b[i:i + 1]).view(1)[0], full[i])
    pair = net(torch.cat([a[3:4], a[1:2]]), torch.cat([b[3:4], b[1:2]])).view(2)
    assert torch.equal(pair[0], full[3]) and torch.equal(pair[1], full[1])
    val, per = net(a, b, retPerLayer=True)
    val_ba, per_ba = net(b, a, retPerLayer=True)
    assert torch.equal(val_ba, val) and all(torch.equal(p, q) for p, q in zip(per, per_ba))
    same, per_same = net(a, a.clone(), retPerLayer=True)
    assert (same == 0).all() and all((p == 0).all() for p in per_same)
    assert (full > 0).all()


def test_input_checks(net):
    x = torch.rand(2, 3, 31, 31, device=DEV)
    for bad in ((2, 3, 30, 31), (2, 3, 31, 30)):
        with pytest.raises(ValueError, match="31"):
            net(torch.rand(bad, device=DEV), torch.rand(bad, device=DEV))
    with pytest.raises(RuntimeError, match="shape"):
        net(x, x[:1])
    with pytest.raises(RuntimeError, match="no CPU path"):
        net(x.cpu(), x.cpu())


def test_evaluation_step_end_to_end(net, sd, oracle_model):
    """The script's call: compute_lpips(imgs, composed_imgs, normalize=True).detach().cpu().numpy().tolist()."""
    R, n = 256, 8
    gen_sd = MO.make_state_dict(R, seed=3)
    pipe = migan_b200.EvalPipeline(gen_sd, resolution=R, device=DEV, seed=0)
    rng = np.random.default_rng(5)
    imgs = [rng.integers(0, 256, size=(R, R, 3), dtype=np.uint8) for _ in range(n)]
    real, composed = pipe.forward_batch(imgs)
    got = net(real, composed, normalize=True)
    values = got.detach().cpu().numpy().tolist()
    assert len(values) == n and all(len(v) == 1 and len(v[0]) == 1 and len(v[0][0]) == 1 for v in values)
    want_per, want = O.distance(sd, real, composed, normalize=True, m=oracle_model)
    err = ((got.view(n).double() - want).abs() / want.clamp_min(1e-30))
    print("evaluation step: LPIPS %s, rel err %.3e" % (np.round(want.cpu().numpy(), 5).tolist(), float(err.max())))
    assert float(err.max()) < TOTAL_TOL


def test_launch_count_matches_profiler(net):
    a, b = _pairs(2, 128, 128, seed=9)
    a, b = a.to(DEV), b.to(DEV)
    net(a, b)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        # a tracer started after an earlier session in the process can miss its first few kernel records: lead with
        # torch kernels that are not counted
        pad = torch.zeros(1, device=DEV)
        for _ in range(256):
            pad.add_(1)
        torch.cuda.synchronize()
        net(a, b)
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and "memset" not in e.name.lower() and "memcpy" not in e.name.lower()]
    ours = [e for e in kernels if "incep" in e.name or "ck_items_kernel" in e.name or "lpips" in e.name]
    assert net.last_launch_count() == len(net.launch_plan(2, 128, 128)) == 14
    assert len(ours) == net.last_launch_count(), sorted({e.name for e in kernels})
