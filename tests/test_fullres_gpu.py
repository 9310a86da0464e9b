"""The full-resolution request path on the H100 (mi-gan_b200/csrc/fullres.cu, migan_b200.FullResPipeline) and the
library's per-shape plan cache:

* every case of tests/test_fullres_emul.py at R = 256 and 512 (1080 x 1920 included) equals `forward_fc_u8` on the
  host-padded photo and known-mask, cropped, byte for byte; at a valid size, `forward_fc_u8` on the photo itself;
* at R = 64 / 128 against the CPU oracle end to end, with test_u8_gpu.py's uint8 bound;
* a 40-request mixed batch (two passes, photos below and above R) equals the requests one by one for numpy, CPU-tensor
  and CUDA-tensor inputs, `wait=False` on pinned tensors equals `wait=True`, and a pass launches 2 + its chunks' kernels;
* plans cached across shapes, weights and workspaces give the bytes of fresh ones, and the refusals come before any work."""
import numpy as np
import pytest
import torch

import migan_b200
from migan_b200 import synthetic
from migan_b200.fullres import FullResPipeline, plan_passes
from oracle import fullconv_oracle as FC
from oracle import fullres_oracle as F
from oracle import migan_oracle as O

from test_fullres_emul import CASES, _request

pytestmark = pytest.mark.gpu
_PIPES = {}


def _pipe(R, device, seed=5):
    if (R, seed) not in _PIPES:
        _PIPES[(R, seed)] = FullResPipeline(synthetic.export_style_state_dict(R, seed=seed), R, device=device)
    return _PIPES[(R, seed)]


def _padded_reference(model, img, mask, inv, R, device):
    """forward_fc_u8 on the host-padded photo and known-mask, cropped to the photo."""
    H, W = img.shape[:2]
    pi, pm = F.pad(img, F.known_mask(mask, inv), *F.extent(H, W, R))
    out = model.forward_fc_u8(torch.from_numpy(pi[None]).to(device), torch.from_numpy(pm[None]).to(device))
    return out[0, :H, :W].cpu().numpy()


@pytest.mark.parametrize("case", [i for i, c in enumerate(CASES) if c[0] in (256, 512)])
def test_equals_forward_fc_u8_on_padded_photo(cuda_device, case):
    R, H, W, C, inv = CASES[case]
    pipe = _pipe(R, cuda_device)
    img, mask = _request(np.random.default_rng(100 + case), H, W, C)
    got = pipe(img, mask, invert=inv)
    assert isinstance(got, np.ndarray) and got.shape == (H, W, 3) and got.dtype == np.uint8
    assert pipe.last_extents == [F.extent(H, W, R)]
    assert np.array_equal(got, _padded_reference(pipe.model, img, mask, inv, R, cuda_device)), CASES[case]


@pytest.mark.parametrize("R,H,W", [(256, 256, 256), (256, 320, 448), (512, 640, 896), (512, 1152, 1920)])
def test_valid_size_equals_forward_fc_u8(cuda_device, R, H, W):
    pipe = _pipe(R, cuda_device)
    img, mask = _request(np.random.default_rng(H + W), H, W, 1)
    got = pipe(torch.from_numpy(img).to(cuda_device), torch.from_numpy(mask).to(cuda_device))
    assert got.is_cuda and pipe.last_extents == [(H, W)]
    want = pipe.model.forward_fc_u8(torch.from_numpy(img[None]).to(cuda_device), torch.from_numpy(mask[None]).to(cuda_device))
    assert torch.equal(got, want[0])


@pytest.mark.parametrize("R,H,W,C", [(64, 50, 90, 1), (64, 64, 64, 4), (128, 100, 140, 3), (128, 200, 33, 2)])
def test_against_cpu_oracle(cuda_device, R, H, W, C):
    sd = O.make_state_dict(R, seed=1)
    pipe = FullResPipeline(sd, R, device=cuda_device)
    rng = np.random.default_rng(R + H)
    img, mask = _request(rng, H, W, C)
    got = pipe(img, mask, invert=False)
    y = FC.generator_forward_fc(sd, F.preprocess(img, mask, False, R), R)
    want = F.postprocess(y, img, mask, False)
    diff = np.abs(got.astype(int) - want.astype(int))
    assert int(diff.max()) <= 1 and float((diff > 0).mean()) < 1e-3
    known = F.known_mask(mask, False) == 255
    assert np.array_equal(got[known], img[known])


def _mixed(rng, n, R):
    sizes = [(100, 150), (256, 256), (300, 700), (90, 400), (600, 260), (256, 320), (57, 31)]
    out = []
    for k in range(n):
        H, W = sizes[k % len(sizes)]
        out.append(_request(rng, H, W, int(rng.integers(1, 5))) + (bool(k % 3 == 1),))
    return out


def test_mixed_batch_equals_single_requests(cuda_device):
    R = 256
    pipe = _pipe(R, cuda_device)
    reqs = _mixed(np.random.default_rng(40), 40, R)
    exts = [F.extent(i.shape[0], i.shape[1], R) for i, _, _ in reqs]
    assert len(set(exts)) >= 3 and min(i.shape[0] for i, _, _ in reqs) < R < max(i.shape[1] for i, _, _ in reqs)
    alone = [pipe(i, m, invert=v) for i, m, v in reqs]
    invs = [v for _, _, v in reqs]
    got_np = pipe.forward_batch([i for i, _, _ in reqs], [m for _, m, _ in reqs], invert=invs)
    assert pipe.last_extents == exts
    got_cpu = pipe.forward_batch([torch.from_numpy(i) for i, _, _ in reqs], [torch.from_numpy(m) for _, m, _ in reqs], invert=invs)
    got_cuda = pipe.forward_batch([torch.from_numpy(i).to(cuda_device) for i, _, _ in reqs],
                                  [torch.from_numpy(m).to(cuda_device) for _, m, _ in reqs], invert=invs)
    pinned = [torch.from_numpy(i).pin_memory() for i, _, _ in reqs]
    got_async = pipe.forward_batch(pinned[:25], [torch.from_numpy(m) for _, m, _ in reqs[:25]], invert=invs[:25], wait=False)
    got_async += pipe.forward_batch(pinned[25:], [torch.from_numpy(m) for _, m, _ in reqs[25:]], invert=invs[25:], wait=False)
    pipe.wait()
    assert pipe.last_extents == exts
    for k in range(40):
        assert isinstance(got_np[k], np.ndarray) and np.array_equal(got_np[k], alone[k]), k
        assert not got_cpu[k].is_cuda and np.array_equal(got_cpu[k].numpy(), alone[k]), k
        assert got_cuda[k].is_cuda and np.array_equal(got_cuda[k].cpu().numpy(), alone[k]), k
        assert np.array_equal(got_async[k].numpy(), alone[k]), k


def test_launches_per_pass(cuda_device):
    R = 256
    pipe = _pipe(R, cuda_device)
    reqs = _mixed(np.random.default_rng(41), 40, R)
    pipe.forward_batch([i for i, _, _ in reqs], [m for _, m, _ in reqs])
    last = plan_passes(pipe.last_extents, {e: 1 << 20 for e in pipe.last_extents})[-1]
    want = 2
    for c in last:
        pipe.model.forward_fc(torch.zeros(len(c.requests), 4, c.Hp, c.Wp, device=cuda_device))
        want += pipe.model.last_launch_count()
    assert len(last) >= 3 and pipe.last_launches == want


def test_plan_cache_alternating_shapes(cuda_device):
    """forward_fc over three shapes, twice round, equals each call alone; forward (graph and plain) and forward_u8 in
    between are unchanged."""
    g = migan_b200.Generator(256)
    g.load_state_dict(O.make_state_dict(256, seed=2))
    g = g.to(cuda_device).eval()
    xs = [FC.make_input_hw(256, n, H, W, seed=H + W).to(cuda_device) for n, H, W in [(2, 320, 448), (1, 256, 256), (3, 512, 320)]]
    xg = O.make_input(256, 2, seed=1).to(cuda_device)
    xp = O.make_input(256, 6, seed=2).to(cuda_device)
    rng = np.random.RandomState(0)
    img = torch.from_numpy(rng.randint(0, 256, size=(2, 256, 256, 3)).astype(np.uint8))
    mask = torch.from_numpy((rng.rand(2, 256, 256) > 0.3).astype(np.uint8) * 255)
    alone = [g.forward_fc(x) for x in xs] + [g(xg), g(xp), g.forward_u8(img, mask).clone()]
    for _ in range(2):
        seq = []
        for x in xs:
            seq.append(g.forward_fc(x))
        seq += [g(xg), g(xp), g.forward_u8(img, mask).clone()]
        for i, (a, b) in enumerate(zip(alone, seq)):
            assert torch.equal(a, b), i


def test_plan_cache_new_weights_and_new_workspace(cuda_device):
    R = 256
    pipe = FullResPipeline(synthetic.export_style_state_dict(R, seed=7), R, device=cuda_device)
    reqs = _mixed(np.random.default_rng(42), 6, R)
    imgs, masks = [i for i, _, _ in reqs], [m for _, m, _ in reqs]
    first = pipe.forward_batch(imgs, masks)
    xg = O.make_input(R, 2, seed=3).to(cuda_device)
    y_graph = pipe.model(xg)
    # a larger request grows the workspace: the same shapes then run on new memory
    pipe.forward_batch([np.zeros((1500, 1500, 3), np.uint8)], [np.full((1500, 1500), 255, np.uint8)])
    again = pipe.forward_batch(imgs, masks)
    assert all(np.array_equal(a, b) for a, b in zip(first, again))
    assert torch.equal(pipe.model(xg), y_graph)
    # other weights: every cached plan goes, the results are those of a fresh pipeline
    sd2 = synthetic.export_style_state_dict(R, seed=8)
    pipe.model.load_state_dict(sd2)
    got = pipe.forward_batch(imgs, masks)
    fresh = FullResPipeline(sd2, R, device=cuda_device).forward_batch(imgs, masks)
    assert all(np.array_equal(a, b) for a, b in zip(got, fresh))
    assert not all(np.array_equal(a, b) for a, b in zip(got, first))


def test_refusals_before_any_work(cuda_device):
    pipe = _pipe(512, cuda_device)
    ok_img, ok_mask = np.zeros((40, 50, 3), np.uint8), np.full((40, 50), 255, np.uint8)
    assert np.array_equal(pipe(ok_img, ok_mask), ok_img)          # all known: the photo itself (weights and workspace set up)
    torch.cuda.synchronize()
    mem0 = torch.cuda.memory_allocated()
    bad = [
        (ValueError, "request 1: mask of 40 x 49", [ok_img, ok_img], [ok_mask, ok_mask[:, :49]]),
        (ValueError, "request 1: .*uint8", [ok_img, ok_img.astype(np.float32)], [ok_mask, ok_mask]),
        (ValueError, "request 0: photo of shape", [ok_img[..., :2]], [ok_mask]),
        (ValueError, "request 0: photo of shape", [ok_img[0]], [ok_mask]),
        (ValueError, "request 0: mask of shape", [ok_img], [np.zeros((40, 50, 5), np.uint8)]),
        (ValueError, "request 1: photo of 4096 x 8191", [ok_img, np.zeros((4096, 8191, 3), np.uint8)],
         [ok_mask, np.zeros((4096, 8191), np.uint8)]),
        (TypeError, "request 0", [[[1, 2, 3]]], [ok_mask]),
        (TypeError, "request 0", [ok_img], [None]),
    ]
    for exc, match, imgs, masks in bad:
        with pytest.raises(exc, match=match):
            pipe.forward_batch(imgs, masks)
    with pytest.raises(RuntimeError, match="pinned"):
        pipe.forward_batch([torch.from_numpy(ok_img)], [ok_mask], wait=False)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == mem0
