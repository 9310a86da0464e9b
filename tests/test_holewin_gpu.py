"""The hole-window request path on the H100 (mi-gan_b200/csrc/holewin.cu, the window kernels of fullres.cu,
migan_b200.HoleWindowPipeline):

* at R = 256 and 512 the output is the photo with every window replaced by `FullResPipeline` on the host-cropped window,
  byte for byte; the pixels outside every window are the photo's and `last_windows` is the oracle planner's;
* one hole over most of the photo gives the whole-photo window and `FullResPipeline`'s bytes; a photo without a hole comes
  back unchanged after the cells launch alone;
* a 6000 x 8000 photo, too large for one forward at R = 256, is inpainted through its windows; a window too large for one
  forward is refused before any generator work and the next call succeeds;
* a 40-request mixed batch with several windows per request (more than one window pass) equals the single calls for numpy,
  CPU-tensor, CUDA-tensor and pinned `wait=False` inputs; the launches are 1 per 32 requests + 2 per pass + the chunks';
* `wait=False` on pinned inputs returns while the stream is still busy, with the waiting call's bytes after `wait()`."""
import numpy as np
import pytest
import torch

from migan_b200 import synthetic
from migan_b200.fullres import FullResPipeline, plan_passes
from migan_b200.holewin import HoleWindowPipeline
from oracle import fullres_oracle as F
from oracle import holewin_oracle as HW

pytestmark = pytest.mark.gpu
_PIPES = {}


def _pipes(R, device):
    """(HoleWindowPipeline, FullResPipeline) on one generator."""
    if R not in _PIPES:
        hw = HoleWindowPipeline(synthetic.export_style_state_dict(R, seed=5), R, device=device)
        _PIPES[R] = (hw, FullResPipeline(hw.model, R, device=device))
    return _PIPES[R]


def _photo(rng, H, W, C, holes, inv=False):
    """A random photo and a mask of C channels with rectangular holes (y, x, h, w) and a few stray hole pixels."""
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    m = rng.integers(0, 256, (H, W, C), dtype=np.uint8)
    ch = {1: 0, 2: 1, 3: 0, 4: 3}[C]
    m[..., ch] = 255
    for y, x, h, w in holes:
        m[y:y + h, x:x + w, ch] = rng.choice(np.array([0, 1, 254], np.uint8), m[y:y + h, x:x + w, ch].shape)
    if inv:
        m = 255 - m
    return img, np.ascontiguousarray(m[..., 0] if C == 1 else m)


def _expected(full, img, mask, inv, R, margin=1):
    wins = HW.windows(HW.cells(mask, inv, R), img.shape[0], img.shape[1], R, margin)
    return wins, HW.compose(img, mask, wins, lambda k, ci, cm: full(ci, cm, invert=inv))


CASES = [  # (R, H, W, C, invert, holes)
    (256, 1080, 1920, 1, False, [(100, 200, 40, 60), (900, 1700, 30, 30)]),
    (256, 700, 1000, 4, True, [(0, 0, 10, 10), (690, 990, 10, 10), (300, 450, 20, 200)]),
    (256, 333, 901, 2, False, [(150, 10, 20, 870)]),
    (256, 200, 150, 3, False, [(20, 20, 5, 5)]),
    (512, 3024, 4032, 4, False, [(1500, 2000, 300, 400)]),
    (512, 2160, 3840, 1, True, [(100, 100, 50, 80), (2000, 3700, 60, 60)]),
    (512, 1000, 1500, 3, False, [(0, 700, 1000, 20)]),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_equals_fullres_on_each_window(cuda_device, case):
    R, H, W, C, inv, holes = CASES[case]
    pipe, full = _pipes(R, cuda_device)
    img, mask = _photo(np.random.default_rng(case), H, W, C, holes, inv)
    got = pipe(img, mask, invert=inv)
    wins, want = _expected(full, img, mask, inv, R)
    assert isinstance(got, np.ndarray) and got.shape == (H, W, 3) and got.dtype == np.uint8
    assert pipe.last_windows == [wins] and len(wins) >= 1
    assert np.array_equal(got, want), CASES[case]
    inside = np.zeros((H, W), bool)
    for y0, x0, h, w in wins:
        inside[y0:y0 + h, x0:x0 + w] = True
    assert np.array_equal(got[~inside], img[~inside])
    hole = F.known_mask(mask, inv) != 255
    assert not np.array_equal(got[hole], img[hole])          # the generator's pixels did land


@pytest.mark.parametrize("R", [256, 512])
def test_whole_photo_window_equals_fullres(cuda_device, R):
    pipe, full = _pipes(R, cuda_device)
    H, W = 900, 1300
    img, mask = _photo(np.random.default_rng(R), H, W, 1, [(5, 5, H - 10, W - 10)])
    got = pipe(img, mask)
    assert pipe.last_windows == [[(0, 0, H, W)]]
    assert np.array_equal(got, full(img, mask))


def test_hole_free_photo_unchanged_without_generator(cuda_device):
    pipe, _ = _pipes(256, cuda_device)
    img, mask = _photo(np.random.default_rng(1), 777, 1234, 4, [])
    got = pipe(torch.from_numpy(img).to(cuda_device), torch.from_numpy(mask).to(cuda_device))
    assert pipe.last_windows == [[]] and pipe.last_launches == 1
    assert got.is_cuda and np.array_equal(got.cpu().numpy(), img)


def test_photo_too_large_for_one_forward(cuda_device):
    R = 256
    pipe, full = _pipes(R, cuda_device)
    H, W = 6000, 8000
    with pytest.raises(ValueError, match="too large for one forward"):
        full._extent(full.model._engine(cuda_device), 0, H, W)
    img, mask = _photo(np.random.default_rng(2), H, W, 1, [(300, 400, 50, 70), (5500, 7300, 80, 40)])
    got = pipe.forward_batch([torch.from_numpy(img)], [torch.from_numpy(mask)])[0].numpy()
    wins, want = _expected(full, img, mask, False, R)
    assert pipe.last_windows == [wins] and len(wins) == 2
    assert np.array_equal(got, want)
    # a window too large for one forward: refused before any generator work, and the pipeline stays usable
    big = np.zeros((H, W), np.uint8)
    small_img, small_mask = _photo(np.random.default_rng(3), 300, 400, 1, [(10, 10, 20, 20)])
    launches, ws = pipe.last_launches, pipe._ws
    with pytest.raises(ValueError, match=r"request 1: window \(y0, x0, h, w\) = \(0, 0, 6000, 8000\)"):
        pipe.forward_batch([small_img, img], [small_mask, big])
    assert pipe.last_launches == launches and pipe._ws is ws
    again = pipe(small_img, small_mask)
    assert np.array_equal(again, _expected(full, small_img, small_mask, False, R)[1])


def _mixed(rng, n):
    sizes = [(700, 1100), (300, 260), (1024, 768), (90, 400), (600, 1500)]
    out = []
    for k in range(n):
        H, W = sizes[k % len(sizes)]
        holes = [(int(rng.integers(0, H - 8)), int(rng.integers(0, W - 8)), 8, 8) for _ in range(3)]
        C = int(rng.integers(1, 5))
        inv = bool(k % 3 == 1)
        out.append(_photo(rng, H, W, C, holes, inv) + (inv,))
    return out


def test_mixed_batch_equals_single_calls(cuda_device):
    R = 256
    pipe, _ = _pipes(R, cuda_device)
    reqs = _mixed(np.random.default_rng(40), 40)
    invs = [v for _, _, v in reqs]
    alone, wins = [], []
    for i, m, v in reqs:
        alone.append(pipe(i, m, invert=v))
        wins += pipe.last_windows
    assert sum(len(w) for w in wins) > 32 and max(len(w) for w in wins) >= 2
    got_np = pipe.forward_batch([i for i, _, _ in reqs], [m for _, m, _ in reqs], invert=invs)
    assert pipe.last_windows == wins
    got_cpu = pipe.forward_batch([torch.from_numpy(i) for i, _, _ in reqs], [torch.from_numpy(m) for _, m, _ in reqs], invert=invs)
    got_cuda = pipe.forward_batch([torch.from_numpy(i).to(cuda_device) for i, _, _ in reqs],
                                  [torch.from_numpy(m).to(cuda_device) for _, m, _ in reqs], invert=invs)
    pinned = [torch.from_numpy(i).pin_memory() for i, _, _ in reqs]
    pinned_m = [torch.from_numpy(m).pin_memory() for _, m, _ in reqs]
    got_async = pipe.forward_batch(pinned[:25], pinned_m[:25], invert=invs[:25], wait=False)
    got_async += pipe.forward_batch(pinned[25:], pinned_m[25:], invert=invs[25:], wait=False)
    pipe.wait()
    assert pipe.last_windows == wins
    for k in range(40):
        assert isinstance(got_np[k], np.ndarray) and np.array_equal(got_np[k], alone[k]), k
        assert not got_cpu[k].is_cuda and np.array_equal(got_cpu[k].numpy(), alone[k]), k
        assert got_cuda[k].is_cuda and np.array_equal(got_cuda[k].cpu().numpy(), alone[k]), k
        assert np.array_equal(got_async[k].numpy(), alone[k]), k


def test_launch_count(cuda_device):
    R = 256
    pipe, _ = _pipes(R, cuda_device)
    reqs = _mixed(np.random.default_rng(41), 40)
    pipe.forward_batch([i for i, _, _ in reqs], [m for _, m, _ in reqs], invert=[v for _, _, v in reqs])
    exts = [F.extent(h, w, R) for ws in pipe.last_windows for _, _, h, w in ws]
    passes = plan_passes(exts, {e: 1 << 20 for e in exts})
    assert len(passes) >= 2
    want = 2                                              # one cells launch per 32 requests
    for p in passes:
        want += 2
        for c in p:
            pipe.model.forward_fc(torch.zeros(len(c.requests), 4, c.Hp, c.Wp, device=cuda_device))
            want += pipe.model.last_launch_count()
    assert pipe.last_launches == want


def test_wait_false_runs_ahead_of_a_busy_stream(cuda_device):
    R = 256
    pipe, _ = _pipes(R, cuda_device)
    reqs = _mixed(np.random.default_rng(6), 6)
    invs = [v for _, _, v in reqs]
    want = pipe.forward_batch([i for i, _, _ in reqs], [m for _, m, _ in reqs], invert=invs)
    want_wins = pipe.last_windows
    imgs = [torch.from_numpy(i).pin_memory() for i, _, _ in reqs]
    masks = [torch.from_numpy(m).pin_memory() for _, m, _ in reqs]
    stream = torch.cuda.current_stream(cuda_device)
    torch.cuda._sleep(1_000_000_000)
    got = pipe.forward_batch(imgs, masks, invert=invs, wait=False)
    busy = not stream.query()
    pipe.wait()
    assert busy, "forward_batch(wait=False) waited for the stream"
    assert pipe.last_windows == want_wins
    for k, o in enumerate(got):
        assert np.array_equal(o.numpy(), want[k]), k


def test_refusals(cuda_device):
    pipe, _ = _pipes(256, cuda_device)
    ok_img, ok_mask = np.zeros((40, 50, 3), np.uint8), np.full((40, 50), 255, np.uint8)
    bad = [
        (ValueError, "HoleWindowPipeline: request 1: mask of 40 x 49", [ok_img, ok_img], [ok_mask, ok_mask[:, :49]]),
        (ValueError, "HoleWindowPipeline: request 1: .*uint8", [ok_img, ok_img.astype(np.float32)], [ok_mask, ok_mask]),
        (ValueError, "HoleWindowPipeline: request 0: photo of shape", [ok_img[..., :2]], [ok_mask]),
        (TypeError, "HoleWindowPipeline: request 0", [[[1, 2, 3]]], [ok_mask]),
    ]
    for exc, match, imgs, masks in bad:
        with pytest.raises(exc, match=match):
            pipe.forward_batch(imgs, masks)
    with pytest.raises(RuntimeError, match="pinned"):
        pipe.forward_batch([torch.from_numpy(ok_img)], [ok_mask], wait=False)
    with pytest.raises(ValueError, match="margin"):
        HoleWindowPipeline(pipe.model, 256, margin=-1, device=cuda_device)
    assert np.array_equal(pipe(ok_img, ok_mask), ok_img)
