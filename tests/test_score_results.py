"""`python -m migan_b200.score_results` on the CPU: the result-file pairing (`<stem>.png`, extra files ignored), the
planning pass that names every missing or unreadable result and mask in one `PlanError` before any device is touched,
and the argument refusals."""
import numpy as np
import pytest
import torch

from migan_b200 import evaluate_fid_lpips as E
from migan_b200 import score_results as S
from migan_b200.demo_command import PlanError


def _png(path, h=6, w=5, mode="RGB"):
    from PIL import Image
    shape = (h, w, 3) if mode == "RGB" else (h, w)
    Image.fromarray(np.full(shape, 200, np.uint8)).save(path)


def _jpg(path, h=6, w=5):
    from PIL import Image
    Image.fromarray(np.full((h, w, 3), 90, np.uint8)).save(path, quality=90)


def test_pairing_keeps_inner_dots_and_ignores_extra_files(tmp_path):
    real, results, masks = tmp_path / "real", tmp_path / "results", tmp_path / "masks"
    for d in (real, results, masks):
        d.mkdir()
    for name in ("a.b.jpg", "c.png", "d.JPEG"):
        (_jpg if name.endswith(("jpg", "JPEG")) else _png)(real / name)
    for stem in ("a.b", "c", "d"):
        _png(results / (stem + ".png"), 9, 11)
        _png(masks / (stem + ".png"), mode="L")
    for extra in ("a.png", "ab.png", "zzz.png", "c.jpg"):              # not the result of any photo
        _png(results / extra)
    (results / "notes.txt").write_text("not a result")
    images = E.list_images(real)
    assert [p.name for p in images] == ["a.b.jpg", "c.png", "d.JPEG"]
    got = S.list_results(images, results)
    assert [p.name for p in got] == ["a.b.png", "c.png", "d.png"] and all(p.parent == results for p in got)
    assert E.stem_pngs(images, masks) == E.list_masks(images, masks)      # the masks' rule
    S.check_files(images, got, E.list_masks(images, masks))              # nothing missing: no error


@pytest.fixture
def no_device(monkeypatch):
    """Any CUDA initialisation, and any setup of the networks, fails the test."""
    def touched(*a, **k):
        raise AssertionError("a device was touched before the planning pass finished")
    monkeypatch.setattr(torch.cuda, "_lazy_init", touched)
    monkeypatch.setattr(torch.cuda, "init", touched)
    monkeypatch.setattr(E, "EvalSetup", touched)


def test_one_plan_error_names_every_bad_file_before_any_device_work(tmp_path, no_device):
    real, results, masks = tmp_path / "real", tmp_path / "results", tmp_path / "masks"
    for d in (real, results, masks):
        d.mkdir()
    for stem in ("p0", "p1", "p2", "p3", "p4", "p5"):
        _jpg(real / (stem + ".jpg"))
    (real / "p6.png").write_bytes(b"not a png")                        # unreadable photo
    for stem in ("p0", "p2", "p3", "p4", "p5", "p6"):                   # p1: no result
        _png(results / (stem + ".png"), 8, 8)
    (results / "p2.png").write_bytes(b"\x89PNG truncated")             # unreadable result
    for stem in ("p0", "p1", "p2", "p3", "p5", "p6"):                   # p4: no mask
        _png(masks / (stem + ".png"), mode="L")
    (masks / "p5.png").write_bytes(b"")                                 # unreadable mask
    with pytest.raises(PlanError) as e:
        S.score(real, results, masks, resolution=256, device="cuda")
    problems = e.value.problems
    assert len(problems) == 5, problems
    assert problems[0].startswith("photo p1.jpg: no result") and problems[0].endswith("p1.png")
    assert problems[1].startswith("result %s: cannot be read" % (results / "p2.png"))
    assert problems[2].startswith("photo p4.jpg: no mask") and problems[2].endswith("p4.png")
    assert problems[3].startswith("mask %s: cannot be read" % (masks / "p5.png"))
    assert problems[4].startswith("photo %s: cannot be read" % (real / "p6.png"))
    assert str(len(problems)) in str(e.value)
    with pytest.raises(PlanError) as e:                                 # generated masks: photos and results only
        S.score(real, results, None, resolution=512, device="cuda")
    assert len(e.value.problems) == 3
    (real / "p6.png").unlink()
    (real / "p6.txt").write_text("")
    _png(real / "p7.png")                                               # p7: no result, no mask
    (real / "p8.PNG").write_bytes(b"garbage")                          # unreadable photo, no result, no mask
    with pytest.raises(PlanError) as e:
        S.score(real, results, masks, resolution=256, device="cuda")
    names = "\n".join(e.value.problems)
    assert len(e.value.problems) == 9, names
    for want in ("photo p7.png: no result", "photo p7.png: no mask", "photo %s: cannot be read" % (real / "p8.PNG"),
                 "photo p8.PNG: no result", "photo p8.PNG: no mask"):
        assert want in names


def _argv(tmp_path, *extra):
    return ["--resolution", "256", "--real-dir", str(tmp_path), "--results-dir", str(tmp_path)] + list(extra)


def test_argument_refusals(tmp_path, no_device):
    with pytest.raises(ValueError, match="--ids"):
        S.main(_argv(tmp_path, "--real-stats", "r.npz", "--ids"))
    with pytest.raises(ValueError, match="exclude each other"):
        S.main(_argv(tmp_path, "--real-stats", "r.npz", "--save-real-stats", "s.npz"))
    with pytest.raises(SystemExit):
        S.main(["--resolution", "384", "--real-dir", str(tmp_path), "--results-dir", str(tmp_path)])
    with pytest.raises(ValueError, match="--resolution"):
        S.score(tmp_path, tmp_path, resolution=384)
    with pytest.raises(RuntimeError, match="CUDA"):
        S.main(_argv(tmp_path, "--device", "cpu"))
    with pytest.raises(RuntimeError, match="CUDA"):
        S.score(tmp_path, tmp_path, resolution=256, device="cpu")
    a = S.get_args(_argv(tmp_path, "--mask-dir", "m", "--batch-size", "8", "--num-workers", "3", "--ids",
                         "--save-real-stats", "s.npz", "--inception-weights", "i.pth", "--lpips-weights", "l.pth"))
    assert (a.resolution, a.batch_size, a.num_workers, a.ids, a.device) == (256, 8, 3, True, "cuda")
    assert (str(a.mask_dir), str(a.save_real_stats), a.real_stats) == ("m", "s.npz", None)
    assert (str(a.inception_weights), str(a.lpips_weights)) == ("i.pth", "l.pth")
    a = S.get_args(_argv(tmp_path))
    assert a.mask_dir is None and a.batch_size == 32 and a.num_workers == 2 and not a.ids


def test_setup_refuses_a_mixed_source(tmp_path):
    for d in ("a", "b"):
        _png(tmp_path / ("%s.png" % d))
    with pytest.raises(ValueError, match="model_name=None"):
        E.EvalSetup("migan-256", None, tmp_path, results=[tmp_path / "a.png", tmp_path / "b.png"], res=256)
    with pytest.raises(ValueError, match="model_name=None"):
        E.EvalSetup(None, None, tmp_path, results=[tmp_path / "a.png", tmp_path / "b.png"])
