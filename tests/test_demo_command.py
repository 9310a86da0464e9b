"""`python -m migan_b200.demo` on the CPU: the reference's flags and the refusals, scripts/demo.py's file rules (recursive
sorted case-sensitive listing, mask and output names, the last of duplicate output names), the planning pass that names
every bad file before anything is written, and the chunk assignment over ranks."""
import numpy as np
import pytest
from PIL import Image

from migan_b200 import demo_command as D
from migan_b200 import evaluate_fid_lpips as E


def _argv(tmp_path, *extra, model="migan-256"):
    return ["--model-name", model, "--model-path", "m.pt", "--images-dir", str(tmp_path / "images"),
            "--masks-dir", str(tmp_path / "masks"), "--output-dir", str(tmp_path / "out")] + list(extra)


def test_reference_flags_parse():
    a = D.get_args(["--model-name", "migan-512", "--model-path", "m.pt", "--images-dir", "imgs", "--masks-dir", "masks",
                    "--invert-mask", "--output-dir", "out", "--device", "cuda"])
    assert (a.model_name, a.model_path, str(a.images_dir), str(a.masks_dir)) == ("migan-512", "m.pt", "imgs", "masks")
    assert a.invert_mask and str(a.output_dir) == "out" and a.device == "cuda"
    assert (a.batch_size, a.num_workers, a.noise_seed, a.pipeline, a.margin) == (32, 2, 0, "demo", None)
    a = D.get_args(["--model-name", "comodgan-256", "--model-path", "m.pt", "--images-dir", "i", "--masks-dir", "m",
                    "--output-dir", "o", "--batch-size", "8", "--num-workers", "6", "--noise-seed", "3",
                    "--pipeline", "holewindow", "--margin", "2"])
    assert not a.invert_mask and a.device == "cuda"
    assert (a.batch_size, a.num_workers, a.noise_seed, a.pipeline, a.margin) == (8, 6, 3, "holewindow", 2)
    with pytest.raises(SystemExit):
        D.get_args(["--model-name", "migan-256", "--model-path", "m.pt", "--images-dir", "i", "--masks-dir", "m",
                    "--output-dir", "o", "--pipeline", "crop"])


def test_refusals(tmp_path):
    with pytest.raises(Exception, match="Unsupported model name."):
        D.main(_argv(tmp_path, model="migan-1024"))
    with pytest.raises(RuntimeError, match="CUDA"):
        D.main(_argv(tmp_path, "--device", "cpu"))
    for pipeline in ("fullres", "holewindow"):
        with pytest.raises(ValueError, match="MI-GAN only"):
            D.main(_argv(tmp_path, "--pipeline", pipeline, model="comodgan-256"))
    with pytest.raises(ValueError, match="--margin"):
        D.main(_argv(tmp_path, "--margin", "2"))
    with pytest.raises(ValueError, match="--batch-size"):
        D.main(_argv(tmp_path, "--batch-size", "0"))
    assert not (tmp_path / "out").exists()


def test_listing_is_recursive_sorted_and_case_sensitive(tmp_path):
    names = ["b.png", "a.jpg", "c.jpeg", "C.JPG", "d.JPEG", "e.PNG", "f.Png", "g.gif", "h.txt", "k", "sub/z.jpg",
             "sub/deeper/y.png", "sub/A.jpeg", "other/x.JPG"]
    for n in names:
        (tmp_path / n).parent.mkdir(parents=True, exist_ok=True)
        (tmp_path / n).write_bytes(b"")
    got = [p[len(str(tmp_path)) + 1:] for p in D.list_photos(tmp_path)]
    assert got == ["a.jpg", "b.png", "c.jpeg", "sub/A.jpeg", "sub/deeper/y.png", "sub/z.jpg"]
    assert got == sorted(got)


def test_mask_and_output_names():
    assert D.mask_path("M", "/data/imgs/a.b.jpg").as_posix() == "M/ab.png"
    assert D.output_name("/data/imgs/a.b.jpg") == "a.b.png"
    assert D.mask_path("M", "sub/photo.png").as_posix() == "M/photo.png"
    assert D.output_name("sub/photo.png") == "photo.png"
    assert D.mask_path("M", "x.y.z.jpeg").as_posix() == "M/xyz.png" and D.output_name("x.y.z.jpeg") == "x.y.z.png"


def test_duplicate_output_names_keep_the_last_and_global_indices():
    photos = sorted(["r/a.jpg", "r/b.png", "r/s/a.png", "r/s/c.jpg", "r/t/a.jpeg", "r/t/b.jpg", "r/u.v.jpg", "r/z.jpg"])
    items = D.plan_items(photos, "M")
    assert photos == ["r/a.jpg", "r/b.png", "r/s/a.png", "r/s/c.jpg", "r/t/a.jpeg", "r/t/b.jpg", "r/u.v.jpg", "r/z.jpg"]
    assert [(it.index, it.photo, it.output) for it in items] == [
        (3, "r/s/c.jpg", "c.png"), (4, "r/t/a.jpeg", "a.png"), (5, "r/t/b.jpg", "b.png"), (6, "r/u.v.jpg", "u.v.png"),
        (7, "r/z.jpg", "z.png")]
    assert items[3].mask.as_posix() == "M/uv.png"
    assert len({it.output for it in items}) == len(items)


def _save(path, arr, mode=None, fmt=None):
    path.parent.mkdir(parents=True, exist_ok=True)
    im = Image.fromarray(arr) if mode is None else Image.fromarray(arr).convert(mode)
    im.save(path, format=fmt)


def test_planning_names_every_bad_file_and_writes_nothing(tmp_path):
    images, masks = tmp_path / "images", tmp_path / "masks"
    rgb = np.zeros((40, 60, 3), np.uint8)
    gray = np.full((40, 60), 255, np.uint8)
    for name in ("ok_l", "ok_p", "ok_la", "ok_rgba", "ok_cmyk", "nomask", "bad1", "badi16", "badf", "badsize"):
        _save(images / (name + ".jpg"), rgb)
    _save(images / "sub" / "nomask2.png", rgb)
    _save(masks / "ok_l.png", gray)
    _save(masks / "ok_p.png", gray, "P")
    _save(masks / "ok_la.png", gray, "LA")
    _save(masks / "ok_rgba.png", gray, "RGBA")
    _save(masks / "ok_cmyk.png", gray, "CMYK", fmt="JPEG")     # a JPEG under a .png name: PIL reads by content
    _save(masks / "bad1.png", gray, "1")
    Image.fromarray(gray.astype(np.uint16) * 257).save(masks / "badi16.png")
    Image.fromarray(gray.astype(np.float32)).save(masks / "badf.png", format="TIFF")
    _save(masks / "badsize.png", np.full((40, 61), 255, np.uint8))
    with Image.open(masks / "badi16.png") as im:
        i16_mode = im.mode
    assert i16_mode.startswith("I")
    with pytest.raises(D.PlanError) as err:
        D.main(_argv(tmp_path))
    problems = err.value.problems
    text = str(err.value)
    assert len(problems) == 6, text
    for bad in ("nomask.png", "nomask2.png", "bad1.png", "badi16.png", "badf.png", "badsize.png"):
        assert sum(bad in p for p in problems) == 1, (bad, text)
    assert "mode 1 " in text and "mode %s " % i16_mode in text and "mode F " in text
    assert not any(s in text for s in ("ok_l.png", "ok_p.png", "ok_la.png", "ok_rgba.png", "ok_cmyk.png"))
    assert not (tmp_path / "out").exists()


def test_fullres_size_rule_is_the_photo_size(tmp_path):
    images, masks = tmp_path / "images", tmp_path / "masks"
    _save(images / "a.png", np.zeros((300, 500, 3), np.uint8))
    _save(masks / "a.png", np.full((600, 1000), 255, np.uint8))         # the demo rule takes it, full resolution not
    items = D.plan_items(D.list_photos(images), masks)
    D.check_items(items, "demo", 256)
    for pipeline in ("fullres", "holewindow"):
        with pytest.raises(D.PlanError, match="a.png"):
            D.check_items(items, pipeline, 256)


@pytest.mark.parametrize("mode,supported", [("L", True), ("P", True), ("LA", True), ("PA", True), ("RGB", True),
                                            ("RGBA", True), ("CMYK", True), ("1", False), ("I", False),
                                            ("I;16", False), ("F", False), ("no such mode", False)])
def test_mask_modes(mode, supported):
    assert D.mask_mode_supported(mode) == supported


def test_decode_mask_refuses_other_modes(tmp_path):
    Image.fromarray(np.zeros((4, 4), np.uint8)).convert("1").save(tmp_path / "m.png")
    with pytest.raises(ValueError, match="m.png: mode 1"):
        D.decode_mask(tmp_path / "m.png")


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("batch", [1, 7, 32])
def test_chunk_assignment_covers_every_image_once(n, world, batch):
    chunks = E.chunk_bounds(n, batch)
    seen = []
    for rank in range(world):
        mine = D.rank_chunks(len(chunks), rank, world)
        assert mine == sorted(mine) and all(j % world == rank for j in mine)
        seen += [i for j in mine for i in range(*chunks[j])]
    assert sorted(seen) == list(range(n))


def test_seeds_use_the_index_in_the_full_list():
    setup = D.DemoSetup.__new__(D.DemoSetup)             # the seeds need only the plan and the chunking
    setup.comodgan, setup.noise_seed = True, 5
    setup.items = D.plan_items(["a.jpg", "s/a.jpg", "s/b.jpg", "t/a.jpg"], "M")
    setup.chunks = E.chunk_bounds(len(setup.items), 1)
    assert [it.index for it in setup.items] == [2, 3]
    assert [int(setup.seeds(j)[0]) for j in range(2)] == [(5 << 32) + 2, (5 << 32) + 3]
    assert setup.seeds(0).dtype == np.uint64
    setup.comodgan = False
    assert setup.seeds(0) is None
