"""`python -m migan_b200.crop_results` on the CPU: the reference's flags and the new ones, the refusals, the file rules of
create_onnx_pipeline.py's loop (recursive sorted listing, mask names without inner dots, `sample_results/<stem>.png`,
the last of duplicate names), the planning pass that names every bad file before anything is written, and the chunk
assignment over ranks."""
import numpy as np
import pytest
from PIL import Image

from migan_b200 import crop_results as C
from migan_b200 import demo_command as D
from migan_b200 import evaluate_fid_lpips as E


def _argv(tmp_path, *extra, resolution=256):
    return ["--resolution", str(resolution), "--model-path", "m.pt", "--images-dir", str(tmp_path / "images"),
            "--masks-dir", str(tmp_path / "masks"), "--output-dir", str(tmp_path / "out")] + list(extra)


def _save(path, a):
    path.parent.mkdir(parents=True, exist_ok=True)
    Image.fromarray(a).save(path)


def test_reference_flags_parse():
    a = C.get_args(["--resolution", "512", "--model-path", "m.pt", "--images-dir", "imgs", "--masks-dir", "masks",
                    "--invert-mask", "--output-dir", "out", "--device", "cuda"])
    assert (a.resolution, a.model_path, str(a.images_dir), str(a.masks_dir)) == (512, "m.pt", "imgs", "masks")
    assert a.invert_mask and str(a.output_dir) == "out" and a.device == "cuda"
    assert (a.generator, a.padding, a.batch_size, a.num_workers, a.noise_seed) == ("migan", 128, 32, 2, 0)
    a = C.get_args(["--resolution", "256", "--model-path", "m.pt", "--images-dir", "i", "--masks-dir", "m",
                    "--output-dir", "o", "--generator", "comodgan", "--padding", "0", "--batch-size", "8",
                    "--num-workers", "6", "--noise-seed", "3"])
    assert not a.invert_mask and a.device == "cuda"
    assert (a.generator, a.padding, a.batch_size, a.num_workers, a.noise_seed) == ("comodgan", 0, 8, 6, 3)
    with pytest.raises(SystemExit):
        C.get_args(_argv(__import__("pathlib").Path("x"), "--generator", "lama"))


def test_refusals(tmp_path):
    with pytest.raises(ValueError, match="--padding"):
        C.main(_argv(tmp_path, "--padding", "-1"))
    with pytest.raises(RuntimeError, match="CUDA"):
        C.main(_argv(tmp_path, "--device", "cpu"))
    for res in (384, 128, 1024):
        with pytest.raises(ValueError, match="comodgan"):
            C.main(_argv(tmp_path, "--generator", "comodgan", resolution=res))
    with pytest.raises(ValueError, match="--batch-size"):
        C.main(_argv(tmp_path, "--batch-size", "0"))
    with pytest.raises(ValueError, match="--noise-seed"):
        C.main(_argv(tmp_path, "--noise-seed", "-1"))
    with pytest.raises(ValueError, match="--resolution"):
        C.main(_argv(tmp_path, resolution=2))
    with pytest.raises(ValueError, match="--padding"):                 # the library call refuses before any file
        C.CropSetup("m.pt", 256, tmp_path / "images", tmp_path / "masks", tmp_path / "out", padding=-5)
    with pytest.raises(RuntimeError, match="CUDA"):
        C.CropSetup("m.pt", 256, tmp_path / "images", tmp_path / "masks", tmp_path / "out", device="cpu")
    assert not (tmp_path / "out").exists()


def test_listing_names_and_duplicates(tmp_path):
    """create_onnx_pipeline.py:323-333: .jpg / .jpeg / .png under the directory, sorted; a.b.jpg takes mask ab.png and
    writes sample_results/a.b.png; of photos with one output name only the last in sorted order is processed."""
    names = ["b.png", "a.jpg", "c.jpeg", "C.JPG", "g.gif", "sub/z.jpg", "sub/a.png", "x.y.jpg"]
    for n in names:
        (tmp_path / "images" / n).parent.mkdir(parents=True, exist_ok=True)
        (tmp_path / "images" / n).write_bytes(b"")
    photos = D.list_photos(tmp_path / "images")
    got = [p[len(str(tmp_path / "images")) + 1:] for p in photos]
    assert got == ["a.jpg", "b.png", "c.jpeg", "sub/a.png", "sub/z.jpg", "x.y.jpg"]
    items = D.plan_items(photos, tmp_path / "masks")
    by_output = {it.output: it for it in items}
    assert [it.output for it in items] == ["b.png", "c.png", "a.png", "z.png", "x.y.png"]
    assert by_output["a.png"].photo.endswith("sub/a.png") and by_output["a.png"].index == 3
    assert by_output["x.y.png"].mask == tmp_path / "masks" / "xy.png"
    assert C.RESULTS == "sample_results"


def _plan_tree(tmp_path):
    images, masks = tmp_path / "images", tmp_path / "masks"
    _save(images / "ok.png", np.zeros((40, 50, 3), np.uint8))
    _save(masks / "ok.png", np.full((7, 9), 255, np.uint8))              # any mask size is taken
    _save(images / "ok_rgba.jpg", np.zeros((30, 20, 3), np.uint8))
    _save(masks / "ok_rgba.png", np.full((300, 200, 4), 255, np.uint8))
    _save(images / "nomask.png", np.zeros((10, 10, 3), np.uint8))
    _save(images / "bad1.png", np.zeros((10, 10, 3), np.uint8))
    Image.fromarray(np.zeros((10, 10), np.uint8)).convert("1").save(masks / "bad1.png")
    _save(images / "badf.png", np.zeros((10, 10, 3), np.uint8))
    Image.fromarray(np.zeros((10, 10), np.float32), mode="F").save(masks / "badf.tiff")
    (masks / "badf.tiff").rename(masks / "badf.png")
    _save(images / "tiny.png", np.zeros((2, 40, 3), np.uint8))          # under 3 x 3: the feathering needs 3 x 3
    _save(masks / "tiny.png", np.full((2, 40), 255, np.uint8))
    _save(images / "thin.png", np.zeros((40, 2, 3), np.uint8))
    _save(masks / "thin.png", np.full((40, 40), 255, np.uint8))
    return images, masks


def test_plan_error_names_every_bad_file(tmp_path):
    images, masks = _plan_tree(tmp_path)
    items = D.plan_items(D.list_photos(images), masks)
    with pytest.raises(D.PlanError) as err:
        D.check_items(items, C.CropPipeline, 256)
    text = str(err.value)
    assert len(err.value.problems) == 5, text
    for bad in ("nomask.png", "bad1.png", "badf.png", "tiny.png", "thin.png"):
        assert sum(bad in p for p in err.value.problems) == 1, (bad, text)
    assert "mode 1 " in text and "mode F " in text and "3 x 3" in text
    assert "ok.png" not in text and "ok_rgba" not in text
    # through the command: the same error, and nothing is written
    with pytest.raises(D.PlanError):
        C.CropSetup("m.pt", 256, images, masks, tmp_path / "out", device="cuda")
    assert not (tmp_path / "out").exists()


def test_size_rule_takes_any_mask_size(tmp_path):
    images, masks = tmp_path / "images", tmp_path / "masks"
    _save(images / "a.png", np.zeros((3, 3, 3), np.uint8))
    _save(masks / "a.png", np.full((1, 1000), 255, np.uint8))
    D.check_items(D.plan_items(D.list_photos(images), masks), C.CropPipeline, 512)


@pytest.mark.parametrize("n", [1, 5, 32, 33, 100])
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("batch", [1, 8, 32])
def test_rank_assignment(n, world, batch):
    chunks = E.chunk_bounds(n, batch)
    seen = []
    for rank in range(world):
        mine = D.rank_chunks(len(chunks), rank, world)
        assert mine == sorted(mine) and all(j % world == rank for j in mine)
        seen += [i for j in mine for i in range(*chunks[j])]
    assert sorted(seen) == list(range(n))


def test_seeds_use_the_index_in_the_full_list():
    setup = C.CropSetup.__new__(C.CropSetup)
    setup.comodgan, setup.noise_seed = True, 7
    setup.items = D.plan_items(["a.jpg", "s/a.jpg", "s/b.jpg"], "M")
    setup.chunks = E.chunk_bounds(len(setup.items), 8)
    assert [int(v) for v in setup.seeds(0)] == [(7 << 32) + 1, (7 << 32) + 2]
    setup.comodgan = False
    assert setup.seeds(0) is None
