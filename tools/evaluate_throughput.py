"""End-to-end rate of `python -m migan_b200.evaluate_fid_lpips` at migan-512 on a seeded synthetic directory, next to the
loop the unmodified evaluation script runs under `dropin` on the same files.

* data: 2,048 JPEG photos of 1.5R x R (768 x 512) at R = 512 and their PNG masks, written once under --data (seeded);
* command: the module in a subprocess, wall time from start to exit (interpreter start, weight upload and the GPU
  Fréchet distance included), at W = 1 and, under torchrun, at W = 2, 4, 8 when the box has that many GPUs;
* in process: `evaluate()` called twice, the second timed: the chunk loop's images/s, the host time spent waiting for
  decoded chunks against the loop's wall time, with --mask-dir and with generated masks;
* dropin: the script's loop under `dropin` (decode on --num-workers threads, PIL BICUBIC / NEAREST resizes and x on the
  host, `Generator(x)`, the composite on the host, LPIPS and Inception on the GPU, batch 8 as the script's default), then
  `np.cov` of the activations and `calculate_frechet_distance` (scipy `sqrtm`) on the host;
* the rounding dependence on --batch-size: FID and LPIPS at batch sizes 32, 8 and 7 (in process);
* the generated-mask cost every rank pays at any W: `RandomMaskStream(512).next(2048)`.

Seeded random weights (MI-GAN from `synthetic`, Inception and LPIPS as tools/fid_throughput.py and
tools/lpips_throughput.py build them).  Records the card name and power limit of the same run.

    python tools/evaluate_throughput.py [--data /tmp/evaldata] [--num-workers 8] [--out tools/out/evaluate_throughput.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import migan_b200  # noqa: E402
from migan_b200 import evaluate_fid_lpips as E  # noqa: E402
from migan_b200 import fid, lpips, synthetic  # noqa: E402
from comodgan_eval_throughput import dropin_batch  # noqa: E402
from fid_throughput import card, seeded_weights as inception_weights  # noqa: E402
from lpips_throughput import seeded_weights as lpips_weights  # noqa: E402

R = 512
N = 2048
DROPIN_BATCH = 8


def write_data(root, n=N, seed=0):
    """n seeded JPEG photos of 1.5R x R (smooth blobs plus noise) and their hole masks; kept when already there."""
    from PIL import Image
    real, masks = os.path.join(root, "real"), os.path.join(root, "masks")
    os.makedirs(real, exist_ok=True)
    os.makedirs(masks, exist_ok=True)
    H, W = R, R * 3 // 2

    def one(i):
        name = "photo_%05d" % i
        if os.path.exists(os.path.join(masks, name + ".png")):
            return
        rng = np.random.default_rng([seed, i])
        low = Image.fromarray((rng.random((H // 32, W // 32, 3)) * 255).astype(np.uint8)).resize((W, H), Image.BILINEAR)
        img = 0.85 * np.asarray(low, dtype=np.float64) + 0.15 * rng.integers(0, 256, (H, W, 3))
        Image.fromarray(img.astype(np.uint8)).save(os.path.join(real, name + ".jpg"), quality=90)
        m = np.where(rng.random((H // 16, W // 16)) < 0.3, 0, 255).astype(np.uint8)
        Image.fromarray(m).resize((W, H), Image.NEAREST).save(os.path.join(masks, name + ".png"))

    with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as pool:
        list(pool.map(one, range(n)))
    return real, masks


def command(files, real, masks, workers, world):
    args = ["-m", "migan_b200.evaluate_fid_lpips", "--model-name", "migan-512", "--model-path", files["model"],
            "--real-dir", real, "--mask-dir", masks, "--num-workers", str(workers),
            "--inception-weights", files["inception"], "--lpips-weights", files["lpips"]]
    if world > 1:
        args = ["-m", "torch.distributed.run", "--standalone", "--nproc_per_node=%d" % world] + args
    env = dict(os.environ, PYTHONPATH=ROOT)
    t = time.perf_counter()
    p = subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True, text=True)
    wall = time.perf_counter() - t
    if p.returncode != 0:
        raise RuntimeError("command failed at W=%d:\n%s" % (world, p.stderr[-4000:]))
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith(("FID:", "LPIPS:"))]
    return {"world_size": world, "wall_s": wall, "images_per_s": N / wall, "lines": lines}


def dropin_loop(sd, inception, net, real, masks, workers, dev):
    """The script's loop under dropin: host dataset work, Generator(x), host composite, GPU metrics, host FID."""
    from PIL import Image
    model = migan_b200.Generator(R)
    model.load_state_dict(sd)
    model = model.to(dev).eval()
    paths = E.list_images(real)
    mpaths = E.list_masks(paths, masks)

    def load(i):
        return np.array(Image.open(paths[i]).convert("RGB")), np.array(Image.open(mpaths[i]).convert("L"))

    acts_r, acts_f, vals = np.empty((len(paths), 2048)), np.empty((len(paths), 2048)), []
    t = time.perf_counter()
    with ThreadPoolExecutor(max_workers=workers) as pool, torch.no_grad():
        for b0 in range(0, len(paths), DROPIN_BATCH):
            items = list(pool.map(load, range(b0, min(b0 + DROPIN_BATCH, len(paths)))))
            im, comp = dropin_batch(model, [a for a, _ in items], [m for _, m in items], R, dev)
            vals.extend(net(im, comp, normalize=True).detach().cpu().numpy().reshape(-1).tolist())
            acts_r[b0:b0 + len(items)] = inception(im)[0].view(len(items), -1).cpu().numpy()
            acts_f[b0:b0 + len(items)] = inception(comp)[0].view(len(items), -1).cpu().numpy()
    loop = time.perf_counter() - t
    value = fid.calculate_frechet_distance(np.mean(acts_r, 0), np.cov(acts_r, rowvar=False), np.mean(acts_f, 0),
                                           np.cov(acts_f, rowvar=False))
    wall = time.perf_counter() - t
    return {"loop_s": loop, "wall_s": wall, "images_per_s": len(paths) / wall, "loop_images_per_s": len(paths) / loop,
            "fid": value, "lpips": float(np.mean(vals))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", default="/tmp/migan_evaluate_throughput")
    ap.add_argument("--num-workers", type=int, default=8)
    ap.add_argument("--skip-dropin", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda:0")
    res = {"card": card(), "gpus": torch.cuda.device_count(), "n": N, "R": R, "photo": "%dx%d JPEG" % (R * 3 // 2, R),
           "num_workers": a.num_workers}
    t = time.perf_counter()
    real, masks = write_data(a.data)
    res["data_write_s"] = time.perf_counter() - t
    sd, isd, lsd = synthetic.export_style_state_dict(R, seed=1), inception_weights(dev), lpips_weights()
    files = {k: os.path.join(a.data, k + ".pth") for k in ("model", "inception", "lpips")}
    for k, v in zip(("model", "inception", "lpips"), (sd, isd, lsd)):
        torch.save(v, files[k])
    print(json.dumps({"card": res["card"], "gpus": res["gpus"]}), flush=True)

    res["command"] = [command(files, real, masks, a.num_workers, 1)]
    print(json.dumps(res["command"][-1]), flush=True)
    for world in (2, 4, 8):
        if world <= res["gpus"]:
            res["command"].append(command(files, real, masks, a.num_workers, world))
            print(json.dumps(res["command"][-1]), flush=True)

    def in_process(mask_dir, batch_size=32):
        kw = dict(device=dev, batch_size=batch_size, num_workers=a.num_workers, inception_weights=isd, lpips_weights=lsd)
        E.evaluate("migan-512", sd, real, mask_dir, **kw)                  # warm-up: uploads, workspaces
        r = E.evaluate("migan-512", sd, real, mask_dir, **kw)
        return {"batch_size": batch_size, "masks": "dir" if mask_dir else "generated", "fid": r.fid, "lpips": r.lpips,
                "loop_s": r.seconds, "images_per_s": r.count / r.seconds, "decode_wait_s": r.decode_wait_s,
                "decode_wait_share": r.decode_wait_s / r.seconds}

    res["in_process"] = [in_process(masks), in_process(None)]
    for row in res["in_process"]:
        print(json.dumps(row), flush=True)
    rows = [res["in_process"][0]] + [in_process(masks, b) for b in (8, 7)]
    base = rows[0]
    res["batch_size_dependence"] = [{"batch_size": r["batch_size"], "fid": r["fid"], "lpips": r["lpips"],
                                     "fid_rel_diff_vs_32": abs(r["fid"] - base["fid"]) / abs(base["fid"]),
                                     "lpips_rel_diff_vs_32": abs(r["lpips"] - base["lpips"]) / abs(base["lpips"])}
                                    for r in rows]
    print(json.dumps({"batch_size_dependence": res["batch_size_dependence"]}), flush=True)

    stream = migan_b200.RandomMaskStream(R, seed=0, device=dev)
    stream.next(256)
    torch.cuda.synchronize()
    t = time.perf_counter()
    stream.next(N)
    torch.cuda.synchronize()
    res["generated_masks_every_rank_s"] = time.perf_counter() - t
    print(json.dumps({"generated_masks_every_rank_s": res["generated_masks_every_rank_s"]}), flush=True)

    if not a.skip_dropin:
        net = lpips.LPIPS(net="alex", weights=lsd).to(dev)
        res["dropin"] = dropin_loop(sd, fid.InceptionV3(weights=isd), net, real, masks, a.num_workers, dev)
        print(json.dumps({"dropin": res["dropin"], "card": res["card"]}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
