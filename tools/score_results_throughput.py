"""End-to-end rate of `python -m migan_b200.score_results` at R = 512 next to `python -m migan_b200.evaluate_fid_lpips` at
migan-512 on the same photos and masks.

* data: `tools/evaluate_throughput.py`'s 2,048 seeded JPEG photos of 768 x 512 with their PNG masks, plus one seeded
  512 x 512 PNG result per photo (a method's output at R x R), written once under --data;
* commands: each module in a subprocess, wall time from start to exit (interpreter start, weight upload and the GPU
  Fréchet distance included), the two alternating, --repeats times, reported as p50 and range;
* in process: `score()` and `evaluate()` each called once to warm up, then alternating, --repeats times: the chunk
  loop's images/s and the share of its wall time spent waiting for host decode (`EvalResult.decode_wait_s`).

Seeded random weights (MI-GAN from `synthetic`, Inception and LPIPS as tools/fid_throughput.py and
tools/lpips_throughput.py build them).  Records the card name and power limit of the same run.

    python tools/score_results_throughput.py [--data /tmp/evaldata] [--num-workers 8] [--out tools/out/score.json]
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
from migan_b200 import evaluate_fid_lpips as E  # noqa: E402
from migan_b200 import score_results as S  # noqa: E402
from migan_b200 import synthetic  # noqa: E402
from evaluate_throughput import N, R, write_data  # noqa: E402
from fid_throughput import card, seeded_weights as inception_weights  # noqa: E402
from lpips_throughput import seeded_weights as lpips_weights  # noqa: E402


def write_results(root, real, seed=1):
    """One seeded R x R PNG per photo of `real`, named `<stem>.png`; kept when already there."""
    from PIL import Image
    out = os.path.join(root, "results")
    os.makedirs(out, exist_ok=True)
    paths = S.list_results(E.list_images(real), out)

    def one(i):
        if paths[i].exists():
            return
        rng = np.random.default_rng([seed, i])
        low = Image.fromarray((rng.random((R // 32, R // 32, 3)) * 255).astype(np.uint8)).resize((R, R), Image.BILINEAR)
        img = 0.85 * np.asarray(low, dtype=np.float64) + 0.15 * rng.integers(0, 256, (R, R, 3))
        Image.fromarray(img.astype(np.uint8)).save(paths[i])

    with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as pool:
        list(pool.map(one, range(len(paths))))
    return out


def run_command(args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    t = time.perf_counter()
    p = subprocess.run([sys.executable, "-m"] + args, cwd=ROOT, env=env, capture_output=True, text=True)
    wall = time.perf_counter() - t
    if p.returncode != 0:
        raise RuntimeError("%s failed:\n%s" % (args[0], p.stderr[-4000:]))
    return wall, [ln for ln in p.stdout.splitlines() if ln.startswith(("FID:", "LPIPS:"))]


def summary(values):
    return {"p50": float(np.median(values)), "min": float(min(values)), "max": float(max(values)),
            "runs": [float(v) for v in values]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", default="/tmp/migan_evaluate_throughput")
    ap.add_argument("--num-workers", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda:0")
    res = {"card": card(), "n": N, "R": R, "photo": "%dx%d JPEG" % (R * 3 // 2, R), "result": "%dx%d PNG" % (R, R),
           "num_workers": a.num_workers, "repeats": a.repeats}
    print(json.dumps({"card": res["card"]}), flush=True)
    t = time.perf_counter()
    real, masks = write_data(a.data)
    results = write_results(a.data, real)
    res["data_write_s"] = time.perf_counter() - t
    sd, isd, lsd = synthetic.export_style_state_dict(R, seed=1), inception_weights(dev), lpips_weights()
    files = {k: os.path.join(a.data, k + ".pth") for k in ("model", "inception", "lpips")}
    for k, v in zip(("model", "inception", "lpips"), (sd, isd, lsd)):
        torch.save(v, files[k])
    common = ["--real-dir", real, "--mask-dir", masks, "--num-workers", str(a.num_workers),
              "--inception-weights", files["inception"], "--lpips-weights", files["lpips"]]
    commands = {"score_results": ["migan_b200.score_results", "--resolution", str(R), "--results-dir", results] + common,
                "evaluate_fid_lpips": ["migan_b200.evaluate_fid_lpips", "--model-name", "migan-512",
                                       "--model-path", files["model"]] + common}
    walls = {k: [] for k in commands}
    for rep in range(a.repeats):
        for name, args in commands.items():
            wall, lines = run_command(args)
            walls[name].append(wall)
            print(json.dumps({"command": name, "repeat": rep, "wall_s": wall, "lines": lines}), flush=True)
    res["command_wall_s"] = {k: summary(v) for k, v in walls.items()}
    res["command_images_per_s"] = {k: summary([N / w for w in v]) for k, v in walls.items()}

    kw = dict(device=dev, num_workers=a.num_workers, inception_weights=isd, lpips_weights=lsd)
    calls = {"score_results": lambda: S.score(real, results, masks, resolution=R, **kw),
             "evaluate_fid_lpips": lambda: E.evaluate("migan-512", sd, real, masks, **kw)}
    for call in calls.values():
        call()                                                   # warm-up: uploads, workspaces
    loops = {k: [] for k in calls}
    for rep in range(a.repeats):
        for name, call in calls.items():
            r = call()
            loops[name].append(r)
            print(json.dumps({"in_process": name, "repeat": rep, "loop_s": r.seconds, "decode_wait_s": r.decode_wait_s,
                              "fid": r.fid, "lpips": r.lpips}), flush=True)
    res["loop_images_per_s"] = {k: summary([N / r.seconds for r in v]) for k, v in loops.items()}
    res["decode_wait_share"] = {k: summary([r.decode_wait_s / r.seconds for r in v]) for k, v in loops.items()}
    print(json.dumps({k: res[k] for k in ("card", "command_images_per_s", "loop_images_per_s", "decode_wait_share")}),
          flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
