"""Keep every fixture under tests/golden/ below 1 MB: run after make_golden.py, make_golden_comodgan.py and
make_golden_pipeline.py.  Large reference outputs are replaced by a fixed row sample (rows r with r % 8 in {0, 1}, so
both phases of every 2x resampling stay covered); the tests compare the same rows of what they compute.

  migan_R*.npz        y [N,3,R,R]       -> y = y[:, :, y_rows], y_rows                (when y is above 1 MB)
  conv2d_resample.npz <case>.y          -> <case>.y = y[:, :, <case>.yrows], <case>.yrows, <case>.yshape (above 40 KB)
  pipeline.npz        the r256 request  -> pipeline_r256.npz: y_r256 in full (it is the generator output the pipeline is
                                           fed), x_r256 / final_r256 on rows_r256 (rows of x) and frows_r256 (of final)

    python tests/golden/shrink_golden.py
"""
import glob
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def rows_of(n):
    r = np.arange(n)
    return r[r % 8 < 2]


def load(path):
    z = np.load(path)
    return {k: z[k] for k in z.files}


def main():
    for path in sorted(glob.glob(os.path.join(HERE, "migan_R*.npz"))):
        d = load(path)
        if "y_rows" not in d and d["y"].nbytes > 1000000:
            d["y_rows"] = rows_of(d["y"].shape[2])
            d["y"] = np.ascontiguousarray(d["y"][:, :, d["y_rows"]])
            np.savez_compressed(path, **d)
    path = os.path.join(HERE, "conv2d_resample.npz")
    d = load(path)
    for k in [k for k in d if k.endswith(".y")]:
        name = k[:-2]
        if name + ".yrows" not in d and d[k].nbytes > 40000:
            d[name + ".yrows"], d[name + ".yshape"] = rows_of(d[k].shape[2]), np.array(d[k].shape)
            d[k] = np.ascontiguousarray(d[k][:, :, d[name + ".yrows"]])
    np.savez_compressed(path, **d)
    path = os.path.join(HERE, "pipeline.npz")
    d = load(path)
    if "x_r256" in d:
        r = {k: d.pop(k) for k in list(d) if k.endswith("_r256")}
        r["rows_r256"], r["frows_r256"] = rows_of(r["x_r256"].shape[2]), rows_of(r["final_r256"].shape[2])
        r["x_r256"] = np.ascontiguousarray(r["x_r256"][:, :, r["rows_r256"]])
        r["final_r256"] = np.ascontiguousarray(r["final_r256"][:, :, r["frows_r256"]])
        np.savez_compressed(os.path.join(HERE, "pipeline_r256.npz"), **r)
        np.savez_compressed(path, **d)
    for path in sorted(glob.glob(os.path.join(HERE, "*.npz"))):
        assert os.path.getsize(path) < 1000000, path


if __name__ == "__main__":
    main()
