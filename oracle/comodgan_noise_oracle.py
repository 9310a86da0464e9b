"""The seeded noise streams of `comodgan_seeded_noise` (include/comodgan_b200.h) in numpy: an oracle independent of the
CUDA code.

Request i with seed s has stream p = 0 (z, 512 values) and p = 1 + j (noise plane j, r_j^2 values, row-major).  Stream p
is numpy's Philox4x64-10 with key [s, p]; values 2t, 2t+1 come from the words w[2t], w[2t+1] by Box-Muller in float64,
each rounded once to float32.
"""
from typing import List, Sequence, Tuple

import numpy as np

Z_DIM = 512


def raw_words(seed: int, stream: int, count: int) -> np.ndarray:
    """The first `count` 64-bit words of stream `stream` of a request with seed `seed`."""
    return np.random.Philox(key=np.array([seed, stream], np.uint64)).random_raw(count)


def normals(seed: int, stream: int, count: int) -> np.ndarray:
    """The first `count` (even) float32 values of the stream."""
    w = raw_words(seed, stream, count)
    a, b = w[0::2], w[1::2]
    u1 = ((a >> np.uint64(11)) + np.uint64(1)).astype(np.float64) * 2.0 ** -53
    u2 = (b >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    rho = np.sqrt(-2.0 * np.log(u1))
    t = 2.0 * np.pi * u2
    out = np.empty(count, np.float64)
    out[0::2], out[1::2] = rho * np.cos(t), rho * np.sin(t)
    return out.astype(np.float32)


def plane_res(resolution: int) -> List[int]:
    """r_j of the noise planes in forward order (b4.conv, b8.conv0, b8.conv1, ...)."""
    return [4] + [2 ** i for i in range(3, int(np.log2(resolution)) + 1) for _ in range(2)]


def seeded_noise(seeds: Sequence[int], resolution: int) -> Tuple[np.ndarray, np.ndarray]:
    """(z [n, 512], planes) for `seeds`; planes are concatenated plane by plane, each [n, r_j, r_j] (comodgan_forward's
    RANDOM layout)."""
    seeds = [int(s) for s in seeds]
    z = np.stack([normals(s, 0, Z_DIM) for s in seeds])
    planes = [np.stack([normals(s, 1 + j, r * r) for s in seeds]) for j, r in enumerate(plane_res(resolution))]
    return z, np.concatenate([p.reshape(-1) for p in planes])


def plane_dict(planes: np.ndarray, keys, n: int) -> dict:
    """The flat planes as `comodgan_oracle.generator_forward`'s noise dict: {layer prefix: [n, 1, r, r]}, keys from
    `comodgan_oracle.noise_keys`."""
    out, off = {}, 0
    for key, r in keys:
        out[key] = planes[off:off + n * r * r].reshape(n, 1, r, r)
        off += n * r * r
    return out
