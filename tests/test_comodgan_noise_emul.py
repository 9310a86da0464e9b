"""CPU check of the seeded Co-Mod-GAN noise (`comodgan_seeded_noise`, `comodgan_forward_seeded`) through the emulation
build, against numpy's own Philox (oracle/comodgan_noise_oracle.py), and of the argument checks of the Python layer."""
import contextlib
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))

import build_emul  # noqa: E402
from migan_b200 import _abi, comodgan  # noqa: E402
from migan_b200._request_path import NoiseSeeds, load_generator  # noqa: E402
from oracle import comodgan_noise_oracle as N  # noqa: E402
from oracle import comodgan_oracle as C  # noqa: E402
from oracle import migan_oracle as O  # noqa: E402

SEEDS = [0, 1, 12345, 2 ** 32 + 7, 2 ** 63, 2 ** 64 - 1]


@pytest.fixture(scope="module")
def emul():
    return _abi.bind(ctypes.CDLL(build_emul.build()), _abi.COMOD_SYMBOLS)


@pytest.fixture(scope="module")
def harness():
    lib = ctypes.CDLL(build_emul.build_harness("noise_emul.cpp"))
    lib.noise_words.argtypes = [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int64, ctypes.c_void_p]
    lib.noise_values.argtypes = [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_int64, ctypes.c_void_p]
    return lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _ulps(got: np.ndarray, want: np.ndarray) -> np.ndarray:
    """Distance in float32 ulps (both finite; the values straddle no sign change at the sizes compared)."""
    g, w = got.astype(np.float32).view(np.int32).astype(np.int64), want.astype(np.float32).view(np.int32).astype(np.int64)
    g = np.where(g < 0, -(g & 0x7FFFFFFF), g)
    w = np.where(w < 0, -(w & 0x7FFFFFFF), w)
    return np.abs(g - w)


@pytest.mark.parametrize("seed", SEEDS)
def test_raw_words_equal_numpy_philox(harness, seed):
    for stream in (0, 1, 2, 17, 2 ** 64 - 1):
        words = np.empty(4 * 300, np.uint64)
        harness.noise_words(seed, stream, 300, _ptr(words))
        assert np.array_equal(words, N.raw_words(seed, stream, words.size)), (seed, stream)


def test_normals_within_one_ulp_of_numpy(harness):
    total, differ = 0, 0
    for seed in SEEDS:
        for stream in (0, 1, 9):
            got = np.empty(4 * 20000, np.float32)
            harness.noise_values(seed, stream, 20000, _ptr(got))
            want = N.normals(seed, stream, got.size)
            d = _ulps(got, want)
            assert int(d.max()) <= 1, (seed, stream)
            total += d.size
            differ += int((d != 0).sum())
    print("seeded normals: %d of %d values differ from numpy (by one float32 ulp)" % (differ, total))
    # the stream is N(0, 1)
    v = N.normals(3, 1, 1 << 20).astype(np.float64)
    assert abs(v.mean()) < 5e-3 and abs(v.std() - 1.0) < 5e-3


def _ctx(lib, R):
    h = ctypes.c_void_p()
    _abi.check_comod(lib.comodgan_create(R, 0, ctypes.byref(h)), lib)
    return h


def test_plane_layout_n3_r16(emul):
    R, seeds = 16, np.array([5, 2 ** 64 - 1, 0], np.uint64)
    h = _ctx(emul, R)
    z_want, planes_want = N.seeded_noise(seeds, R)
    assert planes_want.size == 3 * sum(r * r for r in N.plane_res(R))
    z = np.full((3, 512), np.nan, np.float32)
    planes = np.full(planes_want.size, np.nan, np.float32)
    _abi.check_comod(emul.comodgan_seeded_noise(h, _ptr(seeds), 3, _ptr(z), _ptr(planes), None), emul)
    assert int(_ulps(z, z_want).max()) <= 1 and int(_ulps(planes, planes_want).max()) <= 1
    # a request's values do not depend on n or its position; z and the planes are drawn independently
    z1 = np.empty((1, 512), np.float32)
    p1 = np.empty(sum(r * r for r in N.plane_res(R)), np.float32)
    _abi.check_comod(emul.comodgan_seeded_noise(h, _ptr(seeds[1:2]), 1, None, _ptr(p1), None), emul)
    _abi.check_comod(emul.comodgan_seeded_noise(h, _ptr(seeds[1:2]), 1, _ptr(z1), None, None), emul)
    assert np.array_equal(z1[0], z[1])
    off = 0
    for r in N.plane_res(R):
        assert np.array_equal(planes[off * 3 + r * r:off * 3 + 2 * r * r], p1[off:off + r * r]), r
        off += r * r
    # more than 64 requests: one launch per 64, the same values
    many = np.arange(70, dtype=np.uint64) * np.uint64(977)
    zm = np.empty((70, 512), np.float32)
    _abi.check_comod(emul.comodgan_seeded_noise(h, _ptr(many), 70, _ptr(zm), None, None), emul)
    assert int(_ulps(zm, N.seeded_noise(many, R)[0]).max()) <= 1
    # refusals
    assert emul.comodgan_seeded_noise(h, None, 3, _ptr(z), None, None) == _abi.ERR_INVALID
    assert emul.comodgan_seeded_noise(h, _ptr(seeds), 0, _ptr(z), None, None) == _abi.ERR_INVALID
    assert emul.comodgan_seeded_noise(h, _ptr(seeds), 3, None, None, None) == _abi.ERR_INVALID
    assert emul.comodgan_seeded_noise(h, _ptr(seeds), 3, ctypes.c_void_p(z.ctypes.data + 4), None, None) == _abi.ERR_INVALID
    emul.comodgan_destroy(h)


def _finalized(lib, R, sd):
    h = _ctx(lib, R)
    keep = []
    for k, v in sd.items():
        a = np.ascontiguousarray(v.numpy(), np.float32)
        keep.append(a)
        _abi.check_comod(lib.comodgan_set_weight(h, k.encode(), _ptr(a), a.size), lib)
    _abi.check_comod(lib.comodgan_finalize_weights(h), lib)
    return h


def _aligned(nbytes):
    raw = np.empty(nbytes + 256, dtype=np.uint8)
    off = (-raw.ctypes.data) % 256
    return raw, raw[off:off + nbytes]


def test_forward_seeded_equals_random_mode_on_oracle_planes(emul):
    R, n = 16, 3
    sd = C.make_state_dict(R, seed=1)
    h = _finalized(emul, R, sd)
    x = np.ascontiguousarray(O.make_input(R, n, seed=77).numpy(), np.float32)
    seeds = np.array([11, 0, 2 ** 64 - 1], np.uint64)
    need = emul.comodgan_workspace_bytes_seeded(h, n)
    assert need > emul.comodgan_workspace_bytes(h, n)
    _raw, ws = _aligned(need)
    y_seeded = np.empty((n, 3, R, R), np.float32)
    _abi.check_comod(emul.comodgan_forward_seeded(h, _ptr(x), _ptr(seeds), None, _ptr(y_seeded), n, 1.0, -1, _ptr(ws), need,
                                                  None), emul)
    seeded_launches = emul.comodgan_last_launch_count(h)
    # the planes and z it drew, through the noise call itself
    z = np.empty((n, 512), np.float32)
    planes = np.empty(n * sum(r * r for r in N.plane_res(R)), np.float32)
    _abi.check_comod(emul.comodgan_seeded_noise(h, _ptr(seeds), n, _ptr(z), _ptr(planes), None), emul)
    need_f = emul.comodgan_workspace_bytes(h, n)
    _raw2, ws2 = _aligned(need_f)
    y_random = np.empty_like(y_seeded)
    _abi.check_comod(emul.comodgan_forward(h, _ptr(x), _ptr(z), _ptr(y_random), n, 1.0, -1, 2, _ptr(planes), _ptr(ws2), need_f,
                                           None), emul)
    assert np.array_equal(y_seeded, y_random)
    assert seeded_launches == emul.comodgan_last_launch_count(h) + 1     # the noise launch
    # with the oracle's draws, against the Co-Mod-GAN oracle
    z_or, planes_or = N.seeded_noise(seeds, R)
    noise = {k: torch.from_numpy(v) for k, v in N.plane_dict(planes_or, C.noise_keys(R), n).items()}
    y_or = C.generator_forward(sd, torch.from_numpy(x), torch.from_numpy(z_or), R, noise_mode="random", noise=noise)
    assert float((torch.from_numpy(y_seeded) - y_or).abs().max()) < 2e-4
    # an explicit z is used as it is
    y_z = np.empty_like(y_seeded)
    _abi.check_comod(emul.comodgan_forward_seeded(h, _ptr(x), _ptr(seeds), _ptr(z), _ptr(y_z), n, 1.0, -1, _ptr(ws), need,
                                                  None), emul)
    assert np.array_equal(y_z, y_seeded)
    # refusals
    assert emul.comodgan_forward_seeded(h, _ptr(x), None, None, _ptr(y_z), n, 1.0, -1, _ptr(ws), need, None) == _abi.ERR_INVALID
    assert emul.comodgan_forward_seeded(h, _ptr(x), _ptr(seeds), None, _ptr(y_z), n, 1.0, -1, _ptr(ws), need - 256,
                                        None) == _abi.ERR_WORKSPACE
    emul.comodgan_destroy(h)


def test_batch_coupling_of_the_style_normalisation(emul):
    """The forward is not batch invariant: the demodulated layers scale the styles by one RMS over the whole batch
    (stylegan.py:146, InvRmsAllK), so an image's bytes depend on its batch.  The seeded draws are per image; the
    difference is rounding only."""
    R = 16
    sd = C.make_state_dict(R, seed=1)
    h = _finalized(emul, R, sd)
    seeds = np.array([3, 4, 5], np.uint64)
    x = np.ascontiguousarray(O.make_input(R, 3, seed=9).numpy(), np.float32)

    def run(xs, ss):
        n = len(ss)
        need = emul.comodgan_workspace_bytes_seeded(h, n)
        _raw, ws = _aligned(need)
        y = np.empty((n, 3, R, R), np.float32)
        _abi.check_comod(emul.comodgan_forward_seeded(h, _ptr(np.ascontiguousarray(xs)), _ptr(np.ascontiguousarray(ss)), None,
                                                      _ptr(y), n, 1.0, -1, _ptr(ws), need, None), emul)
        return y

    y3 = run(x, seeds)
    assert np.array_equal(run(x, seeds), y3)                             # same batch: same bytes
    y1 = run(x[1:2], seeds[1:2])
    assert np.abs(y1[0] - y3[1]).max() < 1e-4
    emul.comodgan_destroy(h)


# ---- the Python layer --------------------------------------------------------------------------------------------------
@pytest.fixture()
def emul_generator(emul, monkeypatch):
    """migan_b200.comodgan routed to the emulation library, CPU tensors standing in for device memory."""
    monkeypatch.setattr(_abi, "load", lambda build_if_missing=False: emul)
    monkeypatch.setattr(comodgan, "_guard", lambda device: contextlib.nullcontext())
    monkeypatch.setattr(comodgan, "_stream", lambda device: None)
    monkeypatch.setattr(comodgan, "_device_index", lambda device: 0)

    class EmulGenerator(comodgan.Generator):
        def _validate(self, x, z, draw_z=True):
            if z is None and draw_z:
                z = torch.randn([x.shape[0], 512])
            return x.contiguous(), None if z is None else z.contiguous()

    sd = C.make_state_dict(16, seed=1)
    g = EmulGenerator(comodgan.Mapping(num_ws=6), comodgan.Encoder(resolution=16), comodgan.Synthesis(resolution=16))
    g.load_state_dict(sd, strict=True)
    return g.eval()


def test_python_forward_seeds(emul_generator):
    g = emul_generator
    x = O.make_input(16, 3, seed=4)
    seeds = [7, 2 ** 64 - 1, 0]
    y = g(x, seeds=seeds)
    z_or, planes_or = N.seeded_noise(seeds, 16)
    # the oracle's draws agree to one float32 ulp, so the outputs agree to rounding
    assert float((y - g(x, z=torch.from_numpy(z_or), noise=torch.from_numpy(planes_or))).abs().max()) < 1e-4
    assert torch.equal(g(x, seeds=torch.tensor([7, -1, 0], dtype=torch.int64)), y)    # int64 bits = uint64 seeds
    z = torch.from_numpy(z_or)
    assert torch.equal(g(x, z=z, seeds=seeds), y)
    with pytest.raises(ValueError):
        g(x, seeds=[1, 2])                                               # length != n
    with pytest.raises(ValueError):
        g(x, seeds=seeds, noise_mode="const")
    with pytest.raises(ValueError):
        g(x, seeds=seeds, noise=torch.from_numpy(planes_or))
    with pytest.raises(ValueError):
        g(x, seeds=[-1, 0, 1])
    with pytest.raises(ValueError):
        g(x, seeds=torch.tensor([1.0, 2.0, 3.0]))


def test_seed_checks_without_a_device(lib):
    g16 = comodgan.Generator(comodgan.Mapping(num_ws=6), comodgan.Encoder(resolution=16), comodgan.Synthesis(resolution=16))
    x = torch.zeros(2, 4, 16, 16)
    with pytest.raises(ValueError):
        g16(x, seeds=[1, 2], noise_mode="const")
    with pytest.raises(ValueError):
        comodgan.load(g16, 32)                                          # resolution mismatch
    assert comodgan.load(g16, 16) is g16 and not g16.training
    g = comodgan.load(C.make_state_dict(16, seed=2), 16)
    assert g.num_ws == C.num_ws(16) and not g.training
    assert torch.equal(g.synthesis.b16.torgb.bias, C.make_state_dict(16, seed=2)["synthesis.b16.torgb.bias"])
    with pytest.raises(RuntimeError):                                   # a pipeline of another resolution
        load_generator(torch.nn.Module(), g16, 32, "cuda", accept_comodgan=True)
    # seeds with a MI-GAN generator are refused; MI-GAN runs the pass whole
    import migan_b200
    noise = NoiseSeeds(migan_b200.Generator(resolution=256), 0, 16)
    assert not noise.comodgan and noise.take("EvalPipeline", 3, None) is None
    with pytest.raises(ValueError):
        noise.take("EvalPipeline", 3, [1, 2, 3])
    # Co-Mod-GAN: the counter, explicit seeds, their count
    noise = NoiseSeeds(g16, 5, 4)
    assert list(noise.take("DemoPipeline", 3, None)) == [(5 << 32) + k for k in range(3)]
    assert list(noise.take("DemoPipeline", 2, None)) == [(5 << 32) + 3, (5 << 32) + 4] and noise.noise_index == 5
    assert list(noise.take("DemoPipeline", 2, [9, 10])) == [9, 10] and noise.noise_index == 5
    with pytest.raises(ValueError):
        noise.take("DemoPipeline", 3, [9, 10])
    with pytest.raises(ValueError):
        NoiseSeeds(g16, 2 ** 32, 4)
    with pytest.raises(ValueError):
        NoiseSeeds(g16, 0, 0)
