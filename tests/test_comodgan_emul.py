"""CPU check of the Co-Mod-GAN / conv2d_resample host runtime + item kernels through the HOST-EMULATION build
(tests/emul/build_emul.py: same C++ source and kernel functors, ck_launch = host loop, GEMM = triple loop).

What this proves without a GPU: the state_dict registry, weight packing (gain folding, demodulation pre-normalisation,
NCHW<->NHWC permutations, transposed-conv operand), the workspace walk, chunking, and the index math of every item
kernel reproduce the oracle.  What it cannot prove: anything about the CUDA launch itself -- that is
tests/test_comodgan_gpu.py.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import comodgan_oracle as C  # noqa: E402
from oracle import migan_oracle as O  # noqa: E402
from migan_b200 import _abi  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import build_emul  # noqa: E402


@pytest.fixture(scope="module")
def emul():
    return _abi.bind(ctypes.CDLL(build_emul.build()), _abi.COMOD_SYMBOLS)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _aligned(nbytes):
    raw = np.empty(nbytes + 256, dtype=np.uint8)
    off = (-raw.ctypes.data) % 256
    return raw, raw[off:off + nbytes]


class EmulGen:
    def __init__(self, lib, resolution, sd):
        self.lib, self.R = lib, resolution
        h = ctypes.c_void_p()
        _abi.check_comod(lib.comodgan_create(resolution, 0, ctypes.byref(h)), lib)
        self.h = h
        n = lib.comodgan_num_weights(h)
        names = []
        for i in range(n):
            name, nd, shape = ctypes.c_char_p(), ctypes.c_int(), (ctypes.c_int64 * 4)()
            _abi.check_comod(lib.comodgan_weight_info(h, i, ctypes.byref(name), ctypes.byref(nd), shape), lib)
            names.append((name.value.decode(), tuple(shape[:nd.value])))
        self.names = names
        for name, shape in names:
            a = np.ascontiguousarray(sd[name].numpy(), dtype=np.float32)
            assert tuple(sd[name].shape) == shape, name
            _abi.check_comod(lib.comodgan_set_weight(h, name.encode(), _ptr(a), a.size), lib)
        _abi.check_comod(lib.comodgan_finalize_weights(h), lib)

    def __call__(self, x, z, psi=1.0, cutoff=None, noise_mode=1, noise=None, tap=None, tap_shape=None):
        lib, n = self.lib, x.shape[0]
        xa = np.ascontiguousarray(x.numpy(), np.float32)
        za = np.ascontiguousarray(z.numpy(), np.float32)
        y = np.empty((n, 3, self.R, self.R), np.float32)
        need = lib.comodgan_workspace_bytes(self.h, n)
        assert need > 0
        _raw, ws = _aligned(need)
        tap_out = None
        if tap is not None:
            tap_out = np.zeros((n,) + tuple(tap_shape), np.float32)
            _abi.check_comod(lib.comodgan_set_tap(self.h, tap.encode(), _ptr(tap_out)), lib)
        na = np.ascontiguousarray(noise, np.float32) if noise is not None else None
        _abi.check_comod(lib.comodgan_forward(self.h, _ptr(xa), _ptr(za), _ptr(y), n, psi, -1 if cutoff is None else cutoff,
                                              noise_mode, _ptr(na), _ptr(ws), need, None), lib)
        if tap is not None:
            lib.comodgan_set_tap(self.h, None, None)
            return torch.from_numpy(y), torch.from_numpy(tap_out)
        return torch.from_numpy(y)

    def close(self):
        self.lib.comodgan_destroy(self.h)


def test_state_dict_registry_matches_oracle(emul):
    for R in (16, 256):
        h = ctypes.c_void_p()
        _abi.check_comod(emul.comodgan_create(R, -1, ctypes.byref(h)), emul)
        spec = C.state_dict_spec(R)
        assert emul.comodgan_num_weights(h) == len(spec)
        for i, (k, shape) in enumerate(spec.items()):
            name, nd, sh = ctypes.c_char_p(), ctypes.c_int(), (ctypes.c_int64 * 4)()
            emul.comodgan_weight_info(h, i, ctypes.byref(name), ctypes.byref(nd), sh)
            assert name.value.decode() == k and tuple(sh[:nd.value]) == tuple(shape)
        assert emul.comodgan_num_noise_planes(h) == len(C.noise_keys(R))
        assert [emul.comodgan_noise_plane_res(h, i) for i in range(len(C.noise_keys(R)))] == [r for _, r in C.noise_keys(R)]
        emul.comodgan_destroy(h)
    h = ctypes.c_void_p()
    assert emul.comodgan_create(48, -1, ctypes.byref(h)) == 1      # ValueError in the reference
    assert b"power of two" in emul.comodgan_last_error()


@pytest.fixture(scope="module")
def gen16(emul):
    sd = C.make_state_dict(16, seed=1)
    g = EmulGen(emul, 16, sd)
    yield g, sd
    g.close()


def test_forward_r16_matches_oracle_and_reference_fixture(gen16):
    g, sd = gen16
    x, z = O.make_input(16, 2, seed=1234), C.make_latent(2, seed=1235)
    y = g(x, z)
    y_or = C.generator_forward(sd, x, z, 16)
    gold = np.load(os.path.join(ROOT, "tests", "golden", "comodgan_R16_n2_w1.npz"))
    assert float((y - y_or).abs().max()) < 2e-4
    assert float((y - torch.from_numpy(gold["y"])).abs().max()) < 2e-4   # output of the REAL reference
    y0 = g(x, z, noise_mode=0)
    assert float((y0 - torch.from_numpy(gold["y_noise_none"])).abs().max()) < 2e-4


@pytest.mark.parametrize("tap", ["mapping.w", "encoder.b16.fromrgb.out", "encoder.b16.conv0.out", "encoder.b16.conv1.out",
                                 "encoder.b4.conv.out", "encoder.b4.fc.out", "synthesis.b4.conv.out",
                                 "synthesis.b4.torgb.out", "synthesis.b8.conv0.out", "synthesis.b8.conv1.out",
                                 "synthesis.b8.img", "synthesis.b16.torgb.out"])
def test_intermediates_r16(gen16, tap):
    g, sd = gen16
    x, z = O.make_input(16, 2, seed=5), C.make_latent(2, seed=6)
    taps = {}
    C.generator_forward(sd, x, z, 16, taps=taps)
    if tap == "mapping.w":
        want = taps["mapping.ws"][:, 0].reshape(2, 512, 1, 1)
    elif tap == "encoder.b4.fc.out":
        want = taps[tap].reshape(2, 1024, 1, 1)
    elif tap == "synthesis.b8.conv0.out":    # the kernel epilogue also adds the encoder feature (comodgan.py:324)
        want = taps[tap] + taps["encoder.b8.conv0.out"]
    else:
        want = taps[tap]
    _, got = g(x, z, tap=tap, tap_shape=tuple(want.shape[1:]))
    scale = max(1.0, float(want.abs().max()))
    assert float((got - want).abs().max()) < 1e-4 * scale, tap


def test_truncation_and_random_noise_r16(gen16):
    g, sd = gen16
    x, z = O.make_input(16, 3, seed=8), C.make_latent(3, seed=9)
    for psi, cutoff in ((0.6, None), (0.7, 3)):
        y = g(x, z, psi=psi, cutoff=cutoff)
        y_or = C.generator_forward(sd, x, z, 16, truncation_psi=psi, truncation_cutoff=cutoff)
        assert float((y - y_or).abs().max()) < 2e-4
    gen = torch.Generator().manual_seed(3)
    planes, noise = [], {}
    for key, r in C.noise_keys(16):
        p = torch.randn(3, 1, r, r, generator=gen)
        noise[key] = p
        planes.append(p.reshape(-1))
    y = g(x, z, noise_mode=2, noise=torch.cat(planes).numpy())
    y_or = C.generator_forward(sd, x, z, 16, noise_mode="random", noise=noise)
    assert float((y - y_or).abs().max()) < 2e-4


def test_chunked_convolutions_r32(emul, monkeypatch):
    """Force one-image chunks (COMOD_COL_CAP_MB=1) so the chunk loop and its pointer offsets are exercised."""
    monkeypatch.setenv("COMOD_COL_CAP_MB", "1")
    sd = C.make_state_dict(32, seed=3)
    g = EmulGen(emul, 32, sd)
    x, z = O.make_input(32, 2, seed=77), C.make_latent(2, seed=78)
    y = g(x, z, psi=0.7, cutoff=4)
    gold = np.load(os.path.join(ROOT, "tests", "golden", "comodgan_R32_n2_w3.npz"))
    assert float((y - torch.from_numpy(gold["y"])).abs().max()) < 3e-4
    g.close()


def test_errors(emul, gen16):
    g, _ = gen16
    lib = emul
    x = np.zeros((1, 4, 16, 16), np.float32)
    z = np.zeros((1, 512), np.float32)
    y = np.zeros((1, 3, 16, 16), np.float32)
    _raw, ws = _aligned(1024)
    assert lib.comodgan_forward(g.h, _ptr(x), _ptr(z), _ptr(y), 1, 1.0, -1, 1, None, _ptr(ws), 1024, None) == 4
    assert b"workspace too small" in lib.comodgan_last_error()
    assert lib.comodgan_forward(g.h, _ptr(x), _ptr(z), _ptr(y), 1, 1.0, -1, 2, None, _ptr(ws), 1024, None) == 1
    h = ctypes.c_void_p()
    lib.comodgan_create(16, 0, ctypes.byref(h))
    a = np.zeros(7, np.float32)
    assert lib.comodgan_set_weight(h, b"mapping.w_avg", _ptr(a), 7) == 1
    assert lib.comodgan_set_weight(h, b"nope", _ptr(a), 7) == 1
    assert lib.comodgan_finalize_weights(h) == 1 and b"missing key" in lib.comodgan_last_error()
    assert lib.comodgan_forward(h, _ptr(x), _ptr(z), _ptr(y), 1, 1.0, -1, 1, None, _ptr(ws), 1024, None) == 3
    lib.comodgan_destroy(h)


# ---- conv2d_resample: every branch against the vectors the real reference produced -----------------------------------
def _conv2d_resample(lib, x, w, f, up, down, padding, groups, flip_weight, flip_filter=False):
    n, cin, h, wd = x.shape
    cout, _, kh, kw = w.shape
    fh, fw = (f.shape if f is not None else (0, 0))
    need, oh, ow = ctypes.c_size_t(), ctypes.c_int(), ctypes.c_int()
    args = [n, cin, h, wd, cout, kh, kw, fh, fw, up, down] + list(padding) + [groups, int(flip_weight), int(flip_filter)]
    _abi.check_comod(lib.b200_conv2d_resample(None, None, None, None, *args, None, 0, ctypes.byref(need), ctypes.byref(oh),
                                              ctypes.byref(ow), None), lib)
    y = np.empty((n, cout, oh.value, ow.value), np.float32)
    _raw, ws = _aligned(need.value)
    _abi.check_comod(lib.b200_conv2d_resample(_ptr(x), _ptr(w), _ptr(f), _ptr(y), *args, _ptr(ws), need.value, None, None,
                                              None, None), lib)
    return y


def test_conv2d_resample_all_branches(emul):
    from test_oracle import _c2r_cases, _c2r_stored_rows
    g = np.load(os.path.join(ROOT, "tests", "golden", "conv2d_resample.npz"))
    cases = list(_c2r_cases(g))
    assert len(cases) == 15
    for name, x, w, f, kw in cases:
        y = _conv2d_resample(emul, np.ascontiguousarray(x.numpy()), np.ascontiguousarray(w.numpy()),
                             None if f is None else np.ascontiguousarray(f.numpy()), kw["up"], kw["down"], kw["padding"],
                             kw["groups"], kw["flip_weight"], kw["flip_filter"])
        y = _c2r_stored_rows(g, name, y)
        assert float(np.abs(y - g[name + ".y"]).max()) < 1e-4, name


def test_conv2d_resample_odd_channels_and_filters(emul):
    """Channel counts that are not multiples of 4 (scalar im2col), f=None, flip_filter, asymmetric filter."""
    gen = torch.Generator().manual_seed(2)
    fa = torch.tensor([[1., 2., 0.5], [0.25, 3., 1.], [2., 1., 0.125]]) / 10.875
    for (cin, cout, k, up, down, pad, groups, flipw, f, flipf) in [
        (3, 5, 3, 1, 1, 1, 1, True, None, False), (6, 10, 3, 2, 1, 1, 2, False, fa, False),
        (3, 7, 1, 1, 2, 0, 1, True, fa, True), (5, 3, 3, 1, 2, 1, 1, False, fa, False),
        (3, 6, 3, 1, 1, [1, 0, 2, 0], 3, True, None, False),
    ]:
        x = torch.randn(2, cin, 9, 7, generator=gen)
        w = torch.randn(cout, cin // groups, k, k, generator=gen)
        want = C.conv2d_resample_ref(x, w, f=f, up=up, down=down, padding=pad, groups=groups, flip_weight=flipw,
                                     flip_filter=flipf)
        padl = pad if isinstance(pad, list) else [pad] * 4
        got = _conv2d_resample(emul, x.numpy(), w.numpy(), None if f is None else np.ascontiguousarray(f.numpy()), up, down,
                               padl, groups, flipw, flipf)
        assert got.shape == tuple(want.shape)
        assert float((torch.from_numpy(got) - want).abs().max()) < 1e-4


# ---- the Python mirror's ctypes plumbing, driven against the emulation library ---------------------------------------
@pytest.fixture()
def emul_python(emul, monkeypatch):
    """Route migan_b200.comodgan / ops.conv2d_resample to the emulation library with CPU tensors standing in for device
    memory.  Only the device/stream seams are patched; argument marshalling is the product code."""
    import contextlib
    from migan_b200 import comodgan, ops
    monkeypatch.setattr(_abi, "load", lambda build_if_missing=False: emul)
    for mod in (comodgan, ops):
        monkeypatch.setattr(mod, "_guard", lambda device: contextlib.nullcontext())
    monkeypatch.setattr(comodgan, "_stream", lambda device: None)
    monkeypatch.setattr(comodgan, "_device_index", lambda device: 0)
    monkeypatch.setattr(ops, "_stream", lambda t: None)
    monkeypatch.setattr(ops, "_require_cuda_f32", lambda x, what: x.contiguous())

    class EmulGenerator(comodgan.Generator):
        def _validate(self, x, z):
            if z is None:
                z = torch.randn([x.shape[0], 512])
            return x.contiguous(), z.contiguous()

    return comodgan, ops, EmulGenerator


def test_python_mirror_marshalling(emul_python):
    comodgan, _, EmulGenerator = emul_python
    sd = C.make_state_dict(16, seed=1)
    g = EmulGenerator(comodgan.Mapping(num_ws=6), comodgan.Encoder(resolution=16), comodgan.Synthesis(resolution=16))
    g.load_state_dict(sd, strict=True)
    x, z = O.make_input(16, 2, seed=1234), C.make_latent(2, seed=1235)
    y = g(x, z=z, noise_mode="const")
    assert float((y - C.generator_forward(sd, x, z, 16)).abs().max()) < 2e-4
    y = g(x, z=z, truncation_psi=0.7, truncation_cutoff=3, noise_mode="none")
    assert float((y - C.generator_forward(sd, x, z, 16, truncation_psi=0.7, truncation_cutoff=3, noise_mode="none")).abs().max()) < 2e-4
    gen = torch.Generator().manual_seed(3)
    planes, noise = [], {}
    for (key, r), shape in zip(C.noise_keys(16), g.noise_plane_shapes(2)):
        assert shape == (2, r, r)
        noise[key] = torch.randn(2, 1, r, r, generator=gen)
        planes.append(noise[key].reshape(-1))
    y = g(x, z=z, noise_mode="random", noise=torch.cat(planes))
    assert float((y - C.generator_forward(sd, x, z, 16, noise_mode="random", noise=noise)).abs().max()) < 2e-4
    assert torch.isfinite(g(x)).all()                                  # z and noise drawn by the module
    y, t = g(x, z=z, noise_mode="const", _tap=("synthesis.b8.img", (3, 8, 8)))
    taps = {}
    C.generator_forward(sd, x, z, 16, taps=taps)
    assert float((t - taps["synthesis.b8.img"]).abs().max()) < 2e-4
    # weights edited in place -> re-upload on the next call
    with torch.no_grad():
        g.synthesis.b16.torgb.bias.add_(1.0)
    sd2 = {k: v.clone() for k, v in g.state_dict().items()}
    assert float((g(x, z=z, noise_mode="const") - C.generator_forward(sd2, x, z, 16)).abs().max()) < 2e-4
    with pytest.raises(NotImplementedError):
        g(x, z=z, return_intermediate_outs=True)
    with pytest.raises(AssertionError):
        g(x, z=z, noise_mode="bogus")
    assert g.last_launch_count() > 50


def test_python_conv2d_resample_marshalling(emul_python):
    _, ops, _ = emul_python
    gen = torch.Generator().manual_seed(4)
    f1 = torch.tensor([1., 3., 3., 1.]) / 8
    f2 = O.setup_filter([1, 3, 3, 1])
    for (cin, cout, k, up, down, pad, groups, flipw, f) in [
        (8, 12, 3, 2, 1, 1, 2, False, f2), (8, 12, 3, 1, 2, 1, 1, True, f1), (3, 5, 3, 1, 1, [2, 0, 1, 0], 1, True, None),
        (6, 4, 1, 2, 2, 0, 1, True, f2),
    ]:
        x = torch.randn(2, cin, 6, 10, generator=gen)
        w = torch.randn(cout, cin // groups, k, k, generator=gen)
        want = C.conv2d_resample_ref(x, w, f=f, up=up, down=down, padding=pad, groups=groups, flip_weight=flipw)
        got = ops.conv2d_resample(x, w, f, up=up, down=down, padding=pad, groups=groups, flip_weight=flipw)
        assert tuple(got.shape) == tuple(want.shape)
        assert float((got - want).abs().max()) < 1e-4


# ---- uint8 pre/post-processing kernels (prepost.cu) in the same emulation library ------------------------------------
def test_prepost_u8_kernels_bit_exact(emul):
    from oracle import prepost_oracle as P
    lib = _abi.bind(emul, _abi.PREPOST_SYMBOLS)
    gold = np.load(os.path.join(ROOT, "tests", "golden", "prepost.npz"))
    img, mask, y = np.ascontiguousarray(gold["img"]), np.ascontiguousarray(gold["mask"]), np.ascontiguousarray(gold["y"])
    n, r = img.shape[0], img.shape[1]
    x = np.empty((n, 4, r, r), np.float32)
    assert lib.b200_preprocess_u8(_ptr(img), _ptr(mask), _ptr(x), n, r, None) == 0
    assert np.array_equal(x, gold["x"]) and np.array_equal(x, P.preprocess(img, mask).numpy())
    out = np.empty((n, r, r, 3), np.uint8)
    assert lib.b200_postprocess_u8(_ptr(y), _ptr(img), _ptr(mask), _ptr(out), n, r, None) == 0
    assert np.array_equal(out, gold["out"]) and np.array_equal(out, P.postprocess(torch.from_numpy(y), img, mask))
    # mask values other than 255 are holes (`// 255`), every uint8 image value
    rng = np.random.RandomState(0)
    img = np.ascontiguousarray(np.tile(np.arange(256, dtype=np.uint8)[None, :, None, None], (1, 1, 256, 3)))
    mask = np.ascontiguousarray(rng.choice(np.array([0, 1, 128, 254, 255], np.uint8), size=(1, 256, 256)))
    x = np.empty((1, 4, 256, 256), np.float32)
    lib.b200_preprocess_u8(_ptr(img), _ptr(mask), _ptr(x), 1, 256, None)
    assert np.array_equal(x, P.preprocess(img, mask).numpy())
    y = (torch.linspace(-1.2, 1.2, 256 * 256 * 3).reshape(1, 3, 256, 256)).contiguous()
    out = np.empty((1, 256, 256, 3), np.uint8)
    lib.b200_postprocess_u8(_ptr(y.numpy()), _ptr(img), _ptr(mask), _ptr(out), 1, 256, None)
    assert np.array_equal(out, P.postprocess(y, img, mask))


def test_staged_tcgen05_route_operands(emul, monkeypatch):
    """COMOD_GEMM=tc (off by default): plain / strided / 1x1 convolutions feed the wgmma GEMM of the
    MI-GAN path (sepconv_tc.cu, A_TMA mode) with an fp16 hi/lo split im2col and K-major hi/lo weights.  The emulation
    replaces only that GEMM by its arithmetic (Ah*Bh + Ah*Bl + Al*Bh, fp32 accumulate); the operand packing, scales,
    K/N padding and chunking around it are the product code.  tests/test_staged_gpu.py runs the route on the GPU."""
    monkeypatch.setenv("COMOD_GEMM", "tc")
    monkeypatch.setenv("COMOD_COL_CAP_MB", "2")
    sd = C.make_state_dict(16, seed=1)
    g = EmulGen(emul, 16, sd)
    x, z = O.make_input(16, 2, seed=1234), C.make_latent(2, seed=1235)
    y = g(x, z, psi=0.8, cutoff=2)
    y_or = C.generator_forward(sd, x, z, 16, truncation_psi=0.8, truncation_cutoff=2)
    err = float((y - y_or).abs().max())
    assert err < 1e-3, err
    g.close()


def test_conv2d_resample_randomized_sweep(emul):
    """200 random small configurations -- non-square kernels and filters, f=None with up/down > 1 (negative padding
    adjustments: Python floor division), up/down in {1,2,3}, asymmetric padding, groups, both flips -- through the
    emulated kernels against the oracle restatement of conv2d_resample.py:59-154."""
    rng = np.random.RandomState(0)
    gen = torch.Generator().manual_seed(0)
    checked = 0
    for _ in range(200):
        groups = int(rng.choice([1, 1, 2, 3]))
        cin, cout = groups * int(rng.choice([1, 2, 4, 5, 8])), groups * int(rng.choice([1, 2, 3, 4, 16]))
        kh = int(rng.choice([1, 2, 3, 4]))
        kw = int(rng.choice([1, 2, 3, 4])) if rng.rand() < 0.3 else kh
        up, down = int(rng.choice([1, 1, 2, 3])), int(rng.choice([1, 1, 2, 3]))
        f = [None, O.setup_filter([1, 3, 3, 1]), torch.tensor([1., 2., 1.]) / 4, torch.rand(3, 5, generator=gen)][rng.randint(0, 4)]
        pad = [int(v) for v in rng.randint(0, 3, size=4)] if rng.rand() < 0.5 else int(rng.randint(0, 3))
        flipw, flipf = bool(rng.randint(0, 2)), bool(rng.randint(0, 2))
        h, w, n = int(rng.randint(4, 9)), int(rng.randint(4, 9)), int(rng.randint(1, 3))
        x = torch.randn(n, cin, h, w, generator=gen)
        wt = torch.randn(cout, cin // groups, kh, kw, generator=gen)
        try:
            want = C.conv2d_resample_ref(x, wt, f=f, up=up, down=down, padding=pad, groups=groups, flip_weight=flipw, flip_filter=flipf)
        except RuntimeError:
            continue                      # shapes torch itself rejects (kernel larger than the padded input)
        if want.numel() == 0:
            continue
        f2 = None if f is None else np.ascontiguousarray((torch.outer(f, f) if f.ndim == 1 else f).numpy())
        got = _conv2d_resample(emul, x.numpy(), wt.numpy(), f2, up, down, pad if isinstance(pad, list) else [pad] * 4, groups,
                               flipw, flipf)
        cfg = (cin, cout, kh, kw, up, down, pad, groups, flipw, flipf, None if f is None else tuple(f.shape), h, w)
        assert got.shape == tuple(want.shape), cfg
        assert float(np.abs(got - want.numpy()).max()) <= 1e-5 * max(1.0, float(want.abs().max())), cfg
        checked += 1
    assert checked > 150


def test_feather_composite_matches_reference_pipeline(emul):
    """The feathered blend of the deployed pipeline (create_onnx_pipeline.py:233-245): kernel source compiled for the host
    against (a) the outputs of the reference's own MIGAN_Pipeline.postprocess (tests/golden/feather.npz, written by
    make_golden_prepost.py in the build container) and (b) the oracle on fresh inputs, including free-form masks."""
    from migan_b200 import ops, synthetic
    from oracle import prepost_oracle as P
    lib = _abi.bind(emul, _abi.PREPOST_SYMBOLS)
    k = np.ascontiguousarray(ops.feather_kernel().numpy())
    assert np.array_equal(k, P.gaussian_kernel_5x5().numpy())
    gold = np.load(os.path.join(ROOT, "tests", "golden", "feather.npz"))
    for tag in ("a", "b"):
        image, mask, y = (np.ascontiguousarray(gold[n + "_" + tag]) for n in ("image", "mask", "y"))
        n, _, H, W = image.shape
        out = np.empty_like(image)
        assert lib.b200_feather_composite(_ptr(y), _ptr(image), _ptr(mask), _ptr(out), n, H, W, _ptr(k), None) == 0
        diff = np.abs(out.astype(np.int32) - gold["out_" + tag].astype(np.int32))
        assert diff.max() <= 1 and (diff > 0).mean() < 1e-3, (tag, int(diff.max()), float((diff > 0).mean()))
        known = np.broadcast_to(mask == 255, image.shape)
        # deep inside the known region the weight is exactly 1: the image must come back unchanged
    rng = np.random.RandomState(5)
    H = W = 96
    image = np.ascontiguousarray(rng.randint(0, 256, size=(2, 3, H, W), dtype=np.uint8))
    mask = np.stack([synthetic.free_form_mask(H, rng) for _ in range(2)])[:, None] * np.uint8(255)
    mask = np.ascontiguousarray(mask.astype(np.uint8))
    y = np.ascontiguousarray((rng.randn(2, 3, H, W) * 0.7).astype(np.float32))
    out = np.empty_like(image)
    assert lib.b200_feather_composite(_ptr(y), _ptr(image), _ptr(mask), _ptr(out), 2, H, W, _ptr(k), None) == 0
    want = P.feather_composite(torch.from_numpy(image), torch.from_numpy(mask), torch.from_numpy(y)).numpy()
    diff = np.abs(out.astype(np.int32) - want.astype(np.int32))
    assert diff.max() <= 1 and (diff > 0).mean() < 1e-3, (int(diff.max()), float((diff > 0).mean()))
    allk = np.full((1, 1, 32, 32), 255, np.uint8)
    img1 = np.ascontiguousarray(image[:1, :, :32, :32])
    out1 = np.empty_like(img1)
    lib.b200_feather_composite(_ptr(np.ascontiguousarray(y[:1, :, :32, :32])), _ptr(img1), _ptr(allk), _ptr(out1), 1, 32, 32, _ptr(k), None)
    assert np.array_equal(out1, img1)                       # fully known: weight exactly 1 everywhere
