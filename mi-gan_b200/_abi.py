"""ctypes binding of include/migan_b200.h.  Fails loudly when the library is missing:
there is no Python/CPU fallback for the compute path."""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int64, c_size_t, c_void_p

import torch

from . import build as _build

OK, ERR_INVALID, ERR_CUDA, ERR_STATE, ERR_WORKSPACE = 0, 1, 2, 3, 4
PATH_SIMT, PATH_TC, PATH_TC_FAST = 0, 1, 2
PATHS = {"simt": PATH_SIMT, "tc": PATH_TC, "tc_fast": PATH_TC_FAST}
PIPE_MAX_BATCH = 32


class PipeRequest(ctypes.Structure):
    """migan_pipe_request: one request of the batched crop-pipeline entry points."""
    _fields_ = [("image", c_void_p), ("mask", c_void_p), ("H", c_int), ("W", c_int), ("box", c_int * 4)]


class DemoRequest(ctypes.Structure):
    """migan_demo_request: one request of the demo request path (b200_demo_*)."""
    _fields_ = [("img", c_void_p), ("H", c_int), ("W", c_int), ("mask", c_void_p), ("Hm", c_int), ("Wm", c_int),
                ("mask_channels", c_int), ("invert", c_int), ("out", c_void_p), ("out_w", c_int), ("out_h", c_int)]


class FullResRequest(ctypes.Structure):
    """migan_fullres_request: one request of the full-resolution request path (b200_fullres_*)."""
    _fields_ = [("img", c_void_p), ("mask", c_void_p), ("H", c_int), ("W", c_int), ("mask_channels", c_int),
                ("invert", c_int), ("x", c_void_p), ("y", c_void_p), ("Hp", c_int), ("Wp", c_int), ("out", c_void_p)]


class CellsRequest(ctypes.Structure):
    """migan_cells_request: one mask of b200_hole_cells."""
    _fields_ = [("mask", c_void_p), ("H", c_int), ("W", c_int), ("mask_channels", c_int), ("invert", c_int)]


class WindowRequest(ctypes.Structure):
    """migan_window_request: one window of the hole-window request path (b200_window_*)."""
    _fields_ = [("img", c_void_p), ("mask", c_void_p), ("H", c_int), ("W", c_int), ("mask_channels", c_int),
                ("invert", c_int), ("y0", c_int), ("x0", c_int), ("h", c_int), ("w", c_int), ("x", c_void_p),
                ("y", c_void_p), ("Hp", c_int), ("Wp", c_int), ("out", c_void_p)]


MASK_MIN_SIZE, MASK_MAX_SIZE, MASK_MAX_ATTEMPTS = 2, 4096, 65535


class NpRandom(ctypes.Structure):
    """migan_np_random: numpy's legacy RandomState state, as np.random.get_state() lists it."""
    _fields_ = [("key", ctypes.c_uint32 * 624), ("pos", c_int), ("has_gauss", c_int), ("gauss", ctypes.c_double)]


class MaskRecord(ctypes.Structure):
    """migan_mask_record: the primitives of one RandomMask attempt."""
    _fields_ = [("n_rects", c_int), ("n_segments", c_int), ("n_discs", c_int), ("flips", c_int),
                ("rects", (ctypes.c_int16 * 4) * 13), ("quads", (ctypes.c_int16 * 8) * 323),
                ("discs", (ctypes.c_int16 * 4) * 342)]


class SepconvTcIO(ctypes.Structure):
    """migan_sepconv_tc_io: the operands of one tensor-core SeparableConv2d launch (test hook)."""
    _fields_ = [("source", c_int), ("n", c_int), ("h", c_int), ("w", c_int), ("cin", c_int), ("cout", c_int),
                ("act", c_int), ("passes", c_int), ("in_", c_void_p), ("up_t", c_void_p), ("up_noise", c_void_p),
                ("up_fir", c_void_p), ("x", c_void_p), ("fromrgb_w", c_void_p), ("fromrgb_b", c_void_p),
                ("a_hi", c_void_p), ("a_lo", c_void_p), ("dw_w", c_void_p), ("dw_b", c_void_p), ("pw_w", c_void_p),
                ("noise", c_void_p), ("noise_pitch", c_int), ("torgb", c_int), ("rgb_w", c_void_p), ("rgb_b", c_void_p),
                ("rgb_fir", c_void_p), ("img_lo", c_void_p), ("img_out", c_void_p), ("store_out", c_int),
                ("out", c_void_p)]


class SepconvTcPlan(ctypes.Structure):
    """migan_sepconv_tc_plan: what the planner chose for one launch."""
    _fields_ = [(name, c_int) for name in ("n_group", "in_stages", "a_stages", "b_stages", "b_resident", "dw_global",
                                           "tile_w", "tile_h", "tile_n", "n_tile", "grid", "num_tiles",
                                           "num_candidates", "ep_stages", "ep_offset", "ep_stage_bytes",
                                           "smem_bytes")]

    # Where the epilogue window ring went: it depends on the launch's noise and image pointers, not only on its shapes.
    RING_FIELDS = ("ep_stages", "ep_offset", "ep_stage_bytes", "smem_bytes")

    def as_dict(self):
        """The schedule: a function of the shapes, the source and torgb alone."""
        return {name: getattr(self, name) for name, _ in self._fields_ if name not in self.RING_FIELDS}

    def ring(self):
        return {name: getattr(self, name) for name in self.RING_FIELDS}


STAGE_STEM, STAGE_DW, STAGE_DOWN, STAGE_UP2, STAGE_TORGB, STAGE_NOISE_TILE, STAGE_ADD = range(7)
DOWN_AUTO, DOWN_F32, DOWN_SPLIT, DOWN_TMA = -1, 0, 1, 2


class StageIO(ctypes.Structure):
    """migan_stage_io: the operands of one stage-kernel launch (test hook)."""
    _fields_ = [("kind", c_int), ("n", c_int), ("h", c_int), ("w", c_int), ("c", c_int), ("tc", c_int), ("level", c_int),
                ("r", c_int), ("noise_pitch", c_int), ("in_", c_void_p), ("dw_w", c_void_p), ("dw_b", c_void_p),
                ("fir", c_void_p), ("fromrgb_w", c_void_p), ("fromrgb_b", c_void_p), ("rgb_w", c_void_p),
                ("rgb_b", c_void_p), ("img_lo", c_void_p), ("noise", c_void_p), ("skip", c_void_p), ("out", c_void_p),
                ("out_hi", c_void_p), ("out_lo", c_void_p)]


class StagePlan(ctypes.Structure):
    """migan_stage_plan: what one stage launch ran."""
    _fields_ = [(name, c_int) for name in ("kind", "down_form", "rs", "cg", "grid", "groups", "fir_shift")]

    def as_dict(self):
        return {name: getattr(self, name) for name, _ in self._fields_}


# Every symbol include/migan_b200.h declares: (name, restype, argtypes)
SYMBOLS = [
    ("migan_last_error", c_char_p, []),
    ("migan_version", c_char_p, []),
    ("migan_create", c_int, [c_int, c_int, POINTER(c_void_p)]),
    ("migan_destroy", c_int, [c_void_p]),
    ("migan_num_weights", c_int, [c_void_p]),
    ("migan_weight_info", c_int, [c_void_p, c_int, POINTER(c_char_p), POINTER(c_int), POINTER(c_int64)]),
    ("migan_set_weight", c_int, [c_void_p, c_char_p, c_void_p, c_int64]),
    ("migan_finalize_weights", c_int, [c_void_p]),
    ("migan_workspace_bytes", c_size_t, [c_void_p, c_int]),
    ("migan_forward", c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_int, c_void_p]),
    ("migan_workspace_bytes_hw", c_size_t, [c_void_p, c_int, c_int, c_int]),
    ("migan_forward_hw", c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_size_t, c_int, c_void_p]),
    ("migan_graph_staging_bytes", c_size_t, [c_void_p, c_int]),
    ("migan_forward_graph", c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_int, c_void_p]),
    ("migan_host_staging_bytes", c_size_t, [c_void_p, c_int]),
    ("migan_forward_host", c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_int, c_void_p]),
    ("migan_forward_host_async", c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_int, c_void_p]),
    ("migan_host_wait", c_int, [c_void_p]),
    ("migan_u8_staging_bytes", c_size_t, [c_void_p, c_int]),
    ("migan_forward_u8", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_int, c_void_p]),
    ("migan_forward_u8_async", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_int, c_void_p]),
    ("b200_preprocess_u8", c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    ("b200_postprocess_u8", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    ("b200_preprocess_u8_hw", c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    ("b200_postprocess_u8_hw", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    ("b200_feather_composite", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    ("b200_pipeline_scratch_bytes", c_size_t, [c_int, c_int, c_int]),
    ("b200_resize_nearest_u8", c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    ("b200_hole_flags", c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    ("migan_crop_box", c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    ("b200_pipeline_preprocess", c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("b200_pipeline_postprocess", c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("b200_hole_flags_batch", c_int, [POINTER(PipeRequest), c_int, c_void_p, c_void_p]),
    ("b200_pipeline_batch_scratch_bytes", c_size_t, [POINTER(PipeRequest), c_int, c_int]),
    ("b200_pipeline_preprocess_batch", c_int, [POINTER(PipeRequest), c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("b200_pipeline_postprocess_batch", c_int, [c_void_p, POINTER(PipeRequest), c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("b200_pipeline_batch_scratch_bound", c_size_t, [POINTER(PipeRequest), c_int, c_int]),
    ("b200_pipeline_plan_batch", c_int, [POINTER(PipeRequest), c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("b200_pipeline_preprocess_planned", c_int, [POINTER(PipeRequest), c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("b200_pipeline_postprocess_planned", c_int, [c_void_p, POINTER(PipeRequest), c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("migan_demo_resized_size", c_int, [c_int, c_int, c_int, POINTER(c_int), POINTER(c_int)]),
    ("b200_demo_scratch_bytes", c_size_t, [POINTER(DemoRequest), c_int, c_int]),
    ("b200_demo_preprocess", c_int, [POINTER(DemoRequest), c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("b200_demo_postprocess", c_int, [c_void_p, POINTER(DemoRequest), c_int, c_int, c_void_p, c_size_t, c_void_p]),
    ("b200_eval_scratch_bytes", c_size_t, [POINTER(DemoRequest), c_int, c_int]),
    ("b200_eval_preprocess", c_int, [POINTER(DemoRequest), c_int, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("b200_eval_composite", c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    ("migan_fullres_extent", c_int, [c_void_p, c_int, c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    ("b200_fullres_preprocess", c_int, [POINTER(FullResRequest), c_int, c_void_p]),
    ("b200_fullres_postprocess", c_int, [POINTER(FullResRequest), c_int, c_void_p]),
    ("b200_hole_cells_bytes", c_size_t, [POINTER(CellsRequest), c_int, c_int]),
    ("b200_hole_cells", c_int, [POINTER(CellsRequest), c_int, c_int, c_void_p, c_void_p]),
    ("migan_hole_windows", c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(c_int), c_int, POINTER(c_int)]),
    ("migan_hole_windows_max", c_int, [c_int, c_int, c_int, POINTER(c_int)]),
    ("b200_window_preprocess", c_int, [POINTER(WindowRequest), c_int, c_void_p]),
    ("b200_window_postprocess", c_int, [POINTER(WindowRequest), c_int, c_void_p]),
    ("migan_np_seed", c_int, [POINTER(NpRandom), ctypes.c_uint32]),
    ("migan_mask_plan", c_int, [POINTER(NpRandom), c_int, c_int, c_void_p, c_void_p]),
    ("b200_mask_raster", c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    ("b200_mask_compact", c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    ("b200_reparam_filter", c_int, [c_void_p, c_int, c_int, c_int64, c_void_p, c_void_p]),
    ("b200_stream_memops_available", c_int, []),
    ("b200_stream_wait_value32", c_int, [c_void_p, c_void_p, ctypes.c_uint32]),
    ("b200_stream_write_value32", c_int, [c_void_p, c_void_p, ctypes.c_uint32]),
    ("b200_memcpy_async", c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    ("b200_enable_peer_access", c_int, [c_int]),
    ("migan_last_launch_count", c_int, [c_void_p]),
    ("migan_set_profiling", c_int, [c_void_p, c_int]),
    ("migan_profile_num_steps", c_int, [c_void_p]),
    ("migan_profile_step", c_int, [c_void_p, c_int, POINTER(c_char_p), POINTER(c_float), POINTER(ctypes.c_double), POINTER(ctypes.c_double)]),
    ("migan_set_tap", c_int, [c_void_p, c_char_p, c_void_p]),
    ("migan_tap_info", c_int, [c_void_p, c_int, c_int, POINTER(c_char_p), POINTER(c_int)]),
    ("migan_debug_tc_timeout", c_int, [c_int]),
    ("migan_debug_sepconv_tc", c_int, [POINTER(SepconvTcIO), c_int, c_int, POINTER(SepconvTcPlan), c_void_p]),
    ("migan_debug_stage", c_int, [POINTER(StageIO), c_int, POINTER(StagePlan), c_void_p]),
    ("b200_upfirdn2d", c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 14 + [c_int, c_float, c_void_p]),
    ("b200_conv1x1_nhwc", c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p]),
    ("b200_bias_act", c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_float, c_float, c_float, c_void_p]),
]

# Every symbol include/comodgan_b200.h declares
COMOD_SYMBOLS = [
    ("comodgan_last_error", c_char_p, []),
    ("comodgan_create", c_int, [c_int, c_int, POINTER(c_void_p)]),
    ("comodgan_destroy", c_int, [c_void_p]),
    ("comodgan_num_weights", c_int, [c_void_p]),
    ("comodgan_weight_info", c_int, [c_void_p, c_int, POINTER(c_char_p), POINTER(c_int), POINTER(c_int64)]),
    ("comodgan_set_weight", c_int, [c_void_p, c_char_p, c_void_p, c_int64]),
    ("comodgan_finalize_weights", c_int, [c_void_p]),
    ("comodgan_workspace_bytes", c_size_t, [c_void_p, c_int]),
    ("comodgan_num_noise_planes", c_int, [c_void_p]),
    ("comodgan_noise_plane_res", c_int, [c_void_p, c_int]),
    ("comodgan_forward", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_int, c_int, c_void_p,
                                 c_void_p, c_size_t, c_void_p]),
    ("comodgan_seeded_noise", c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    ("comodgan_workspace_bytes_seeded", c_size_t, [c_void_p, c_int]),
    ("comodgan_forward_seeded", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_int,
                                        c_void_p, c_size_t, c_void_p]),
    ("comodgan_last_launch_count", c_int, [c_void_p]),
    ("comodgan_set_tap", c_int, [c_void_p, c_char_p, c_void_p]),
    ("b200_conv2d_resample", c_int, [c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 18 +
     [c_void_p, c_size_t, POINTER(c_size_t), POINTER(c_int), POINTER(c_int), c_void_p]),
]

PREPOST_SYMBOLS = [s for s in SYMBOLS if s[0] in ("b200_preprocess_u8", "b200_postprocess_u8", "b200_feather_composite",
                                                   "b200_preprocess_u8_hw", "b200_postprocess_u8_hw")]

_lib = None


def bind(lib, symbols):
    """Set restype / argtypes for `symbols` on an already dlopen-ed library (AttributeError if an export is missing)."""
    for name, restype, argtypes in symbols:
        fn = getattr(lib, name)
        fn.restype = restype
        fn.argtypes = argtypes
    return lib


_bound = set()


def library(symbols, handle=None):
    """`handle` (the product library when None) with `symbols` bound; each list is bound once per handle.  A handle can
    be another build of the same sources, such as an emulation build."""
    h = handle if handle is not None else load()
    if (id(h), id(symbols)) not in _bound:
        bind(h, symbols)
        _bound.add((id(h), id(symbols)))
    return h


class Workspace:
    """One device buffer, kept while the key of the calls that use it stays the same: a new key frees it and allocates
    nbytes() bytes."""

    def __init__(self):
        self.key, self.buf = None, None

    def get(self, key, nbytes, device) -> torch.Tensor:
        if self.buf is None or key != self.key:
            self.buf = None
            self.buf = torch.empty(int(nbytes()), dtype=torch.uint8, device=device)
            self.key = key
        return self.buf


class MiganError(RuntimeError):
    """A C-ABI call returned a non-zero code."""

    def __init__(self, code: int, message: str):
        super().__init__("migan_b200 error %d: %s" % (code, message))
        self.code = code


def library_path() -> str:
    return os.environ.get("MIGAN_B200_LIB", _build.LIBPATH)


def path_id(name) -> int:
    """Id of the kernel path `name`; None selects $MIGAN_B200_PATH, or "tc" when that is unset."""
    name = name or os.environ.get("MIGAN_B200_PATH", "tc")
    if name not in PATHS:
        raise ValueError("unknown path %r (expected one of %s)" % (name, sorted(PATHS)))
    return PATHS[name]


def load(build_if_missing: bool = False):
    """dlopen the shared library and bind every declared symbol."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        if build_if_missing:
            _build.build()
        else:
            raise ImportError(
                "migan_b200: %s not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). There is no CPU / pure-PyTorch fallback." % path)
    lib = ctypes.CDLL(path)
    bind(lib, SYMBOLS)
    bind(lib, COMOD_SYMBOLS)
    _lib = lib
    return lib


_LAST_ERROR = ctypes.CFUNCTYPE(c_char_p)


def check(rc: int, lib=None) -> None:
    """Raise MiganError for a non-zero return code of `lib` (the loaded library when None), with the calling thread's last
    error.  The message is read from the library's own migan_last_error export, whichever symbols the caller bound."""
    if rc != 0:
        msg = _LAST_ERROR(("migan_last_error", lib or load()))()
        raise MiganError(rc, msg.decode() if msg else "unknown error")


check_comod = check   # the Co-Mod-GAN callers' name: comodgan_last_error() is the same thread-local message
