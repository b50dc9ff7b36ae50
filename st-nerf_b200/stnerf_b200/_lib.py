"""ctypes binding of libstnerf_b200.so (the C ABI declared in include/stnerf.h).

There is no CPU fallback: if the shared library is missing or a call fails, this module raises.
"""
from __future__ import annotations

import ctypes as C
import os

MAX_LAYERS = 8
MAX_N1 = 128
MAX_S = 512

# stnerf_set_rotation modes: no rotation, about an explicit centre, about the centre of the layer's box in each call's scene
ROT_OFF, ROT_CENTRE, ROT_BOX = 0, 1, 2

# stnerf_td_select modes: keep label == layer, keep a box's projected rectangle
TD_BY_LABEL, TD_BY_RECT = 0, 1

PREC_FP32_SIMT, PREC_TC_3XF16, PREC_TC_F16, PREC_TC_MIXED, PREC_TC_3XF16_CF = 0, 1, 2, 3, 4
PRECISIONS = {"fp32": PREC_FP32_SIMT, "exact": PREC_TC_3XF16, "tc3": PREC_TC_3XF16, "fast": PREC_TC_F16, "mixed": PREC_TC_MIXED,
              "exact_cf": PREC_TC_3XF16_CF}
# training precision of the differentiable networks (STNERF_TRAIN_*): cfg.MODEL.B200_TRAIN_PRECISION / train_precision=
TRAIN_FP32, TRAIN_TC_3XTF32 = 0, 1
TRAIN_PRECISIONS = {"fp32": TRAIN_FP32, "tf32x3": TRAIN_TC_3XTF32}


def train_precision_code(name: str) -> int:
    """STNERF_TRAIN_* value of a training precision name; unknown names raise ValueError."""
    if name not in TRAIN_PRECISIONS:
        raise ValueError("unknown training precision %r (one of %s)" % (name, ", ".join(sorted(TRAIN_PRECISIONS))))
    return TRAIN_PRECISIONS[name]

# STNERF_B200_LIB selects another build of the same ABI (e.g. to compare two builds with scripts/dump_networks.py)
LIB_PATH = os.environ.get("STNERF_B200_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "libstnerf_b200.so")


class ModelDesc(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("space_time", C.c_int32 * MAX_LAYERS), ("precision", C.c_int32),
                ("chunk_rays", C.c_int32)]


class Scene(C.Structure):
    _fields_ = [("bmin", (C.c_float * 3) * MAX_LAYERS), ("bmax", (C.c_float * 3) * MAX_LAYERS),
                ("shown", C.c_int32 * MAX_LAYERS),
                ("shift_on", C.c_int32 * MAX_LAYERS), ("shift", (C.c_float * 3) * MAX_LAYERS),
                ("scale_coarse_on", C.c_int32 * MAX_LAYERS), ("scale_fine_on", C.c_int32 * MAX_LAYERS),
                ("scale", C.c_float * MAX_LAYERS), ("pivot", C.c_float * 3),
                ("near_plane", C.c_float), ("alpha_layer2", C.c_float), ("density_threshold", C.c_float),
                ("bkgd_density_threshold", C.c_float), ("boarder_weight", C.c_float),
                ("apply_thresholds", C.c_int32), ("shared_frame_id", C.c_int32)]


class View(C.Structure):
    """stnerf_view: one pose of a stnerf_render_views batch."""
    _fields_ = [("Kinv", C.c_float * 9), ("T", C.c_float * 16), ("frame_ids", C.c_float * MAX_LAYERS), ("scene", Scene),
                ("seed", C.c_uint64)]


class Grid(C.Structure):
    """stnerf_grid: point (i,j,k) = origin + (i,j,k)*step, values [dims0][dims1][dims2] (x slowest)."""
    _fields_ = [("origin", C.c_float * 3), ("step", C.c_float * 3), ("dims", C.c_int32 * 3)]


class Profile(C.Structure):
    _fields_ = [("ms", C.c_double * 4), ("points", C.c_double * 4), ("launches", C.c_uint64 * 4)]


_P = C.c_void_p
_SIGNATURES = {
    "stnerf_create": (C.c_int, [C.POINTER(_P), C.POINTER(ModelDesc)]),
    "stnerf_destroy": (None, [_P]),
    "stnerf_reserve": (C.c_int, [_P, C.c_int, C.c_int]),
    "stnerf_workspace_bytes": (C.c_size_t, [_P]),
    "stnerf_strerror": (C.c_char_p, [C.c_int]),
    "stnerf_last_cuda_error": (C.c_char_p, []),
    "stnerf_set_precision": (C.c_int, [_P, C.c_int]),
    "stnerf_load_spacenet": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_size_t]),
    "stnerf_load_motionnet": (C.c_int, [_P, C.c_int, _P, C.c_size_t]),
    "stnerf_weights_export": (C.c_int, [_P, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "stnerf_weights_import": (C.c_int, [_P, _P, C.c_size_t]),
    "stnerf_set_scene": (C.c_int, [_P, C.POINTER(Scene)]),
    "stnerf_set_box_table": (C.c_int, [_P, _P, C.c_int]),
    "stnerf_set_rotation": (C.c_int, [_P, _P, _P, _P]),
    "stnerf_rotate_rays": (C.c_int, [_P, C.c_int64, C.c_int, _P, _P, _P, _P]),
    "stnerf_render": (C.c_int, [_P, _P, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, C.c_uint64, _P, _P, _P]),
    "stnerf_render_host": (C.c_int, [_P, _P, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint64, _P, _P, _P]),
    "stnerf_reserve_host": (C.c_int, [_P, C.c_int64, C.c_int]),
    "stnerf_render_views": (C.c_int, [_P, C.POINTER(View), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                       _P, _P, C.c_int64, _P]),
    "stnerf_render_views_host": (C.c_int, [_P, C.POINTER(View), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "stnerf_raygen": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "stnerf_intersect_sample": (C.c_int, [_P, C.c_int64, C.c_int, _P, _P, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P]),
    "stnerf_composite": (C.c_int, [_P, _P, _P, C.c_int64, C.c_int, C.c_float, _P, _P, _P, _P, _P]),
    "stnerf_sample_pdf": (C.c_int, [_P, _P, _P, C.c_int64, C.c_int, C.c_int, _P, _P, _P]),
    "stnerf_composite_pass": (C.c_int, [C.POINTER(Scene), C.c_int, C.c_int, _P, _P, _P, _P, C.c_uint64, C.c_int64, C.c_int, C.c_int,
                                        C.c_int, _P, _P, _P, _P, _P]),
    "stnerf_positional_encoding": (C.c_int, [_P, C.c_int64, C.c_int, C.c_int, _P, _P]),
    "stnerf_spacenet": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P, C.c_int64, _P, _P, _P]),
    "stnerf_spacenet_pass": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P, C.c_int64, _P, _P, _P]),
    "stnerf_motionnet": (C.c_int, [_P, C.c_int, _P, C.c_int64, C.c_int, _P, _P]),
    "stnerf_layer_field": (C.c_int, [_P, C.c_int, C.c_int, C.c_float, _P, _P, C.c_int64, _P, _P, _P]),
    "stnerf_layer_grid": (C.c_int, [_P, C.c_int, C.c_int, C.c_float, C.POINTER(Grid), _P, _P]),
    "stnerf_mc_scratch_bytes": (C.c_size_t, [C.POINTER(Grid)]),
    "stnerf_mc_count": (C.c_int, [_P, C.POINTER(Grid), C.c_float, _P, C.c_size_t, C.POINTER(C.c_int64), C.POINTER(C.c_int64), _P]),
    "stnerf_mc_fill": (C.c_int, [_P, C.POINTER(Grid), C.c_float, _P, C.c_size_t, _P, _P, _P]),
    "stnerf_train_saved_floats": (C.c_size_t, [C.c_int, C.c_int, C.c_int64]),
    "stnerf_train_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int64]),
    "stnerf_spacenet_train_forward": (C.c_int, [_P, C.c_int, _P, _P, _P, C.c_int64, _P, _P, _P, _P]),
    "stnerf_spacenet_backward": (C.c_int, [_P, C.c_int, C.c_int64, _P, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "stnerf_motionnet_train_forward": (C.c_int, [_P, _P, C.c_int64, C.c_int, _P, _P, _P, C.c_size_t, _P]),
    "stnerf_motionnet_backward": (C.c_int, [_P, C.c_int64, _P, _P, _P, _P, C.c_size_t, _P]),
    "stnerf_train_scratch_bytes_prec": (C.c_size_t, [C.c_int, C.c_int, C.c_int64, C.c_int]),
    "stnerf_spacenet_train_forward_prec": (C.c_int, [_P, C.c_int, _P, _P, _P, C.c_int64, _P, _P, _P, C.c_int, _P]),
    "stnerf_spacenet_backward_prec": (C.c_int, [_P, C.c_int, C.c_int64, _P, _P, _P, _P, _P, _P, C.c_size_t, C.c_int, _P]),
    "stnerf_motionnet_train_forward_prec": (C.c_int, [_P, _P, C.c_int64, C.c_int, _P, _P, _P, C.c_size_t, C.c_int, _P]),
    "stnerf_motionnet_backward_prec": (C.c_int, [_P, C.c_int64, _P, _P, _P, _P, C.c_size_t, C.c_int, _P]),
    "stnerf_composite_backward": (C.c_int, [_P, _P, _P, C.c_int64, C.c_int, C.c_float, _P, _P, _P, _P, _P, _P, _P]),
    "stnerf_train_sample": (C.c_int, [_P, _P, C.c_int64, C.c_int, C.c_int, _P, C.c_uint64, _P, _P, _P, _P, _P, _P]),
    "stnerf_train_points": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int64, C.c_int, _P, C.c_int, _P, C.c_int64, _P, _P, _P, _P,
                                      _P]),
    "stnerf_train_scatter": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int64, C.c_int, _P, C.c_int64, _P, _P, _P, _P, _P, _P]),
    "stnerf_train_gather": (C.c_int, [_P, C.c_int, _P, C.c_int64, _P, _P, _P, _P, _P, _P]),
    "stnerf_train_uniforms": (C.c_int, [_P, C.c_int64, C.c_int, C.c_uint64, _P, _P]),
    "stnerf_td_select_scratch_ints": (C.c_int64, [C.c_int, C.c_int]),
    "stnerf_td_select_count": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P]),
    "stnerf_td_select_write": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P,
                                         _P, _P, _P]),
    "stnerf_td_batch": (C.c_int, [_P, _P, C.c_int, C.c_int64, _P, _P, C.c_int, C.c_int, _P, _P, C.c_int, C.c_float, C.c_int,
                                  _P, _P, _P, _P, _P, _P, _P]),
    "stnerf_debug_read_depths": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int64, C.c_int, _P]),
    "stnerf_launch_count": (C.c_uint64, []),
    "stnerf_set_ray_ids": (C.c_int, [_P, C.c_int64, C.c_int32, C.c_int64]),
    "stnerf_selftest_umma": (C.c_int, [C.POINTER(C.c_float)]),
    "stnerf_selftest_umma_accum": (C.c_int, [C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "stnerf_profile_begin": (C.c_int, [_P]),
    "stnerf_profile_end": (C.c_int, [_P, C.POINTER(Profile)]),
}
EXPORTS = tuple(_SIGNATURES)

_lib = None


class StnerfError(RuntimeError):
    pass


def lib():
    """Load the shared library (once).  Raises if it has not been built: there is no fallback path."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise StnerfError("%s not found -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(the H100 path has no CPU fallback)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(code: int, what: str = ""):
    if code != 0:
        L = lib()
        msg = L.stnerf_strerror(code).decode()
        if code == -3:
            msg += ": " + L.stnerf_last_cuda_error().decode()
        raise StnerfError("%s failed (%d): %s" % (what or "stnerf call", code, msg))


def ptr(t):
    """Device/host pointer of a torch tensor (or None)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
