"""ctypes binding of libdeepim_b200.so (include/deepim_b200.h).  No fallback: if the library is
missing or fails to load, importing this module raises."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "libdeepim_b200.so")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        "libdeepim_b200.so not found at %s -- build it with `python mx-deepim_b200/build.py` "
        "(there is no CPU / PyTorch fallback for this path)" % LIB_PATH)

lib = C.CDLL(LIB_PATH)

vp, i32, i64, u64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_float
pf32 = C.POINTER(C.c_float)
pf64 = C.POINTER(C.c_double)

class TrainConfig(C.Structure):
    """dim_train_config (include/deepim_b200.h): loss weights / normalisers / pose parameterisation of the yaml"""
    _fields_ = [("lw_flow", f32), ("lw_mask", f32), ("lw_pm", f32), ("num_3d_sample", f32), ("normalize_3d_point", f32),
                ("normalize_flow", f32), ("trans_means", f32 * 3), ("trans_stds", f32 * 3), ("rot_coord", i32)]


class Lighting(C.Structure):
    """dim_lighting (include/deepim_b200.h): the ModelNet branch's light -- intensity pointer, offset at zero translation
    (GL frame), brightness ratio"""
    _fields_ = [("intensity", vp), ("offset", C.c_double * 3), ("brightness_ratio", f32)]


plit = C.POINTER(Lighting)


# name -> (restype, argtypes); every symbol declared in include/deepim_b200.h
SIGNATURES = {
    "dim_abi_version": (i32, []),
    "dim_last_error": (C.c_char_p, []),
    "dim_ctx_create": (i32, [i32, i32, i32, i32, i32, i32, i32, C.POINTER(vp)]),
    "dim_ctx_destroy": (None, [vp]),
    "dim_mesh_upload": (i32, [vp, i32, vp, vp, i32, vp, i32, vp, i32, i32]),
    "dim_mesh_upload_colours": (i32, [vp, i32, vp, vp, i32, vp, i32]),
    "dim_render": (i32, [vp, vp, vp, i32, pf32, f32, f32, pf64, i32, vp, vp, vp, vp, vp, vp]),
    "dim_zoom_mask_fwd": (i32, [vp, vp, vp, vp, vp, i32, pf32, vp, vp, vp, vp, vp, vp, vp]),
    "dim_zoom_image_with_factor_fwd": (i32, [vp, vp, vp, vp, i32, pf32, vp, vp, vp]),
    "dim_mesh_upload_normals": (i32, [vp, i32, vp, i32]),
    "dim_render_lit": (i32, [vp, vp, vp, i32, pf32, f32, f32, pf64, vp, vp, f32, vp, vp, vp, vp, vp, vp]),
    "dim_render_dataset": (i32, [vp, vp, vp, i32, pf32, f32, f32, f32, vp, vp, vp, vp, vp, vp, vp, vp]),
    "dim_zoom_image_fwd": (i32, [vp, vp, vp, vp, i32, pf32, pf32, vp, vp, vp, vp, vp, vp]),
    "dim_group_picker": (i32, [vp, vp, vp, i32, i32, i32, i64, i32, vp, vp]),
    "dim_zoom_mask_with_factor_fwd": (i32, [vp, vp, vp, i32, i32, vp, vp]),
    "dim_zoom_flow_fwd": (i32, [vp, vp, vp, vp, i32, i32, i32, vp, vp, vp]),
    "dim_zoom_depth_fwd": (i32, [vp, vp, vp, vp, i32, vp, vp, vp]),
    "dim_zoom_trans_fwd": (i32, [vp, vp, vp, i32, i32, vp, vp]),
    "dim_zoom_trans_bwd": (i32, [vp, vp, vp, i32, i32, i32, vp, vp]),
    "dim_update_mask_box": (i32, [vp, vp, i32, vp, vp]),
    "dim_se3_compose": (i32, [vp, vp, vp, i32, pf64, pf64, i32, vp, vp]),
    "dim_flow_fwd": (i32, [vp, vp, vp, vp, pf32, i32, vp, vp, vp]),
    "dim_transform3d_fwd": (i32, [vp, vp, vp, vp, vp, i32, i32, pf32, pf32, i32, vp, vp]),
    "dim_transform3d_bwd": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, pf32, pf32, i32, vp, vp, vp]),
    "dim_train_update": (i32, [vp, vp, vp, vp, vp, vp, vp, i32, pf64, f32, f32, pf64, pf64, pf64, i32, vp, vp, vp, vp, vp,
                               vp, vp, vp, plit, vp]),
    "dim_net_load": (i32, [vp, C.POINTER(vp), C.POINTER(vp)]),
    "dim_net_fwd": (i32, [vp, vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp]),
    "dim_refine": (i32, [vp, vp, i32, vp, pf32, vp, vp, vp, i32, i32, f32, f32, pf64, i32, vp, vp, vp, vp, vp, vp, plit, vp]),
    "dim_refine_host_async": (i32, [vp, vp, i32, vp, pf32, vp, vp, vp, i32, i32, f32, f32, pf64, i32, vp, vp, vp, f32, plit,
                                    vp]),
    "dim_ctx_set_input_depth": (i32, [vp, i32]),
    "dim_ctx_set_input_mask": (i32, [vp, i32]),
    "dim_transform_image_u8": (i32, [vp, vp, i32, pf64, vp, vp]),
    "dim_bg_upload": (i32, [vp, i32, vp, i32, i32]),
    "dim_bg_geometry": (i32, [i32, i32, i32, i32, C.POINTER(i32), pf64]),
    "dim_replace_background": (i32, [vp, vp, vp, vp, i32, pf64, vp, vp, vp]),
    "dim_mask_dilate": (i32, [vp, vp, vp, i32, vp, vp]),
    "dim_debug_activation": (i32, [vp, i32, i32, vp, u64]),
    "dim_debug_layer_geometry": (i32, [vp, i32, C.POINTER(i32)]),
    "dim_refine_status": (i32, [vp, i32, i32, vp, vp]),
    "dim_icp": (i32, [vp, vp, i32, vp, pf32, vp, vp, vp, i32, i32, f32, f32, f32, i32, vp, vp, vp, vp, vp]),
    "dim_depth_from_u16": (i32, [vp, vp, i32, f32, vp, vp]),
    "dim_pose_error_vsd": (i32, [vp, vp, i32, vp, pf32, vp, vp, vp, vp, i32, f32, f32, f32, pf64, i32, vp, vp, vp]),
    "dim_pose_error_vsd_ex": (i32, [vp, vp, i32, vp, pf32, vp, vp, vp, vp, i32, f32, f32, f32, pf64, i32, i32, pf64, vp, vp,
                                    vp]),
    "dim_pose_error_sym": (i32, [vp, vp, vp, i32, vp, i32, vp, i32, vp, vp, vp, vp]),
    "dim_debug_set_option": (i32, [vp, C.c_char_p, i32]),
    "dim_debug_graph_count": (i32, [vp]),
    "dim_debug_train_update": (i32, [vp, i32, pf32, pf32]),
    "dim_debug_layer_profile": (i32, [vp, i32, pf32]),
    "dim_profile_enable": (i32, [vp, i32]),
    "dim_profile_read": (i32, [vp, pf32, C.POINTER(i32)]),
    "dim_launch_count": (i64, [i32]),
    "dim_pose_error": (i32, [vp, vp, vp, i32, vp, i32, i32, vp, vp]),
    "dim_pose_error_2d": (i32, [vp, vp, vp, i32, vp, i32, vp, vp, vp]),
    "dim_flow_epe": (i32, [vp, vp, vp, vp, vp, i32, vp, vp]),
    "dim_train_create": (i32, [vp, i32]),
    "dim_train_param_count": (i64, [vp]),
    "dim_train_param_info": (i32, [i32, i32, i32, C.POINTER(C.c_char_p), C.POINTER(i64), C.POINTER(i64)]),
    "dim_train_load_params": (i32, [vp, vp, i64, vp]),
    "dim_train_get_params": (i32, [vp, vp, i64, i32, vp]),
    "dim_train_forward_backward": (i32, [vp] + [vp] * 12 + [i32, i32] + [vp] * 7 + [vp, vp, i32] + [vp, vp] + [vp]),
    "dim_train_set_config": (i32, [vp, C.POINTER(TrainConfig)]),
    "dim_train_get_config": (i32, [vp, C.POINTER(TrainConfig)]),
    "dim_train_sgd_update": (i32, [vp, vp, f32, f32, f32, f32, vp]),
    "dim_train_set_precision": (i32, [vp, i32]),
    "dim_train_get_precision": (i32, [vp, C.POINTER(i32)]),
    "dim_train_debug_tensor": (i32, [vp, i32, vp, C.c_uint64]),
    "dim_train_debug_phases": (i32, [vp, pf32]),
    "dim_train_debug_geometry": (i32, [vp, i32, C.POINTER(i32)]),
    "dim_train_debug_wgrad_slices": (i32, [vp, i32, C.POINTER(i32)]),
}

for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(lib, _name)  # AttributeError here = header/library mismatch
    _fn.restype = _res
    _fn.argtypes = _args

PREC_BF16 = 0    # one bf16 pass: fast mode, se3 only within ~2e-3 of the fp32 reference
PREC_BF16X3 = 1  # bf16 hi/lo split, 3 passes: near-fp32
PREC_FP16 = 2    # one fp16 pass: meets the 1e-4 rot / 1e-3 trans se3 tolerance at the bf16 MMA rate (default)
PRECISIONS = {"bf16": PREC_BF16, "bf16x3": PREC_BF16X3, "fp16": PREC_FP16}


def precision_id(p):
    """'fp16' | 'bf16x3' | 'bf16' (or an already numeric id) -> DIM_PREC_* value"""
    if isinstance(p, str):
        if p not in PRECISIONS:
            raise ValueError("unknown precision %r (one of %s)" % (p, sorted(PRECISIONS)))
        return PRECISIONS[p]
    if int(p) not in PRECISIONS.values():
        raise ValueError("unknown precision id %r" % (p,))
    return int(p)

ROT_COORD = {"model": 0, "camera": 1, "camera_new": 2}


class DeepIMError(RuntimeError):
    pass


def check(rc: int):
    if rc != 0:
        raise DeepIMError("libdeepim_b200: rc=%d: %s" % (rc, lib.dim_last_error().decode("utf-8", "replace")))


def farr(values, n=None, ctype=C.c_float):
    vals = [float(v) for v in values]
    if n is not None and len(vals) != n:
        raise ValueError("expected %d values, got %d" % (n, len(vals)))
    return (ctype * len(vals))(*vals)
