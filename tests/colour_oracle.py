"""CPU checker of vertex-coloured meshes (test infrastructure): ctypes face of tests/colour_oracle.c, which compiles the
oracle (oracle/deepim_oracle.c, unchanged) together with the vertex-colour source.  `render`, `render_lit` and
`render_dataset` take the arguments of oracle.render, oracle.render_lit and py_light_oracle.render_dataset and draw a
mesh with `colours` here and a textured one there.  Inside `dispatching()`, oracle.refine and oracle.train_update render
through them, so the oracle's loop and update run on coloured meshes unchanged.  The library is built on first use with
the oracle's compiler flags, into a temporary directory (the tree may be read-only)."""
import contextlib
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

import py_light_oracle as PL

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "colour_oracle.c")
_LIB = None
UNLIT, MODELNET, PY_LIGHT = 0, 1, 2
_TEXTURED = {"render": O.render, "render_lit": O.render_lit}


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="colour_oracle_"), "libcolour_oracle.so")
        with open("/proc/cpuinfo") as f:
            fma = ["-mfma"] if " fma " in f.read() else []  # oracle/Makefile's FMA switch
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c11", "-ffp-contract=off", "-fno-fast-math"] + fma +
                              ["-fPIC", "-fvisibility=hidden", "-Wall", "-Wno-unused-function", "-shared", "-o", so, _SRC, "-lm"])
        L = C.CDLL(so)
        vp, f32p, i32p = C.c_void_p, O.f32p, O.i32p
        L.col_render.argtypes = [f32p, f32p, vp, C.c_int32, i32p, C.c_int32, f32p, f32p, C.c_float, C.c_float, C.c_int32,
                                 C.c_int32, O.f64p, C.c_int32, C.c_int32, vp, vp, C.c_float, C.c_float, vp, vp, vp, vp, vp,
                                 C.c_float, vp, vp, vp, vp]
        L.col_render.restype = None
        _LIB = L
    return _LIB


def _call(mesh, pose, K, zn, zf, H, W, means_rgb, trunc_u8, shader, normals=None, light_pos=None, light_int=None, ratio=0.0,
          out=(), u8=(), depth_factor=0.0):
    """col_render with the float outputs named in `out` and the dataset outputs named in `u8`"""
    bufs = {"bgr": (H, W, 3), "depth": (H, W), "image": (3, H, W), "mask": (H, W)}
    res = {k: (np.empty(s, np.float32) if k in out else None) for k, s in bufs.items()}
    ds = {"bgr": np.zeros((H, W, 3), np.uint8) if "bgr" in u8 else None,
          "lit_bgr": np.zeros((H, W, 3), np.uint8) if "lit_bgr" in u8 else None,
          "depth": np.zeros((H, W), np.uint16) if "depth" in u8 else None,
          "label": np.zeros((H, W), np.uint8) if "label" in u8 else None}
    bbox = np.zeros(4, np.int32)
    means = np.zeros(3, np.float64) if means_rgb is None else np.ascontiguousarray(means_rgb, np.float64)
    keep = [None if a is None else np.ascontiguousarray(a, np.float32) for a in (normals, light_pos, light_int)]
    a1 = float(np.float32(ratio))
    a0 = float(np.float32(1.0 - a1))
    p = O._ptr
    lib().col_render(mesh.verts, np.ascontiguousarray(mesh.colours, np.float32), p(keep[0]), len(mesh.verts), mesh.faces,
                     len(mesh.faces), np.ascontiguousarray(pose, np.float32), O.k4(K), zn, zf, H, W, means, int(trunc_u8),
                     shader, p(keep[1]), p(keep[2]), a0, a1, p(res["bgr"]), p(res["depth"]), p(res["image"]),
                     p(res["mask"]), p(bbox), float(depth_factor), p(ds["bgr"]), p(ds["lit_bgr"]), p(ds["depth"]),
                     p(ds["label"]))
    res["bbox"] = bbox
    return res, ds


def render(mesh, pose, K, zn=0.25, zf=6.0, H=480, W=640, means_rgb=None, trunc_u8=True,
           want=("bgr", "depth", "image", "mask")):
    """oracle.render for either kind of mesh"""
    if mesh.colours is None:
        return _TEXTURED["render"](mesh, pose, K, zn, zf, H, W, means_rgb, trunc_u8, want)
    return _call(mesh, pose, K, zn, zf, H, W, means_rgb, trunc_u8, UNLIT, out=want)[0]


def render_lit(mesh, normals, pose, K, light_position, light_intensity, brightness_ratio=0.7, zn=0.25, zf=6.0, H=480, W=640,
               means_rgb=None, want=("bgr", "depth", "image", "mask")):
    """oracle.render_lit (ModelNet shading) for either kind of mesh"""
    if mesh.colours is None:
        return _TEXTURED["render_lit"](mesh, normals, pose, K, light_position, light_intensity, brightness_ratio, zn, zf, H,
                                       W, means_rgb, want)
    return _call(mesh, pose, K, zn, zf, H, W, means_rgb, True, MODELNET, normals, light_position, light_intensity,
                 brightness_ratio, out=want)[0]


def render_dataset(mesh, pose, K, light_position=None, light_intensity=None, brightness_ratio=None, zn=0.25, zf=6.0, H=480,
                   W=640, depth_factor=1000.0):
    """py_light_oracle.render_dataset for either kind of mesh"""
    if mesh.colours is None:
        return PL.render_dataset(mesh, pose, K, light_position, light_intensity, brightness_ratio, zn, zf, H, W, depth_factor)
    lit = light_position is not None
    return _call(mesh, pose, K, zn, zf, H, W, None, False, PY_LIGHT if lit else UNLIT, mesh.normals if lit else None,
                 light_position, light_intensity, brightness_ratio if lit else 0.0,
                 u8=("bgr", "depth", "label") + (("lit_bgr",) if lit else ()), depth_factor=depth_factor)[1]


@contextlib.contextmanager
def dispatching():
    """oracle.refine / oracle.train_update (and everything else of the oracle that renders) draw coloured meshes here"""
    O.render, O.render_lit = render, render_lit
    try:
        yield
    finally:
        O.render, O.render_lit = _TEXTURED["render"], _TEXTURED["render_lit"]
