"""CPU checker of dim_render_dataset (test infrastructure): ctypes face of tests/py_light_oracle.c, which compiles the
oracle (oracle/deepim_oracle.c, unchanged) together with the Render_Py_Light shading and the dataset files' conversions.
The library is built on first use with the oracle's compiler flags, into a temporary directory (the tree may be
read-only)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "py_light_oracle.c")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="py_light_oracle_"), "libpy_light_oracle.so")
        with open("/proc/cpuinfo") as f:
            fma = ["-mfma"] if " fma " in f.read() else []  # oracle/Makefile's FMA switch
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c11", "-ffp-contract=off", "-fno-fast-math"] + fma +
                              ["-fPIC", "-fvisibility=hidden", "-Wall", "-Wno-unused-function", "-shared", "-o", so, _SRC, "-lm"])
        L = C.CDLL(so)
        vp, f32p, i32p, u8p = C.c_void_p, O.f32p, O.i32p, O.u8p
        L.pyl_render_dataset.argtypes = [f32p, f32p, vp, C.c_int32, i32p, C.c_int32, u8p, C.c_int32, C.c_int32, f32p, f32p,
                                         C.c_float, C.c_float, C.c_int32, C.c_int32, vp, vp, C.c_float, C.c_float, vp, vp, vp,
                                         vp]
        L.pyl_render_dataset.restype = None
        _LIB = L
    return _LIB


def render_dataset(mesh, pose, K, light_position=None, light_intensity=None, brightness_ratio=None, zn=0.25, zf=6.0, H=480,
                   W=640, depth_factor=1000.0):
    """One instance as the dataset files hold it (toolkit/LM6d_ds_1, ds_2, ds_4, LM6d_0): lit_bgr u8 [H,W,3]
    (Render_Py_Light, render_py_light.py; only with a light, needs mesh.normals), bgr u8 [H,W,3] (Render_Py colour
    .astype('uint8')), depth u16 [H,W] ((depth * depth_factor).astype(np.uint16)), label u8 [H,W] (depth != 0)."""
    lit = light_position is not None
    out = {"lit_bgr": np.zeros((H, W, 3), np.uint8) if lit else None, "bgr": np.zeros((H, W, 3), np.uint8),
           "depth": np.zeros((H, W), np.uint16), "label": np.zeros((H, W), np.uint8)}
    keep = [np.ascontiguousarray(mesh.normals, np.float32), np.ascontiguousarray(light_position, np.float32),
            np.ascontiguousarray(light_intensity, np.float32)] if lit else [None, None, None]
    p = O._ptr
    lib().pyl_render_dataset(mesh.verts, mesh.uvs, p(keep[0]), len(mesh.verts), mesh.faces, len(mesh.faces), mesh.tex,
                             mesh.tex.shape[0], mesh.tex.shape[1], np.ascontiguousarray(pose, np.float32), O.k4(K), zn, zf, H,
                             W, p(keep[1]), p(keep[2]), float(np.float32(brightness_ratio)) if lit else 0.0, float(depth_factor),
                             p(out["lit_bgr"]), p(out["bgr"]), p(out["depth"]), p(out["label"]))
    return out
