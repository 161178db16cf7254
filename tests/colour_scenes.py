"""Vertex-coloured versions of the rasteriser's test scenes and their float64 checks (TEST INFRASTRUCTURE), shared by
tests/test_ply_colours.py (the CPU checker) and tests/test_gpu_mesh_colours.py (the device).

A coloured mesh keeps the geometry and normals of its textured original and gets seeded per-vertex colours in [0, 1],
with exact 0 and 1 channels among them.  The ray caster (tests/raster_ref.py) interpolates them perspective-correctly with
`Render._interp`; the five-evaluation rule of raster_ref.py decides which pixels are checked and how tightly:
- float colours (the train path's c * 255): within [min, max] of the five evaluations, widened by 8 ulp of 255 and by
  the interval's own width.  The five points bracket a common shift of the triangle; the device snaps each vertex on
  its own, which on a sliver (the fan scene's hub) moves the barycentrics by about as much again;
- u8 colours (the test path and the dataset's bgr): exact where that widened interval, and 1e-3 level beyond it, holds
  one integer part;
- lit colours (ModelNet and Py_Light): within [min, max] of the five evaluations' levels, widened by its width and by
  0.5 + 1e-3 levels.
On the blobs a triangle covers a pixel or less and the random colours change by up to a full range across it, so the
widening matters there; the bit-exact comparisons with the CPU checker hold the float32 sequence itself."""
from __future__ import annotations

import copy

import numpy as np

from deepim_b200 import synth

import raster_ref as RR

FLOAT_SLACK = 8 * float(np.spacing(np.float32(255.0)))
INT_MARGIN = 1e-3


def coloured(mesh, seed=0):
    """the mesh's geometry and normals with seeded vertex colours"""
    rs = np.random.RandomState(1000 + seed)
    c = rs.uniform(0.0, 1.0, (len(mesh.verts), 3)).astype(np.float32)
    c[rs.uniform(size=c.shape) < 0.05] = 0.0
    c[rs.uniform(size=c.shape) < 0.05] = 1.0
    m = synth.Mesh(mesh.verts, None, mesh.faces, None, mesh.name + "+colours", colours=c)
    if getattr(mesh, "normals", None) is not None:
        m.normals = mesh.normals
    return m


def coloured_scene(s):
    """scene s with every mesh replaced by its coloured version"""
    c = copy.copy(s)
    c.meshes = [coloured(m, k) for k, m in enumerate(s.meshes)]
    return c


def _levels(ref, colours):
    """[5, len(sel), 3] float64 BGR level 255 c of each evaluation"""
    return (ref._interp(colours) * 255.0)[..., ::-1]


def check_colours(rep, ref, bgr, trunc_u8):
    """an unlit render's BGR [H,W,3] (float c * 255, or its u8 truncation) against the interpolated vertex colours"""
    c = bgr.reshape(-1, 3)
    rest = np.ones(len(c), bool)
    rest[ref.sel] = False
    rep.bad("background", (c[rest] != 0).any(-1).sum())
    c = c[ref.sel].astype(np.float64)
    cov = ref.covered
    agree = RR.unanimous(cov)
    on = agree & cov[0] & RR.clear_winner(ref)
    rep.bad("background", (c != 0).any(-1)[agree & ~cov[0]].sum())
    lv = _levels(ref, ref.mesh.colours)
    lo, hi = _widened(lv)
    if trunc_u8:
        fl = np.floor(lo - INT_MARGIN)
        sure = on & (fl == np.floor(hi + INT_MARGIN)).all(-1)
        rep.bad("u8 colour", (c != fl).any(-1)[sure].sum())
        rep.ambiguous_colour = getattr(rep, "ambiguous_colour", 0) + int((on & ~sure).sum())
    else:
        lo, hi = lo - FLOAT_SLACK, hi + FLOAT_SLACK
        rep.worst("colour", RR._ratio(c, lo, hi, np.clip(lv[0], lo, hi))[on])


def _widened(lv):
    """[min, max] of the five evaluations [5, n, 3], widened by its own width on each side"""
    lo, hi = lv.min(0), lv.max(0)
    return lo - (hi - lo), hi + (hi - lo)


def check_lit_colours(rep, ref, bgr, light_pos, light_int, ratio, shader):
    """a lit render's u8-valued BGR against the five evaluations' levels with the interpolated colours, +-(0.5 + 1e-3)"""
    c = bgr.reshape(-1, 3)
    rest = np.ones(len(c), bool)
    rest[ref.sel] = False
    rep.bad("lit background", (c[rest] != 0).any(-1).sum())
    c = c[ref.sel].astype(np.float64)
    cov = ref.covered
    agree = RR.unanimous(cov)
    a1 = float(np.float32(ratio))
    a0 = float(np.float32(1.0 - np.float32(ratio)))
    I = np.asarray(light_int, np.float32).astype(np.float64)
    br = ref.brightness(light_pos)[..., None]
    t = ref._interp(ref.mesh.colours)
    lit = t * ((a0 + a1 * br) * I) if shader == "modelnet" else t * (a0 + a1 * br * I)
    lv = (np.clip(lit, 0.0, 1.0) * 255.0)[..., ::-1]
    lo, hi = _widened(lv)
    lo, hi = lo - RR.COLOUR_LEVELS, hi + RR.COLOUR_LEVELS
    on = agree & cov[0] & RR.clear_winner(ref)
    rep.worst("lit " + shader, RR._ratio(c, lo, hi, np.clip(lv[0], lo, hi))[on])
    rep.bad("lit background", (c != 0).any(-1)[agree & ~cov[0]].sum())
