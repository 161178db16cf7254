"""CPU: the oracle's rasteriser (`orc_render`, `orc_render_lit` and the dataset render of tests/py_light_oracle.c) against
an independent float64 ray caster (tests/raster_ref.py), on the scenes of tests/raster_scenes.py, and known answers
of the ray caster itself.  The device is held bit for bit to the oracle, so what passes here holds for it too;
tests/test_gpu_raster_float64.py checks the device against the ray caster directly."""
import numpy as np
import pytest

from oracle import oracle as O

import py_light_oracle as PL
import raster_ref as RR
import raster_scenes as RS

SCENES = RS.geometry_scenes() + RS.mesh_scenes() + [RS.batch16_scene()]
FACTOR = 1000.0


def check_scene_oracle(s):
    """every instance of scene s through the three oracle renders; returns the tally"""
    rep = RR.Report(repr(s))
    for c, pose, lpos, inten, ratio in s.inst:
        m = s.meshes[c]
        ref = RR.Render(m, pose, s.K, s.H, s.W, s.zn, s.zf, m.normals)
        geo = dict(zn=s.zn, zf=s.zf, H=s.H, W=s.W)
        for trunc in (True, False):
            o = O.render(m, pose, s.K, trunc_u8=trunc, **geo)
            RR.check_render(rep, ref, o["depth"], o["mask"], o["bgr"], trunc)
        o = O.render_lit(m, m.normals, pose, s.K, lpos, inten, ratio, **geo)
        RR.check_render(rep, ref, o["depth"], o["mask"])
        RR.check_lit(rep, ref, o["bgr"], lpos, inten, ratio, "modelnet")
        o = PL.render_dataset(m, pose, s.K, lpos, inten, ratio, depth_factor=FACTOR, **geo)
        RR.check_lit(rep, ref, o["lit_bgr"], lpos, inten, ratio, "py_light")
        RR.check_render(rep, ref, o["label"], bgr=o["bgr"], trunc_u8=True, label=True)
        RR.check_u16(rep, ref, o["depth"], o["label"], FACTOR)
    return rep


@pytest.mark.parametrize("s", SCENES, ids=repr)
def test_oracle_against_float64(s):
    rep = check_scene_oracle(s)
    print(rep)
    assert rep.ok, str(rep)


def test_ownership_grid_oracle():
    """vertices on pixel centres and half-pixels: the owner of every pixel on an edge or a vertex is the one the rule
    gives on the exact geometry, and the grid is watertight"""
    s, tri2 = RS.ownership_grid()
    m = s.meshes[0]
    owner = RS.grid_owner(tri2, s.H, s.W)
    o = O.render(m, s.inst[0][1], s.K, H=s.H, W=s.W)
    got = o["bgr"].astype(np.int64)
    face = np.where(o["depth"] > 0, got[..., 2] + 256 * got[..., 1], -1)  # the texel index is the face index
    assert (owner >= 0).sum() == 140 * 105
    assert np.array_equal(face, owner), int((face != owner).sum())
    assert np.all(np.abs(o["depth"][owner >= 0] - 1.0) <= 2 * np.spacing(np.float32(1.0)))


# ---------------------------------------------------------------------------------------- known answers of raster_ref
K = RS.K_LM


def test_ref_fronto_parallel_depth_is_constant():
    m = RS.quad(0.1, 0.08, RS._tex(37, 53, 1))
    r = RR.Render(m, RS.pose(t=(0.01, 0.02, 1.3)), K, 480, 640)
    z = r.z[r.covered]
    assert len(z) > 5 * 6000 and np.all(np.abs(z - np.float64(np.float32(1.3))) <= 1e-15)


def test_ref_tilted_plane_depth_is_the_ray_plane_depth():
    R = RS.rot((1, 0.4, 0.2), 55)
    p = RS.pose(R, (0.02, -0.01, 1.1))
    r = RR.Render(RS.quad(0.15, 0.1, RS._tex(5, 61, 4)), p, K, 480, 640)
    P = p.astype(np.float64)
    n, t = np.cross(P[:, 0], P[:, 1]), P[:, 3]  # the model's z = 0 plane (the float32 R is not exactly orthonormal)
    fx, fy, cx, cy = RR.camera(K)
    i, j = np.divmod(r.sel, 640)
    z_c = np.dot(n, t) / (n[0] * (j - cx) / fx + n[1] * (i - cy) / fy + n[2])
    cov = r.covered[0]
    assert cov.sum() > 5000 and np.abs(r.z[0][cov] - z_c[cov]).max() <= 1e-12 * z_c.max()


def test_ref_uv_is_perspective_correct():
    """on a quad tilted 70 degrees the UV is the ray-plane hit's; screen-affine interpolation differs from it by the
    closed-form amount, a sizeable fraction of the texture"""
    R = RS.rot((0, 1, 0), 70)
    p = RS.pose(R, (0, 0, 1.0))
    h = float(np.float32(0.2))
    r = RR.Render(RS.quad(h, h, RS._tex(37, 53, 1)), p, K, 480, 640)
    cov = r.covered[0]
    uv = r.uv()[0][cov]
    fx, fy, cx, cy = RR.camera(K)
    i, j = np.divmod(r.sel[cov], 640)
    P = p.astype(np.float64)
    d = np.stack([(j - cx) / fx, (i - cy) / fy, np.ones_like(j, dtype=np.float64)], 1)
    n = np.cross(P[:, 0], P[:, 1])
    s = np.dot(n, P[:, 3]) / (d @ n)
    x_model = np.linalg.solve(P[:, :3], (s[:, None] * d - P[:, 3]).T).T  # back to model coordinates
    assert np.abs(uv - (x_model[:, :2] + h) / (2 * h)).max() < 1e-12
    # screen-affine u: linear in the column between the quad's projected left and right edges
    ends = (np.array([[-h, 0, 0], [h, 0, 0]]) @ P[:, :3].T + P[:, 3])
    uend = fx * ends[:, 0] / ends[:, 2] + cx
    row = i == int(round(cy))
    a = (j[row] - uend[0]) / (uend[1] - uend[0])
    z0, z1 = ends[:, 2]
    assert np.abs(uv[row, 0] - (a / z1) / ((1 - a) / z0 + a / z1)).max() < 1e-9  # 1/z-weighted screen parameter
    assert np.abs(a - uv[row, 0]).max() > 0.09  # screen-affine u is off by up to a tenth of the texture


def test_ref_brightness_facing_the_light():
    """a surface facing a light straight on has brightness 1; turned by 60 degrees from it, cos 60 at the centre"""
    m = RS.quad(0.02, 0.02, RS._tex(1, 1, 2))
    m.normals = np.tile([[0, 0, -1.0]], (4, 1)).astype(np.float32)
    p = RS.pose(t=(0, 0, 1.0))
    r = RR.Render(m, p, K, 480, 640, normals=m.normals)
    br = r.brightness(np.float32([0, 0, 0]))[r.covered]
    assert np.all(br > 0.999)  # light at the eye, 1 m in front of the quad: at most 1.6 degrees off its normal
    i, j = 242, 325
    k = np.searchsorted(r.sel, i * 640 + j)
    assert abs(r.brightness(np.float32([0, 0, 0]))[0, k] - 1.0) < 1e-3
    m.normals = np.tile(RS.rot((0, 1, 0), 60) @ [0, 0, -1.0], (4, 1)).astype(np.float32)
    r = RR.Render(m, p, K, 480, 640, normals=m.normals)
    assert abs(r.brightness(np.float32([0, 0, 0]))[0, k] - 0.5) < 1e-3


def test_ref_drop_rule_and_ties():
    """a vertex projecting beyond 1e6 px drops its triangle; coplanar duplicates resolve to the lowest face index"""
    P = RS.at_pixels([[300.2, 200], [2e6, 230.5], [360.7, 270.3]], K, [0.8, 0.9, 1.1])
    r = RR.Render(RS.tris_mesh(P, RS._tex(1, 1, 2)), RS.pose(), K, 480, 640)
    assert r.dropped == 1 and len(r.sel) == 0
    P = RS.at_pixels([[300.2, 200], [360.5, 230.5], [320.7, 270.3]] * 2, K, [0.8, 0.9, 1.1] * 2)
    r = RR.Render(RS.tris_mesh(P, RS._tex(1, 1, 2)), RS.pose(), K, 480, 640)
    assert r.covered.sum() > 1000 and np.all(r.face[r.covered] == 0)
