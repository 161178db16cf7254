"""Scenes for the rasteriser's float64 tests (TEST INFRASTRUCTURE), shared by tests/test_raster_float64.py (the CPU
oracle) and tests/test_gpu_raster_float64.py (the device).

A scene is one context size and camera and a list of instances (mesh, float32 pose, light).  Every mesh carries
per-vertex normals, so each scene is drawn unlit, ModelNet-lit and as dataset files.  The geometry targets the places
where a rasteriser goes wrong: tilted and grazing surfaces, texture edges and non-power-of-two textures, slivers,
vertices far off screen, the near and far planes, overlaps and exact depth ties, partial blocks and warps, and the
48 / 49-pixel boundary between the coverage kernel's per-thread and warp-cooperative paths."""
from __future__ import annotations

import numpy as np

from deepim_b200 import synth

# cameras: LINEMOD's, an off-centre one with fx != fy, one with its principal point outside the frame, a small one
K_LM = synth.K_LINEMOD
K_OFF = np.array([[150.0, 0, 40.3], [0, 172.0, 60.7], [0, 0, 1]], np.float32)
K_OUT = np.array([[90.0, 0, -15.5], [0, 80.0, 140.2], [0, 0, 1]], np.float32)
K_SMALL = np.array([[40.0, 0, 20.1], [0, 46.0, 14.9], [0, 0, 1]], np.float32)
# (H, W, K): 480 x 640, 120 x 160, 97 x 132 (odd H, W / 4 odd) and 33 x 36
VIEWS = {"lm": (480, 640, K_LM), "out": (120, 160, K_OUT), "off": (97, 132, K_OFF), "small": (33, 36, K_SMALL)}


class Scene:
    def __init__(self, name, view, zn=0.25, zf=6.0):
        self.name, self.view = name, view
        self.H, self.W, self.K = VIEWS[view]
        self.zn, self.zf = zn, zf
        self.meshes, self.inst = [], []  # inst: (mesh index, pose [3,4] f32, light position f32[3], intensity f32[3], ratio)

    def add(self, mesh, pose, seed=0):
        if not any(m is mesh for m in self.meshes):
            self.meshes.append(mesh)
        c = [k for k, m in enumerate(self.meshes) if m is mesh][0]
        rs = np.random.RandomState(seed + 17 * len(self.inst))
        pose = np.asarray(pose, np.float32)
        # the light of tester.py:146-160 (offset + (x, -y, -z) of the translation, GL eye frame), a random colour and ratio
        off = np.array([[0, 0.5, 0.5], [0.5, 0, 0.5], [-0.5, 0.5, 0], [0, -0.5, 0.5]])[len(self.inst) % 4]
        lpos = (off + pose[:, 3].astype(np.float64) * [1, -1, -1]).astype(np.float32)
        inten = rs.uniform(0.5, 1.2, 3).astype(np.float32)
        ratio = np.float32([0.2, 0.5, 0.7, 0.9][len(self.inst) % 4])
        self.inst.append((c, pose, lpos, inten, ratio))
        return self

    @property
    def cls(self):
        return np.array([i[0] for i in self.inst], np.int32)

    def __repr__(self):
        return "%s@%s" % (self.name, self.view)


# ----------------------------------------------------------------------------------------------------------- meshes
def _tex(h, w, seed):
    return np.random.RandomState(seed).randint(0, 256, (h, w, 3)).astype(np.uint8)


def _mesh(verts, uvs, faces, tex, normals=None, name="m"):
    m = synth.Mesh(np.asarray(verts, np.float64), uvs, faces, tex, name)
    m.normals = synth.vertex_normals(m) if normals is None else np.asarray(normals, np.float32)
    return m


def quad(half_w, half_h, tex, uv0=0.0, uv1=1.0, bend=0.0):
    """a quad in the model's z = 0 plane (two triangles sharing the diagonal); `bend` tilts its per-vertex normals apart,
    so that the Lambert term varies across the triangles"""
    v = [[-half_w, -half_h, 0], [half_w, -half_h, 0], [half_w, half_h, 0], [-half_w, half_h, 0]]
    uv = np.array([[uv0, uv0], [uv1, uv0], [uv1, uv1], [uv0, uv1]], np.float32)
    n = np.array([[-bend, -bend, -1], [bend, -0.5 * bend, -1], [0.7 * bend, bend, -1], [-0.3 * bend, bend, -1]])
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    return _mesh(v, uv, [[0, 1, 2], [0, 2, 3]], tex, n, "quad")


def at_pixels(px, K, z):
    """camera-frame points (pose = identity) that project to pixel positions px [n,2] at depths z [n]"""
    fx, fy, cx, cy = [float(a) for a in (K[0, 0], K[1, 1], K[0, 2], K[1, 2])]
    px, z = np.asarray(px, np.float64), np.broadcast_to(np.asarray(z, np.float64), (len(px),))
    return np.stack([(px[:, 0] - cx) * z / fx, (px[:, 1] - cy) * z / fy, z], 1)


def tris_mesh(P, tex, seed=0, name="tris"):
    """unconnected triangles, three rows of P each, with random UVs in [-0.1, 1.1]"""
    n = len(P) // 3
    uv = np.random.RandomState(seed).uniform(-0.1, 1.1, (3 * n, 2)).astype(np.float32)
    return _mesh(P, uv, np.arange(3 * n).reshape(n, 3), tex, name=name)


def pose(R=None, t=(0, 0, 0)):
    p = np.zeros((3, 4))
    p[:, :3] = np.eye(3) if R is None else R
    p[:, 3] = t
    return p.astype(np.float32)


def rot(axis, deg):
    a = np.asarray(axis, np.float64)
    a /= np.linalg.norm(a)
    th = np.deg2rad(deg)
    Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


_MESHES = {}


def meshes():
    """the cube, the C2 blob (5k vertices) and the C5 blob (50k vertices), with normals; built once"""
    if not _MESHES:
        for k, m in (("cube", synth.make_cube()), ("c2", synth.make_blob()),
                     ("c5", synth.make_blob(nlat=158, nlon=316, seed=5, name="c5"))):
            m.normals = synth.vertex_normals(m)
            _MESHES[k] = m
    return _MESHES


def object_poses(n, view, seed):
    """n poses 0.4 ... 2 m deep whose centres project to within [-0.1, 1.1] of the frame (some partly out of it)"""
    H, W, K = VIEWS[view]
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        z = rs.uniform(0.4, 2.0)
        c = at_pixels([[rs.uniform(-0.1, 1.1) * W, rs.uniform(-0.1, 1.1) * H]], K, z)[0]
        out.append(pose(synth.random_rotation(rs), c))
    return out


# ----------------------------------------------------------------------------------------------------------- scenes
def geometry_scenes():
    """the hand-made scenes: quads, slivers, far vertices, near / far planes, overlaps, kernel-path edges"""
    T37, T1, TALL, WIDE = _tex(37, 53, 1), _tex(1, 1, 2), _tex(61, 5, 3), _tex(5, 61, 4)
    S = []
    for view, z0 in (("lm", 1.0), ("off", 0.5)):
        s = Scene("quads fronto-parallel", view)
        s.add(quad(0.12, 0.09, T37), pose(t=(0.02, -0.01, z0)))
        s.add(quad(0.05, 0.05, T1), pose(t=(-0.03, 0.03, z0 * 0.8)))
        s.add(quad(0.1, 0.1, WIDE, -0.25, 1.3), pose(t=(0.0, 0.0, z0 * 1.5)))
        S.append(s)
        s = Scene("quads tilted", view)
        # rotations about x, y and an oblique axis up to 85 degrees; z spans about 0.4 ... 4.5 m on the grazing ones
        s.add(quad(0.15, 0.15, T37, bend=0.4), pose(rot((1, 0, 0), 60), (0, 0, z0)))
        s.add(quad(0.2, 0.12, TALL, bend=0.6), pose(rot((0, 1, 0), 75), (0.02, 0, z0 * 1.2)))
        s.add(quad(2.0, 0.1, WIDE, -0.2, 1.2, bend=0.3), pose(rot((0, 1, 0), 85), (0, 0.02, 2.4)))
        s.add(quad(0.12, 2.1, T37, bend=0.5), pose(rot((1, 0.3, 0), 84), (0.01, 0, 2.45)))
        s.add(quad(0.1, 0.1, T1, bend=0.2), pose(rot((1, 1, 0.4), 50), (-0.02, 0.01, z0)))
        s.add(quad(0.3, 0.2, TALL, 0.0, 1.0, bend=0.5), pose(rot((0.3, 1, 0.2), -70), (0, 0, z0 * 1.6)))
        S.append(s)

    H, W, K = VIEWS["lm"]
    rs = np.random.RandomState(7)
    # slivers: a fan of 200 triangles under a pixel wide around one point, and long thin triangles across the frame
    ang = np.linspace(0, 2 * np.pi, 201)
    c = np.array([320.3, 240.6])
    fan = []
    for k in range(200):
        r = 150.0
        a0, a1 = ang[k], ang[k] + (ang[k + 1] - ang[k]) * 0.2
        fan += [c, c + r * np.array([np.cos(a0), np.sin(a0)]), c + r * np.array([np.cos(a1), np.sin(a1)])]
    long = []
    for k in range(12):
        y = 20 + 37.3 * k
        w = [0.3, 0.6, 1.2, 0.05][k % 4]
        long += [[-50.2, y], [700.3, y + 8.7 * (k % 3)], [-50.2, y + w]]
    s = Scene("slivers", "lm")
    s.add(tris_mesh(at_pixels(fan, K, rs.uniform(0.6, 1.0, 600)), _tex(37, 53, 5), 1), pose())
    s.add(tris_mesh(at_pixels(long, K, np.tile([0.7, 1.9, 1.2], 12)), _tex(61, 5, 6), 2), pose())
    S.append(s)

    # far vertices: one vertex at 1e3 ... 9e5 px off screen (drawn), and one beyond 1e6 px (the drop rule)
    s = Scene("far vertices", "lm")
    for k, far in enumerate((1e3, 1e4, 1e5, 9e5, 2e6)):
        y = 40 + 90 * k
        P = at_pixels([[300.2, y], [far, y + 30.5], [360.7, y + 70.3]], K, [0.8, 0.9, 1.1])
        s.add(tris_mesh(P, T37, 10 + k), pose())
    S.append(s)

    # near and far planes: a plane cut by zn and by zf, and a triangle with a vertex behind the camera (dropped)
    s = Scene("near / far planes", "lm")
    s.add(quad(0.5, 3.75, T37, bend=0.3), pose(rot((1, 0, 0), 88), (0, 0.1, 3.8)))  # z 0.05 ... 7.55 m
    P = np.array([[-0.3, -0.2, 0.8], [0.3, -0.1, 0.9], [0.0, 0.3, -0.5]])
    s.add(tris_mesh(P, T37, 20), pose())
    S.append(s)

    # overlaps: two interpenetrating quads; coplanar duplicates with different UVs (the lowest face index wins the tie)
    s = Scene("overlaps", "lm")
    q = quad(0.1, 0.1, T37, bend=0.2)
    R45 = rot((0, 1, 0), 45)
    both = _mesh(np.vstack([q.verts, q.verts @ R45.T + [0.01, 0.0, 0.0]]), np.vstack([q.uvs, q.uvs[::-1]]),
                 np.vstack([q.faces, q.faces + 4]), T37, np.vstack([q.normals, q.normals @ R45.T]), "crossing quads")
    s.add(both, pose(t=(0, 0, 1.0)))
    s.add(both, pose(rot((1, 0.2, 0), 35), (0.02, -0.01, 0.8)))
    dup = _mesh([[-0.1, -0.1, 0], [0.1, -0.08, 0.02], [0.0, 0.1, -0.03]] * 2,
                np.array([[0.1, 0.1], [0.2, 0.1], [0.1, 0.2], [0.8, 0.8], [0.9, 0.8], [0.8, 0.9]], np.float32),
                [[0, 1, 2], [3, 4, 5]], T37, name="dup")
    s.add(dup, pose(rot((1, 0.5, 0), 30), (0.0, 0.02, 0.9)))
    S.append(s)

    # kernel-path edges: F = 1, 127, 128, 129 and V = 31, 33 (partial blocks and warps of the vertex / coverage grids)
    s = Scene("face / vertex counts", "off")
    for k, F in enumerate((1, 127, 128, 129)):
        cen = np.array([[20 + 30 * k, 50.5]])
        P = at_pixels(cen + rs.uniform(-14, 14, (3 * F, 2)), K_OFF, rs.uniform(0.45, 0.6, 3 * F))
        s.add(tris_mesh(P, _tex(37, 53, 30 + k), 30 + k), pose())
    for k, V in enumerate((31, 33)):
        ang = np.linspace(0, 2 * np.pi, V - 1, endpoint=False)
        rim = np.stack([66 + 30 * np.cos(ang), 48 + 30 * np.sin(ang)], 1)
        P = at_pixels(np.vstack([[[66.3, 48.2]], rim]), K_OFF, np.r_[0.5, 0.55 + 0.1 * np.sin(3 * ang)])
        faces = [[0, 1 + a, 1 + (a + 1) % (V - 1)] for a in range(V - 1)]
        uv = np.random.RandomState(40 + k).uniform(0, 1, (V, 2)).astype(np.float32)
        s.add(_mesh(P, uv, faces, _tex(5, 61, 40 + k), name="fan%d" % V), pose(t=(0, 0, 0.1 * k)))
    S.append(s)

    # one warp of triangles whose screen boxes hold exactly 48 and 49 pixels, alternating
    s = Scene("48 / 49-pixel boxes", "lm")
    P = []
    for k in range(32):
        x0, y0 = 20.3 + 18 * (k % 16), 100.3 + 20 * (k // 16)
        w, h = (8, 6) if k % 2 == 0 else (7, 7)  # j0..j1 = x0 + 0.7 ... + w, i0..i1 likewise
        P += [[x0, y0], [x0 + w + 0.4, y0 + 0.5 * h], [x0 + 0.2 * w, y0 + h + 0.4]]
    s.add(tris_mesh(at_pixels(P, K, 0.7), T37, 50), pose())
    S.append(s)
    return S


def mesh_scenes():
    """the cube, the C2 and the C5 blob at 32 poses each: 8 in each view"""
    ms = meshes()
    S = []
    for v, view in enumerate(VIEWS):
        s = Scene("meshes", view)
        for k, name in enumerate(("cube", "c2", "c5")):
            for p in object_poses(8, view, 100 * v + k):
                s.add(ms[name], p, seed=k)
        S.append(s)
    return S


def batch16_scene():
    """B = max_batch = 16 mixing every mesh"""
    ms = meshes()
    s = Scene("B = 16 mixed", "lm")
    ps = object_poses(16, "lm", 999)
    for b in range(16):
        s.add(ms[("cube", "c2", "c5")[b % 3]], ps[b], seed=b)
    return s


def ownership_grid():
    """40 x 30 quads with vertices on pixel centres and half-pixels at depth 1, split along alternating diagonals, every
    triangle on its own texel: the pixel's owner shows in the colour.  Returns (Scene at 120 x 160 with the camera
    fx = fy = 256, cx = 16, cy = 12, which projects these vertices exactly, and the vertex positions in half-pixel
    units [F,3,2] int)."""
    K = np.array([[256.0, 0, 16.0], [0, 256.0, 12.0], [0, 0, 1]], np.float32)
    xs = 4 + 7 * np.arange(41)  # half-pixels: 2, 5.5, 9, ...
    ys = 4 + 7 * np.arange(31)
    tri2 = []
    for r in range(30):
        for c in range(40):
            a, b, d, e = (xs[c], ys[r]), (xs[c + 1], ys[r]), (xs[c + 1], ys[r + 1]), (xs[c], ys[r + 1])
            tri2 += [[a, b, d], [a, d, e]] if (r + c) % 2 == 0 else [[a, b, e], [b, d, e]]
    tri2 = np.array(tri2, np.int64)  # [2400,3,2] half-pixels
    F = len(tri2)
    Th, Tw = 48, 50
    idx = np.arange(Th * Tw)
    tex = np.stack([idx & 255, idx >> 8, np.full_like(idx, 77)], -1).reshape(Th, Tw, 3).astype(np.uint8)
    uv = np.stack([(np.arange(F) % Tw + 0.5) / Tw, (np.arange(F) // Tw + 0.5) / Th], -1)
    px = tri2.reshape(-1, 2) / 2.0
    P = np.stack([(px[:, 0] - 16.0) / 256.0, (px[:, 1] - 12.0) / 256.0, np.ones(len(px))], 1)
    m = _mesh(P, np.repeat(uv, 3, 0).astype(np.float32), np.arange(3 * F).reshape(F, 3), tex, name="grid")
    VIEWS["grid"] = (120, 160, K)
    s = Scene("ownership grid", "grid")
    s.add(m, pose())
    return s, tri2


def grid_owner(tri2, H, W):
    """[H,W] owning face of every pixel by the top-left-style rule on the exact geometry (-1 where none): the pixel centre
    is inside a (positively oriented) triangle, or on an edge a -> b with dy > 0 or (dy == 0 and dx < 0)"""
    owner = np.full((H, W), -1, np.int64)
    count = np.zeros((H, W), np.int64)
    yy, xx = np.mgrid[0:H, 0:W]
    px, py = 2 * xx, 2 * yy  # half-pixel units
    for f, t in enumerate(tri2):
        a, b, c = t
        if (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0]) < 0:
            b, c = c, b
        inside = np.ones((H, W), bool)
        for p, q in ((b, c), (c, a), (a, b)):
            w = (q[0] - p[0]) * (py - p[1]) - (q[1] - p[1]) * (px - p[0])
            dx, dy = q[0] - p[0], q[1] - p[1]
            owns = dy > 0 or (dy == 0 and dx < 0)
            inside &= (w > 0) | ((w == 0) & owns)
        owner[inside] = f
        count += inside
    assert count.max() <= 1, "the rule gives a pixel to two triangles"
    return owner
