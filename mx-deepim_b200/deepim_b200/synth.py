"""Synthetic inputs for the BASELINE.json configs (meshes, textures, poses, FlowNetS weights).

Nothing here is algorithm: it only manufactures *inputs* of the shapes SURVEY.md 8(d) names
(C1 cube ~500 tris, C2 ~5k-vert blob, C3 13 LINEMOD-scale meshes, C5 ~50k-vert stress mesh), the
pose-perturbation distribution of toolkit/LM6d_1_gen_rendered_pose.py:54,86-101 and random-init
weights with the parameter names/shapes of deepim/symbols/deepIM_flownet.py:63-116,716-717.
Both the product path and the oracle consume the same arrays.
"""
from __future__ import annotations

import numpy as np

# deepim/config/config.py:58-60, experiments/deepim/cfgs/*.yaml:57-59
K_LINEMOD = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]], dtype=np.float32)
ZNEAR, ZFAR = 0.25, 6.0
HEIGHT, WIDTH = 480, 640
PIXEL_MEANS = np.array([123.68, 116.779, 103.939], dtype=np.float64)  # yaml order (python floats)
# channel c of the network blob (R,G,B) is paired with PIXEL_MEANS[2-c] (lib/utils/image.py:592-593)
PIXEL_MEANS_RGB = PIXEL_MEANS[::-1].copy()


class Mesh:
    """verts [V,3] f32 (metres), faces [F,3] i32 and one colour source: a texture, uvs [V,2] f32 with tex [Th,Tw,3] u8
    (row 0 = v 0), or per-vertex colours [V,3] f32 RGB in [0,1] (uvs = tex = None), never both."""

    def __init__(self, verts, uvs, faces, tex, name="mesh", colours=None):
        if colours is None and (uvs is None or tex is None):
            raise ValueError("Mesh: give uvs and tex, or colours")
        if colours is not None and (uvs is not None or tex is not None):
            raise ValueError("Mesh: a mesh has uvs and tex or colours, never both")
        self.verts = np.ascontiguousarray(verts, dtype=np.float32)
        self.uvs = None if uvs is None else np.ascontiguousarray(uvs, dtype=np.float32)
        self.faces = np.ascontiguousarray(faces, dtype=np.int32)
        self.tex = None if tex is None else np.ascontiguousarray(tex, dtype=np.uint8)
        self.colours = None if colours is None else np.ascontiguousarray(colours, dtype=np.float32).reshape(-1, 3)
        self.name = name

    @property
    def diameter(self) -> float:
        # lib/utils/misc.py:56-73 calc_pts_diameter (max pairwise distance); subsample for big meshes
        p = self.verts
        if len(p) > 2000:
            p = p[:: max(1, len(p) // 2000)]
        d = np.linalg.norm(p[:, None, :] - p[None, :, :], axis=2)
        return float(d.max())


def make_texture(size: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:size, 0:size]
    cells = 16
    checker = (((yy * cells) // size + (xx * cells) // size) % 2).astype(np.float32)
    base = rng.uniform(40, 215, size=(cells, cells, 3)).astype(np.float32)
    tile = base[(yy * cells) // size, (xx * cells) // size]
    noise = rng.uniform(-30, 30, size=(size, size, 3)).astype(np.float32)
    tex = tile * (0.6 + 0.4 * checker[..., None]) + noise
    return np.clip(tex, 0, 255).astype(np.uint8)


def make_cube(side: float = 0.1, nu: int = 6, nv: int = 7, tex_size: int = 256, seed: int = 0) -> Mesh:
    """C1: cube, 6 faces x (nu*nv*2 = 84) = 504 triangles, 3x2 UV atlas."""
    h = side / 2.0
    verts, uvs, faces = [], [], []
    # (origin, du, dv) for each face, outward orientation not required (no culling in the reference)
    frames = [
        ((-h, -h, h), (side, 0, 0), (0, side, 0)),
        ((h, -h, -h), (-side, 0, 0), (0, side, 0)),
        ((h, -h, h), (0, 0, -side), (0, side, 0)),
        ((-h, -h, -h), (0, 0, side), (0, side, 0)),
        ((-h, h, h), (side, 0, 0), (0, 0, -side)),
        ((-h, -h, -h), (side, 0, 0), (0, 0, side)),
    ]
    for fi, (o, du, dv) in enumerate(frames):
        o, du, dv = np.array(o), np.array(du), np.array(dv)
        base = len(verts)
        au, av = fi % 3, fi // 3
        for j in range(nv + 1):
            for i in range(nu + 1):
                s, t = i / nu, j / nv
                verts.append(o + s * du + t * dv)
                uvs.append(((au + 0.02 + 0.96 * s) / 3.0, (av + 0.02 + 0.96 * t) / 2.0))
        for j in range(nv):
            for i in range(nu):
                a = base + j * (nu + 1) + i
                b, c, d = a + 1, a + nu + 1, a + nu + 2
                faces.append((a, b, d))
                faces.append((a, d, c))
    return Mesh(np.array(verts), np.array(uvs), np.array(faces), make_texture(tex_size, seed + 100), "cube")


def make_blob(nlat: int = 50, nlon: int = 100, diameter: float = 0.10, tex_size: int = 512, seed: int = 1,
              name: str = "blob") -> Mesh:
    """Asymmetric star-shaped blob on a lat/lon grid: (nlat+1)(nlon+1) verts, 2*nlat*nlon tris.
    50x100 -> 5151 verts / 10000 tris (C2, ape scale); 158x316 -> 50403 verts / 99856 tris (C5)."""
    rng = np.random.default_rng(seed)
    lat = np.linspace(0.0, np.pi, nlat + 1)
    lon = np.linspace(0.0, 2 * np.pi, nlon + 1)
    LON, LAT = np.meshgrid(lon, lat)
    d = np.stack([np.sin(LAT) * np.cos(LON), np.sin(LAT) * np.sin(LON), np.cos(LAT)], axis=-1)
    r = np.ones_like(LAT)
    for _ in range(6):  # low-frequency lobes, periodic in lon by construction
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        amp = rng.uniform(0.05, 0.18)
        k = rng.integers(1, 4)
        r += amp * np.cos(k * np.arccos(np.clip(d @ axis, -1, 1)) + rng.uniform(0, 2 * np.pi))
    r = np.clip(r, 0.35, None)
    scale = np.array([1.0, rng.uniform(0.6, 0.9), rng.uniform(0.5, 0.8)])
    P = d * r[..., None] * scale
    P = P.reshape(-1, 3)
    P -= P.mean(axis=0)
    sub = P[:: max(1, len(P) // 1500)]
    diam = np.linalg.norm(sub[:, None] - sub[None], axis=2).max()
    P *= diameter / diam
    uv = np.stack([LON / (2 * np.pi), LAT / np.pi], axis=-1).reshape(-1, 2)
    faces = []
    for i in range(nlat):
        row = i * (nlon + 1)
        for j in range(nlon):
            a = row + j
            b, c, e = a + 1, a + nlon + 1, a + nlon + 2
            faces.append((a, c, b))
            faces.append((b, c, e))
    return Mesh(P, uv, np.array(faces), make_texture(tex_size, seed + 200), name)


def make_linemod_like_set(n: int = 13, seed: int = 2):
    """C3: 13 meshes, vert counts spread 5k-20k, diameters 0.10-0.28 m."""
    rng = np.random.default_rng(seed)
    meshes = []
    for k in range(n):
        nlat = int(50 + (k / max(1, n - 1)) * 50)
        meshes.append(make_blob(nlat, 2 * nlat, diameter=float(rng.uniform(0.10, 0.28)), tex_size=512,
                                seed=seed * 100 + k, name="obj%02d" % k))
    return meshes


def vertex_normals(mesh) -> np.ndarray:
    """Area-weighted per-vertex normals [V,3] float32 (what an OBJ exporter writes as `vn`; the lit renderer reads them
    through glumpy's objload, render_py_light_modelnet_multi.py:99-101)."""
    v, f = mesh.verts.astype(np.float64), mesh.faces
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    n = np.zeros_like(v)
    for k in range(3):
        np.add.at(n, f[:, k], fn)
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    return (n / np.maximum(ln, 1e-20)).astype(np.float32)


def euler_to_mat(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def random_rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def sample_pose_pairs(n: int, seed: int, z_mean: float = 0.8, K=K_LINEMOD):
    """(pose_observed, pose_init) pairs [n,3,4] float64.
    Observed: t = (U(-.05,.05), U(-.05,.05), z_mean), R uniform.  Init = observed perturbed as in
    toolkit/LM6d_1_gen_rendered_pose.py:54,86-101: euler N(0,15deg)/axis, reject >45deg;
    x,y N(0,.01 m), z N(0,.05 m); projected centre kept 16 px inside the frame."""
    rng = np.random.default_rng(seed)
    obs = np.zeros((n, 3, 4))
    ini = np.zeros((n, 3, 4))
    for k in range(n):
        R = random_rotation(rng)
        t = np.array([rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05), z_mean])
        obs[k, :, :3], obs[k, :, 3] = R, t
        while True:
            ang = rng.normal(0, 15.0, size=3)
            if np.any(np.abs(ang) > 45.0):
                continue
            dt = np.array([rng.normal(0, 0.01), rng.normal(0, 0.01), rng.normal(0, 0.05)])
            t2 = t + dt
            c = K.astype(np.float64) @ t2
            cx, cy = c[0] / c[2], c[1] / c[2]
            if 16 < cx < WIDTH - 16 and 16 < cy < HEIGHT - 16 and t2[2] > 0.4:
                break
        ini[k, :, :3] = euler_to_mat(*np.deg2rad(ang)) @ R
        ini[k, :, 3] = t2
    return obs, ini


# ---------------------------------------------------------------------------------------------
# FlowNetS (deepIM_flownet.py:63-116) + heads (l.716-717): name, (Cout, Cin, k, stride, pad)
CONV_SPECS = [
    ("flow_conv1", 64, 8, 7, 2, 3),
    ("conv2", 128, 64, 5, 2, 2),
    ("conv3", 256, 128, 5, 2, 2),
    ("conv3_1", 256, 256, 3, 1, 1),
    ("conv4", 512, 256, 3, 2, 1),
    ("conv4_1", 512, 512, 3, 1, 1),
    ("conv5", 512, 512, 3, 2, 1),
    ("conv5_1", 512, 512, 3, 1, 1),
    ("conv6", 1024, 512, 3, 2, 1),
    ("conv6_1", 1024, 1024, 3, 1, 1),
]
FC_SPECS = [("fc6", 256, 1024 * 8 * 10), ("fc7", 256, 256), ("rot", 4, 256), ("trans", 3, 256)]


def conv_out_hw(h, w, k, s, p):
    return (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1


def with_depth_channels(weights: dict, depth_weight=None):
    """An 8-channel weight set as the RGB-D network's (config.network.INPUT_DEPTH): flow_conv1_weight (64, 8, 7, 7) ->
    (64, 10, 7, 7) with the depth columns (channels 6, 7: depth_observed, depth_rendered) inserted before the two mask
    channels; depth_weight (64, 2, 7, 7), zeros when None (the network then computes what the RGB one does)."""
    w = dict(weights)
    c1 = np.asarray(weights["flow_conv1_weight"], np.float32)
    d = np.zeros((c1.shape[0], 2) + c1.shape[2:], np.float32) if depth_weight is None else np.asarray(depth_weight, np.float32)
    w["flow_conv1_weight"] = np.ascontiguousarray(np.concatenate([c1[:, :6], d, c1[:, 6:]], axis=1))
    return w


def make_weights(seed: int = 0, input_depth: bool = False):
    """Random-init weights (dict name -> float32 array) with MXNet shapes
    (Convolution (Cout,Cin,kh,kw); FullyConnected (out,in), SURVEY App.B-22).
    He-normal convs (LeakyReLU 0.1 gain), small random biases, Xavier fc6/fc7; rot head biased to
    an identity-ish quaternion (cf. init_weights deepIM_flownet.py:793-800) with a non-degenerate
    small random part so the regressed SE(3) delta actually moves the pose."""
    rng = np.random.default_rng(seed)
    w = {}
    gain = np.sqrt(2.0 / (1.0 + 0.1 ** 2))
    for name, co, ci, k, s, p in CONV_SPECS:
        std = gain / np.sqrt(ci * k * k)
        w[name + "_weight"] = (rng.standard_normal((co, ci, k, k), dtype=np.float32) * np.float32(std))
        w[name + "_bias"] = (rng.standard_normal((co,), dtype=np.float32) * np.float32(0.02))
    for name, co, ci in FC_SPECS:
        if name in ("fc6", "fc7"):
            std = np.sqrt(2.0 / (ci + co))
        elif name == "rot":
            std = 0.02 / np.sqrt(ci)
        else:
            std = 0.01 / np.sqrt(ci)
        w[name + "_weight"] = (rng.standard_normal((co, ci), dtype=np.float32) * np.float32(std))
        w[name + "_bias"] = np.zeros((co,), dtype=np.float32)
    w["fc6_bias"] = (rng.standard_normal((256,), dtype=np.float32) * np.float32(0.02))
    w["fc7_bias"] = (rng.standard_normal((256,), dtype=np.float32) * np.float32(0.02))
    w["rot_bias"] = np.array([1.0, 0.02, -0.03, 0.015], dtype=np.float32)
    w["trans_bias"] = np.array([0.01, -0.015, 0.02], dtype=np.float32)
    if input_depth:  # the 8-channel set plus He-normal depth columns (fan-in of the 10-channel conv1) from a separate stream
        drng = np.random.default_rng(seed + 7919)
        std = gain / np.sqrt(10 * 7 * 7)
        w = with_depth_channels(w, drng.standard_normal((64, 2, 7, 7), dtype=np.float32) * np.float32(std))
    return w


DECODER_SPECS = [  # name, kind, weight shape (MXNet layouts: conv (Cout,Cin,k,k); deconv (Cin,Cout,k,k)), bias length
    ("Convolution1", "conv", (2, 1024, 3, 3), 2), ("deconv5", "deconv", (1024, 512, 4, 4), 512),
    ("upsample_flow6to5", "deconv", (2, 2, 4, 4), 2), ("Convolution2", "conv", (2, 1026, 3, 3), 2),
    ("deconv4", "deconv", (1026, 256, 4, 4), 256), ("upsample_flow5to4", "deconv", (2, 2, 4, 4), 2),
    ("Convolution3", "conv", (2, 770, 3, 3), 2), ("mask_conv3", "conv", (1, 770, 3, 3), 1),
]


def bilinear_upsampling_kernel(k: int = 32) -> np.ndarray:
    """mx.init.Initializer._init_bilinear as called by init_weights (deepIM_flownet.py:806-820)."""
    f = np.ceil(k / 2.0)
    c = (2 * f - 1 - f % 2) / (2.0 * f)
    v = 1 - np.abs(np.arange(k) / f - c)
    return np.outer(v, v).astype(np.float32)


def make_train_weights(seed: int = 0, input_depth: bool = False, input_mask: bool = True):
    """make_weights + the train-only decoder / flow / mask heads (deepIM_flownet.py:121-167,176-193,317-338):
    He-normal decoder convs/deconvs (a k4 s2 deconv sums Cin*4 taps per output), N(0, 0.01) mask_conv3
    (init_weights l.811-813), frozen bilinear `upsampling` (2 groups) / `mask_upsampling` kernels.
    input_mask=False: the image-only network, make_weights' flow_conv1 without its two mask columns (64, 6, 7, 7)."""
    if input_depth and not input_mask:
        raise ValueError("input_depth with input_mask=False is not supported")
    w = make_weights(seed, input_depth)
    if not input_mask:
        w["flow_conv1_weight"] = np.ascontiguousarray(w["flow_conv1_weight"][:, :6])
    rng = np.random.default_rng(seed + 1000003)
    gain = np.sqrt(2.0 / (1.0 + 0.1 ** 2))
    for name, kind, shp, nb in DECODER_SPECS:
        fan = shp[1] * shp[2] * shp[3] if kind == "conv" else shp[0] * (shp[2] // 2) * (shp[3] // 2)
        std = 0.01 if name == "mask_conv3" else (gain if name.startswith("deconv") else 1.0) / np.sqrt(fan)
        w[name + "_weight"] = rng.standard_normal(shp, dtype=np.float32) * np.float32(std)
        w[name + "_bias"] = rng.standard_normal((nb,), dtype=np.float32) * np.float32(0.02)
    bk = bilinear_upsampling_kernel(32)
    w["upsampling_weight"] = np.ascontiguousarray(np.broadcast_to(bk, (2, 1, 32, 32))).copy()
    w["mask_upsampling_weight"] = bk.reshape(1, 1, 32, 32).copy()
    return w


def composite_observed(bgr_render: np.ndarray, mask: np.ndarray, seed: int) -> np.ndarray:
    """observed image = render composited over uniform-noise background, uint8 BGR [H,W,3]
    (what cv2.imread hands the reference's loader)."""
    rng = np.random.default_rng(seed)
    bg = rng.integers(0, 256, size=bgr_render.shape, dtype=np.uint8)
    out = np.where(mask[..., None] > 0, bgr_render.astype(np.uint8), bg)
    return np.ascontiguousarray(out)


def transform_image(bgr_u8_or_f: np.ndarray) -> np.ndarray:
    """lib/utils/image.py:583-594: [H,W,3] BGR -> [3,H,W] float32 RGB minus PIXEL_MEANS_RGB."""
    im = bgr_u8_or_f.astype(np.float64)
    out = np.empty((3,) + im.shape[:2], dtype=np.float32)
    for c in range(3):
        out[c] = (im[:, :, 2 - c] - PIXEL_MEANS_RGB[c]).astype(np.float32)
    return out
