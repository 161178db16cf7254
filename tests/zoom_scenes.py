"""Inputs of the zoom tests (tests/test_zoom_float64.py, tests/test_gpu_zoom_float64.py): frame sizes, images, affines and
box scenes built to hit the sampler's and the zoom factor's edges, each with the case it claims to be, and the float32
coordinate chain of zoom_gather_kernel (for the claims and for the known-answer test of tests/zoom_ref.py's bound)."""
import numpy as np

F32 = np.float32
# 480 x 640; odd H with H W = 5124 (not a multiple of the 256-thread block); H W = 22360 (neither)
SIZES = [(480, 640), (61, 84), (130, 172)]
MEANS = np.array([123.68, 116.779, 103.939], F32)  # synth.PIXEL_MEANS_RGB


def chain_f32(w, t, N):
    """the device's float32 source coordinate of output indices 0 ... N-1 (zoom.cu src_coord, -fmad=false)"""
    step = F32(2.0 / (N - 1))
    o = np.arange(N).astype(F32)
    xt = F32(-1.0) + o * step
    xs = F32(w) * xt + F32(t)
    return ((xs + F32(1.0)) * F32(N - 1)) / F32(2.0)


def images(H, W, seed=0):
    """[H, W] float32 planes: noise, steps, a smooth field and a constant"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    return {
        "noise": rng.uniform(0, 255, (H, W)).astype(F32),
        "steps": (255.0 * (((xx // 7) + (yy // 5)) % 2)).astype(F32),
        "smooth": (127.5 + 100 * np.sin(xx / 13.0) * np.cos(yy / 9.0)).astype(F32),
        "constant": np.full((H, W), 77.0, F32),
    }


def affines(H, W):
    """(name, float32 [wx, wy, tx, ty]) zoom factors"""
    a = [("identity", [1, 1, 0, 0]),
         ("integer shift", [1, 1, 3 * 2.0 / (W - 1), -2 * 2.0 / (H - 1)]),
         ("half-pixel shift", [1, 1, 1.0 / (W - 1), 1.0 / (H - 1)]),
         ("x25", [0.04, 0.04, 0.013, -0.021]),
         ("x500 near a corner", [0.002, 0.002, 0.97, -0.99]),
         ("crop 2.5x", [2.5, 2.5, 0.3, -0.2]),
         ("crop 5x, centre off the frame", [5, 5, 1.7, -1.3]),
         ("centre off the frame", [0.3, 0.3, 1.3, -1.2])]
    return [(n, np.array(v, F32)) for n, v in a]


def assert_affine_claims(H, W):
    """the affines are the cases they claim: magnification >= 20, crops 2x to 5x, a centre off the frame, taps beyond the
    +-4 clamp, and float32 coordinates landing exactly on integers and on W - 1 / H - 1"""
    A = dict(affines(H, W))
    assert 1 / A["x25"][0] >= 20 and 1 / A["x500 near a corner"][0] >= 400
    assert A["crop 2.5x"][0] == 2.5 and A["crop 5x, centre off the frame"][0] == 5
    for n in ("crop 5x, centre off the frame", "centre off the frame"):
        assert abs(A[n][2]) > 1 and abs(A[n][3]) > 1
    for n in ("crop 2.5x", "crop 5x, centre off the frame"):
        x = chain_f32(A[n][0], A[n][2], W)
        assert x.min() < -4 and x.max() > W + 4, n
    last = []
    for w, t, N in ((A["identity"][0], A["identity"][2], W), (A["identity"][1], A["identity"][3], H)):
        x = chain_f32(w, t, N)
        assert (x == np.round(x)).mean() > 0.3
        last.append(x[-1] == N - 1)
    assert any(last)
    x = chain_f32(A["integer shift"][0], A["integer shift"][2], W)
    assert (x == np.round(x)).any()


def camera(H, W):
    """a float32 K for an H x W frame (focal length 1.2 W, principal point off the centre)"""
    return np.array([[1.2 * W, 0, W / 2 + 0.3], [0, 1.2 * W, H / 2 - 0.2], [0, 0, 1]], F32)


def _pose(t):
    p = np.zeros((3, 4), F32)
    p[:, :3] = np.eye(3)
    p[:, 3] = t
    return p


def _rect(H, W, x0, x1, y0, y1, value=1.0):
    m = np.zeros((H, W), F32)
    m[y0:y1 + 1, x0:x1 + 1] = value
    return m


def mask_scenes(H, W, seed=1):
    """ZoomMask inputs: (name, mask_observed, mask_gt_observed, mask_rendered, src_pose) with [H, W] float32 masks.
    mask_observed is soft (values in [0, 1]: round matters), mask_rendered depth-like with values at and around 0.2 (the
    binarisation is strict), the gt mask 0 / 1."""
    rng = np.random.default_rng(seed)
    K = camera(H, W)
    cx, cy = float(K[0, 2]), float(K[1, 2])

    def ren_like(m):
        d = np.where(m > 0, rng.uniform(0.1, 1.5, m.shape), 0.0).astype(F32)
        d[m > 0] = np.where(rng.random(int((m > 0).sum())) < 0.1, F32(0.2), d[m > 0])  # exactly float32(0.2): not > 0.2
        return d

    def soft(m):
        return (m * rng.uniform(0, 1, m.shape)).astype(F32)

    def centre_at(u, v, z=1.0):
        return _pose(((u - cx) * z / K[0, 0], (v - cy) * z / K[1, 1], z))

    q = lambda f, N: int(f * (N - 1))
    s = []
    g = _rect(H, W, 0, q(0.3, W), 0, q(0.4, H))
    s.append(("observed box on the left and top borders", soft(g), g, ren_like(_rect(H, W, 3, q(0.35, W), 2, q(0.3, H))),
              centre_at(q(0.15, W), q(0.2, H))))
    g = _rect(H, W, q(0.6, W), W - 1, q(0.7, H), H - 1)
    s.append(("observed box on the right and bottom borders", soft(g), g,
              ren_like(_rect(H, W, q(0.5, W), W - 2, q(0.6, H), H - 2)), centre_at(q(0.8, W), q(0.85, H))))
    g = _rect(H, W, q(0.5, W), q(0.5, W), q(0.5, H), q(0.5, H))
    s.append(("one-pixel boxes, magnification >= 20", g.copy(), g, ren_like(g), centre_at(q(0.5, W) + 0.25, q(0.5, H) - 0.4)))
    g = _rect(H, W, q(0.2, W), q(0.7, W), q(0.3, H), q(0.3, H))
    s.append(("one-row observed box", soft(g), g, ren_like(_rect(H, W, q(0.25, W), q(0.6, W), q(0.3, H), q(0.31, H))),
              centre_at(q(0.45, W), q(0.3, H))))
    g = _rect(H, W, q(0.4, W), q(0.6, W), q(0.4, H), q(0.6, H))
    s.append(("empty render: the observed box's centre", soft(g), g, np.zeros((H, W), F32), centre_at(q(0.5, W), q(0.5, H))))
    g = _rect(H, W, 0, W - 1, 0, H - 1)
    s.append(("full frame, centre off the frame: crop > 2x", soft(g), g, ren_like(g), centre_at(-0.4 * W, 1.3 * H)))
    r = _rect(H, W, q(0.05, W), q(0.95, W), q(0.05, H), q(0.95, H))
    s.append(("centre near a corner: crop 2x to 3x", soft(r), r, ren_like(r), centre_at(2.0, 1.5)))
    g = np.zeros((H, W), F32)
    s.append(("empty observed mask", g, g, ren_like(r), centre_at(q(0.5, W), q(0.5, H))))
    return s


def image_scenes(H, W, seed=2):
    """ZoomImage inputs: (name, image_observed, image_rendered, src_pose) with [3, H, W] float32 images holding
    colour - mean; the background is 0 - mean, so that sum_c(image + mean) is 0 there"""
    rng = np.random.default_rng(seed)
    K = camera(H, W)
    cx, cy = float(K[0, 2]), float(K[1, 2])

    def img(x0, x1, y0, y1, black_share=0.0):
        c = np.zeros((3, H, W), F32)
        c[:, y0:y1 + 1, x0:x1 + 1] = rng.integers(0, 256, (3, y1 - y0 + 1, x1 - x0 + 1))
        c[:, rng.random((H, W)) < black_share] = 0
        return (c - MEANS[:, None, None]).astype(F32)

    q = lambda f, N: int(f * (N - 1))
    pose = lambda u, v: _pose(((u - cx) / K[0, 0], (v - cy) / K[1, 1], 1.0))
    return [
        ("boxes on all borders", img(0, W - 1, 0, H - 1, 0.2), img(q(0.1, W), q(0.9, W), q(0.2, H), q(0.8, H)),
         pose(q(0.5, W), q(0.5, H))),
        ("one-pixel boxes", img(q(0.3, W), q(0.3, W), q(0.6, H), q(0.6, H)), img(q(0.31, W), q(0.31, W), q(0.6, H), q(0.6, H)),
         pose(q(0.3, W), q(0.6, H))),
        ("empty render", img(q(0.2, W), q(0.6, W), q(0.1, H), q(0.5, H)), (np.zeros((3, H, W), F32) - MEANS[:, None, None]),
         pose(q(0.4, W), q(0.3, H))),
    ]


def _boxes_and_factor(real_valid, ren_valid, pose, H, W):
    import zoom_ref as Z
    real, ren = Z.box(real_valid), Z.box(ren_valid)
    return real, ren, Z.zoom_factor_range(real, ren, pose[:, 3], camera(H, W), H, W)


def assert_mask_scene_claims(H, W):
    """each mask scene is the case its name claims, by the float64 reference's boxes and zoom factor range"""
    import zoom_ref as Z
    got = {}
    for name, mo, mg, mr, pose in mask_scenes(H, W):
        got[name] = _boxes_and_factor(Z.mask_valid(mg[None], False)[0], Z.mask_valid(mr[None], True)[0], pose, H, W)
    real, _, _ = got["observed box on the left and top borders"]
    assert real[0] == 0 and real[2] == 0
    real, _, _ = got["observed box on the right and bottom borders"]
    assert real[1] == W - 1 and real[3] == H - 1
    real, ren, (lo, hi) = got["one-pixel boxes, magnification >= 20"]
    assert real[0] == real[1] and real[2] == real[3] and ren[0] == ren[1] and 1 / hi[0] >= 20
    real, _, _ = got["one-row observed box"]
    assert real[2] == real[3] and real[0] < real[1]
    _, ren, rng = got["empty render: the observed box's centre"]
    assert ren[1] < 0 and rng is not None
    _, _, (lo, hi) = got["full frame, centre off the frame: crop > 2x"]
    assert lo[0] > 2 and (lo[2] > 1 or hi[2] < -1) and (lo[3] > 1 or hi[3] < -1)
    _, _, (lo, hi) = got["centre near a corner: crop 2x to 3x"]
    assert 2 < lo[0] and hi[0] < 3
    assert got["empty observed mask"][2] is None


def assert_image_scene_claims(H, W):
    """each image scene is the case its name claims (no pixel of these scenes is near the 0.01 threshold)"""
    import zoom_ref as Z
    got = {}
    for name, io, ir, pose in image_scenes(H, W):
        (vo, ao), (vr, ar) = Z.image_valid(io, MEANS), Z.image_valid(ir, MEANS)
        assert not ao.any() and not ar.any()
        got[name] = _boxes_and_factor(vo, vr, pose, H, W)
    assert list(got["boxes on all borders"][0]) == [0, W - 1, 0, H - 1]
    real, ren, (lo, hi) = got["one-pixel boxes"]
    assert real[0] == real[1] and real[2] == real[3] and ren[0] == ren[1] and ren[2] == ren[3] and 1 / hi[0] >= 20
    assert got["empty render"][1][1] < 0
