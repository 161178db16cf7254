"""GPU: the front of the fused refinement loop, stage by stage, against the oracle's primitives -- the render into the
box-only ren4 image, the boxes, zoom factor and status bits, and conv1's space-to-depth input written by
zoom_fused_nhwc8_kernel -- held bit for bit, then se3 against float64 fc6 -> fc7 -> heads from the loop's own act[10].

Every network (mask, RGB-D, image-only), unlit and lit, in fp16 / bf16 / bf16x3, on one B = 16 scene built to hit the edges:
objects cut by each border and a corner, a crop wider than the frame, an object straddling the near plane, one-column and
one-row renders (the end-exclusive observed rectangle is empty), an object out of view, a bad and an absent class, a black
object and a 2 x 2 pixel render.  Also: a stale ren4 left by a larger render, a smaller batch on the same context, frames
from several cameras, and conv1's input as dim_net_fwd and the training step pack it.

The expectations are built from the oracle's primitives rather than oracle.refine, which raises where the reference raises:
where the observed box is empty the device flags status bit 0, zooms every plane with the factor (1, 1, 0, 0) and has an
empty observed box (lane 6 all zero)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

import kernel_ref as R  # noqa: E402
from kernel_ref import s2d_decode  # noqa: E402
from oracle import oracle as O  # noqa: E402
from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import lighting, synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.trainer import Trainer  # noqa: E402

K = synth.K_LINEMOD
MEANS = synth.PIXEL_MEANS_RGB
DEV = torch.device("cuda", 0)
H, W = 480, 640
B = 16
ZN, ZF = 0.25, 6.0
MAX_CLASSES = 6
CUBE, BLOB, BLACK, SMALL, BIG, ABSENT, BAD = 0, 1, 2, 3, 4, 5, 6  # ABSENT: no mesh uploaded; BAD: >= max_classes
PREC = {"fp16": capi.PREC_FP16, "bf16": capi.PREC_BF16, "bf16x3": capi.PREC_BF16X3}
NETS = ("mask", "rgbd", "image")

E = synth.euler_to_mat


def pose(R3, t):
    p = np.zeros((3, 4))
    p[:, :3], p[:, 3] = R3, t
    return p


CENTRED = pose(E(0.4, -0.3, 0.2), (0.01, 0.0, 0.8))
# (name, class, pose): fixed poses; the scene fixture asserts that each is the case it claims to be
SCENE = [
    # z such that the float64 pose and its float32 cast give lights one ulp apart, and the lit render differs in a pixel
    ("centred cube", CUBE, pose(E(0.3, 0.5, 0.2), (0.0, 0.0, 0.803400003))),
    ("centred blob", BLOB, pose(E(-0.2, 0.4, 0.1), (0.02, 0.01, 0.7))),
    ("cut left", CUBE, pose(E(0.1, 0.7, 0.3), (-0.44, 0.0, 0.8))),
    ("cut right", BLOB, pose(E(0.2, 0.1, 0.5), (0.44, 0.02, 0.8))),
    ("cut top", CUBE, pose(E(0.5, 0.2, 0.1), (0.05, -0.33, 0.8))),
    ("cut bottom", BLOB, pose(E(0.3, 0.3, 0.3), (-0.05, 0.33, 0.8))),
    ("cut corner", CUBE, pose(E(0.2, 0.2, 0.6), (0.44, 0.33, 0.8))),
    ("near, crop wider than the frame", BIG, pose(E(0.3, 0.4, 0.2), (-0.15, -0.1, 0.45))),
    ("straddles the near plane", BIG, pose(E(0.6, 0.7, 0.3), (0.0, 0.0, 0.2))),
    ("one column", SMALL, pose(np.eye(3), (0.4455, 0.0, 0.8))),
    ("one row", SMALL, pose(np.eye(3), (0.0, 0.0, 3.5))),
    ("out of view", CUBE, pose(np.eye(3), (3.0, 0.0, 0.8))),
    ("class >= max_classes", BAD, CENTRED),
    ("class without a mesh", ABSENT, CENTRED),
    ("black cube", BLACK, pose(E(0.1, 0.2, 0.3), (-0.03, 0.02, 0.75))),
    ("2 x 2 pixels", SMALL, pose(np.eye(3), (0.0, 0.0, 3.0))),
]
IDX = {name: b for b, (name, _, _) in enumerate(SCENE)}
FALLBACK = [IDX["one column"], IDX["one row"], IDX["out of view"], IDX["class >= max_classes"], IDX["class without a mesh"]]
LIT = {"intensity": lighting.sample_intensity(np.random.default_rng(8), (1, B)), "offset": lighting.OFFSET,
       "brightness_ratio": 0.7}


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def rnd(a, prec):
    """conv1's 16-bit storage: fp16, or bf16 round to nearest even"""
    if prec == "fp16":
        return a.astype(np.float16).astype(np.float32)
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).bfloat16().float().numpy()


@pytest.fixture(scope="module")
def meshes():
    return build_meshes()


def build_meshes():
    black = synth.make_cube()
    black.tex = np.zeros_like(black.tex)
    ms = {CUBE: synth.make_cube(), BLOB: synth.make_blob(), BLACK: black,
          SMALL: synth.make_cube(side=0.01, nu=1, nv=1, tex_size=16, seed=3),
          BIG: synth.make_cube(side=0.3, nu=2, nv=2, tex_size=64, seed=4)}
    for m in ms.values():
        m.normals = synth.vertex_normals(m)
    return ms


@pytest.fixture(scope="module")
def weights():
    return {"mask": synth.make_weights(0), "rgbd": synth.make_weights(0, input_depth=True),
            "image": synth.make_train_weights(0, input_mask=False)}


def make_ctx(meshes, weights, net, max_batch=B):
    c = Context(0, max_batch=max_batch, max_classes=MAX_CLASSES, max_verts=6000, max_faces=11000,
                input_depth=net == "rgbd", input_mask=net != "image")
    for i, m in meshes.items():
        c.upload_mesh(i, m)
    c.load_weights(weights[net])
    return c


@pytest.fixture(scope="module")
def ctxs(meshes, weights):
    cs = {net: make_ctx(meshes, weights, net) for net in NETS}
    yield cs
    for c in cs.values():
        c.close()


def render(meshes, cls, p, Kb, lit_intensity=None, want=("image", "depth", "mask")):
    """the loop's render of one instance; a class without a mesh renders nothing (the cube out of view)"""
    if cls not in meshes:
        return O.render(meshes[CUBE], pose(np.eye(3), (100.0, 0.0, 1.0)), Kb, ZN, ZF, H, W, MEANS, True, want=want)
    if lit_intensity is None:
        return O.render(meshes[cls], p, Kb, ZN, ZF, H, W, MEANS, True, want=want)
    return O._render_lit(meshes[cls], p, Kb, lit_intensity, LIT, ZN, ZF, H, W, MEANS, want)


@pytest.fixture(scope="module")
def scene(meshes):
    return build_scene(meshes)


def build_scene(meshes):
    """poses, classes and the observed frames: renders at the observed pose composited over noise (mask and RGB-D networks)
    and on black (image-only network: the observed box is the object's own, cut ones included), a sensor-like depth.  An
    instance that renders nothing observes the centred cube, so the image-only network sees its observed box."""
    poses = np.stack([p for _, _, p in SCENE])
    cls = np.array([c for _, c, _ in SCENE], np.int32)
    obs_cls = np.where(np.isin(cls, [BLACK, ABSENT, BAD]), CUBE, cls)
    obs_pose = poses.copy()
    obs_pose[IDX["out of view"]] = CENTRED
    rng = np.random.default_rng(17)
    noise, black, depth = [], [], []
    for b in range(B):
        r = O.render(meshes[obs_cls[b]], obs_pose[b], K, means_rgb=MEANS)
        noise.append(synth.transform_image(synth.composite_observed(r["bgr"], r["mask"], b)))
        black.append(synth.transform_image(np.where(r["mask"][..., None] > 0, r["bgr"].astype(np.uint8), 0).astype(np.uint8)))
        d = np.where(r["depth"] > 0, r["depth"] + rng.normal(0, 0.002, r["depth"].shape), rng.uniform(1.0, 2.0, r["depth"].shape))
        depth.append(O.depth_from_u16(np.clip(np.rint(d * 1000.0), 0, 65535).astype(np.uint16), 1000.0))
    return dict(poses=poses, cls=cls, img={"mask": np.stack(noise), "rgbd": np.stack(noise), "image": np.stack(black)},
                depth=np.stack(depth)[:, None])


def expect(meshes, scene, net, lit, poses=None, cls=None, Ks=None, frames=None, n=B):
    """The loop's front for instance b = 0 ... n-1 from the oracle's primitives: bbox (8), zoom factor, status, the zoomed
    blobs and conv1's input [n, C, H, W].  Ks[b]: instance b's camera; frames[b]: its observed frame index."""
    poses = scene["poses"] if poses is None else poses
    cls = scene["cls"] if cls is None else cls
    img_o, dep_o = scene["img"][net], scene["depth"]
    m32 = np.asarray(MEANS, np.float32)
    out = {k: [] for k in ("bbox", "zf", "status", "zio", "zir", "zmo", "zmr", "zdo", "zdr", "x")}
    for b in range(n):
        Kb = K if Ks is None else Ks[b]
        f = b if frames is None else frames[b]
        r = render(meshes, int(cls[b]), poses[b], Kb, LIT["intensity"][0, b] if lit else None)
        bad = int(cls[b]) not in meshes
        if net == "image":
            so = ((img_o[f, 0] + m32[0]) + (img_o[f, 1] + m32[1])) + (img_o[f, 2] + m32[2])
            sr = ((r["image"][0] + m32[0]) + (r["image"][1] + m32[1])) + (r["image"][2] + m32[2])
            real, ren = O.mask_bbox(so.astype(np.float32), 0.01), O.mask_bbox(sr.astype(np.float32), 0.01)
        else:
            ren = r["bbox"].astype(np.int32)
            real = O.mask_bbox(O.box_mask(ren, H, W), 0.3)  # the end-exclusive observed rectangle's box
        z = np.zeros(4, np.float32)
        rc = O.lib().orc_zoom_factor(real, ren, np.ascontiguousarray(poses[b], np.float32),
                                     np.ascontiguousarray(Kb, np.float32).reshape(9), H, W, z)
        st = 2 if bad else 0
        if rc != 0:  # the reference raises; the device's documented fallback
            z[:] = (1.0, 1.0, 0.0, 0.0)
            real = np.full(4, -1, np.int32)
            st |= 1
        elif net == "image" and ren[1] < 0:
            st |= 4
        out["bbox"].append(np.concatenate([real, ren]))
        out["zf"].append(z)
        out["status"].append(st)
        zio, zir = O.zoom_image_with_factor(z[None], img_o[f][None], r["image"][None], MEANS)
        zdo = zdr = zmo = zmr = None
        if net == "rgbd":
            zdo, zdr = O.zoom_plane(dep_o[f, 0], z, 0)[None, None], O.zoom_plane(r["depth"], z, 0)[None, None]
        if net != "image":
            zmo = O.zoom_plane(O.box_mask(ren, H, W), z, 1)[None, None]
            zmr = O.zoom_plane(r["mask"], z, 2)[None, None]
        for k, v in (("zio", zio), ("zir", zir), ("zdo", zdo), ("zdr", zdr), ("zmo", zmo), ("zmr", zmr)):
            out[k].append(v)
        out["x"].append(O.conv1_input(zio, zir, zdo, zdr, zmo, zmr))
    res = {k: None if v[0] is None else np.concatenate(v) for k, v in out.items() if k not in ("bbox", "zf", "status")}
    res.update(bbox=np.stack(out["bbox"]), zf=np.stack(out["zf"]), status=np.asarray(out["status"], np.int32))
    return res


@pytest.fixture(scope="module")
def expected(meshes, scene):
    """one expectation per (network, lighting), shared by the precisions"""
    cache = {}

    def get(net, lit):
        if (net, lit) not in cache:
            cache[net, lit] = expect(meshes, scene, net, lit)
        return cache[net, lit]
    return get


def test_scene_covers_the_edges(meshes, scene, expected):
    """each instance is the case it claims to be, by the oracle's renders"""
    e, ei = expected("mask", False), expected("image", False)
    ren, st = e["bbox"][:, 4:], e["status"]
    x0, x1, y0, y1 = ren.T
    i = IDX
    assert x0[i["cut left"]] == 0 and x1[i["cut right"]] == W - 1 and y0[i["cut top"]] == 0 and y1[i["cut bottom"]] == H - 1
    assert x1[i["cut corner"]] == W - 1 and y1[i["cut corner"]] == H - 1
    for b in (i["centred cube"], i["centred blob"], i["black cube"]):
        assert 0 < x0[b] and x1[b] < W - 1 and 0 < y0[b] and y1[b] < H - 1
    wx, _, tx, ty = e["zf"][i["near, crop wider than the frame"]]
    assert wx > 1.5
    # the crop is wider than the frame: its outermost taps lie outside [-4, N + 4], where the sampler clamps them
    assert ((tx - wx) + 1) * (W - 1) / 2 < -4 or ((tx + wx) + 1) * (W - 1) / 2 > W + 4
    p = scene["poses"][i["straddles the near plane"]].astype(np.float32)
    zc = (meshes[BIG].verts.astype(np.float32) @ p[:, :3].T + p[:, 3])[:, 2]
    assert (zc < ZN).any() and (zc <= 1e-6).any() and (zc > ZN).any() and x1[i["straddles the near plane"]] >= 0
    assert x0[i["one column"]] == x1[i["one column"]] and y0[i["one row"]] == y1[i["one row"]]
    assert x1[i["2 x 2 pixels"]] - x0[i["2 x 2 pixels"]] == 1 and y1[i["2 x 2 pixels"]] - y0[i["2 x 2 pixels"]] == 1
    for b in (i["one column"], i["one row"]):
        assert e["x"][b, 7].sum() > 0 and (e["zf"][b] == (1, 1, 0, 0)).all() and st[b] == 1
    assert x1[i["out of view"]] == -1 and st[i["out of view"]] == 1
    assert st[i["class >= max_classes"]] == 3 and st[i["class without a mesh"]] == 3
    assert set(FALLBACK) == set(np.flatnonzero(st & 1))
    assert sorted(set(x0[x0 >= 0] % 4)) == [0, 1, 2, 3]
    # the lit loop's light comes from the float64 pose: from its float32 cast, the centred cube renders differently
    p64 = scene["poses"][i["centred cube"]]
    p32 = p64.astype(np.float32).astype(np.float64)
    lit = [O.render_lit(meshes[CUBE], meshes[CUBE].normals, p64, K, O.light_position(q), LIT["intensity"][0, 0],
                        means_rgb=MEANS, want=("image",))["image"] for q in (p64, p32)]
    assert (lit[0] != lit[1]).any()
    # the image-only network: observed boxes are the objects' own; out of view and the black cube centre on them (bit 2)
    sti = ei["status"]
    assert sti[i["out of view"]] == 4 and sti[i["black cube"]] == 4 and ei["bbox"][i["black cube"], 5] == -1
    assert sti[i["class >= max_classes"]] == 6 and sti[i["class without a mesh"]] == 6
    assert ei["bbox"][i["cut left"], 0] == 0 and ei["bbox"][i["cut corner"], 1] == W - 1
    assert not np.delete(sti, [i["out of view"], i["black cube"], i["class >= max_classes"], i["class without a mesh"]]).any()


def conv1_canvas(ctx, n, prec):
    """conv1's input as stored: (hi, lo) decoded canvases [n, L, 2 rows, 2 cols] (lo None unless bf16x3), and the pad"""
    hi, g = ctx.debug_activation(0, n, fp16=prec == "fp16")
    lo = s2d_decode(ctx.debug_activation(0, n, lo=True)[0]) if prec == "bf16x3" else None
    return s2d_decode(hi), lo, g[3]


def assert_conv1(ctx, x, prec, tag, n=None):
    """conv1's stored input equals the expected [n, C, H, W] blob rounded to the mode's format, bit for bit (bf16x3: both
    halves, the residual rnd(x - rnd(x))), the pad border exactly zero; a failure names the instance, pixel and lane"""
    n = x.shape[0] if n is None else n
    hi, lo, pad = conv1_canvas(ctx, n, prec)
    exp = np.zeros_like(hi)
    exp[:, :x.shape[1], pad:pad + H, pad:pad + W] = x
    want = rnd(exp, prec)
    for name, got, w in (("hi", hi, want), ("lo", lo, None if lo is None else rnd(exp - want, prec))):
        if got is None:
            continue
        bad = np.argwhere(got != w)
        assert not len(bad), "%s: conv1 input %s differs in %d elements; first (instance, lane, y, x) = %s: got %r want %r" % (
            tag, name, len(bad), [tuple(int(v) - (pad if k >= 2 else 0) for k, v in enumerate(j)) for j in bad[:6]],
            float(got[tuple(bad[0])]), float(w[tuple(bad[0])]))


def refine_args(scene, net, cls=None):
    kw = {"depth_observed": dev(scene["depth"])} if net == "rgbd" else {}
    cls = scene["cls"] if cls is None else cls
    return dev(scene["img"][net]), dev(cls), kw


def assert_front(ctx, res, e, n, tag, it=0):
    assert np.array_equal(res["bbox"][it].cpu().numpy(), e["bbox"][:n]), (tag, res["bbox"][it].cpu().numpy(), e["bbox"][:n])
    zf = res["zoom_factor"][it].cpu().numpy()
    assert np.array_equal(zf.view(np.int32), e["zf"][:n].view(np.int32)), (tag, zf, e["zf"][:n])
    st = ctx.refine_status(n, it + 1).numpy()[it]
    assert np.array_equal(st, e["status"][:n]), (tag, st, e["status"][:n])


@pytest.mark.parametrize("prec", sorted(PREC))
@pytest.mark.parametrize("lit", [False, True], ids=["unlit", "lit"])
@pytest.mark.parametrize("net", NETS)
def test_loop_front_bit_for_bit(ctxs, weights, scene, expected, net, lit, prec):
    """dim_refine, one iteration: bbox, zoom factor and status exact, conv1's input bit for bit, se3 against float64 fc6 ->
    heads from the loop's own act[10] with invZoomTrans"""
    ctx, e = ctxs[net], expected(net, lit)
    img, cls, kw = refine_args(scene, net)
    if lit:
        kw["lighting"] = dict(LIT, intensity=dev(LIT["intensity"]))
    res = ctx.refine(img, cls, dev(scene["poses"]), K, 1, pixel_means_rgb=MEANS, precision=PREC[prec], **kw)
    torch.cuda.synchronize()
    tag = "%s %s %s" % (net, "lit" if lit else "unlit", prec)
    assert_front(ctx, res, e, B, tag)
    assert_conv1(ctx, e["x"], prec, tag)
    hi, _ = ctx.debug_activation(10, B, fp16=prec == "fp16")
    lo = ctx.debug_activation(10, B, lo=True)[0] if prec == "bf16x3" else None
    se3 = res["se3"][0]
    R.check_fc6_heads(weights[net], prec, B, (hi, lo), se3[:, :4], se3[:, 4:], tag=" " + tag, zoom_factor=e["zf"])


def test_stale_ren4_is_never_read(ctxs, meshes, scene, expected):
    """ren4 is written only inside the vertex box.  Every slot first renders the large cube near the camera; then iteration 0
    of a two-iteration call renders each slot's own class large and near, and iteration 1 the scene (smaller, shifted, a bad
    class with an empty vertex box): conv1's input after the call is iteration 1's, bit for bit"""
    near = pose(E(0.2, 0.3, 0.1), (0.0, 0.0, 0.35))
    for net in NETS:
        ctx = ctxs[net]
        img, cls, kw = refine_args(scene, net)
        big = dev(np.full(B, BIG, np.int32))
        ctx.refine(img, big, dev(np.stack([near] * B)), K, 1, pixel_means_rgb=MEANS, **kw)
        over = dev(np.stack([np.stack([near] * B), scene["poses"]]))
        res = ctx.refine(img, cls, dev(scene["poses"]), K, 2, pixel_means_rgb=MEANS, pose_override=over, **kw)
        torch.cuda.synchronize()
        e = expected(net, False)
        assert_front(ctx, res, e, B, net + " stale ren4", it=1)
        assert_conv1(ctx, e["x"], "fp16", net + " stale ren4")


def test_smaller_batch_on_the_same_context(ctxs, scene, expected):
    """B = 16, then B = 3: the first 3 images match their expectation, images 3 ... 15 of conv1's input are untouched"""
    for net in NETS:
        ctx, e = ctxs[net], expected(net, False)
        img, cls, kw = refine_args(scene, net)
        ctx.refine(img, cls, dev(scene["poses"]), K, 1, pixel_means_rgb=MEANS, precision=capi.PREC_BF16X3, **kw)
        before = conv1_canvas(ctx, B, "bf16x3")
        kw3 = {"depth_observed": kw["depth_observed"][:3].contiguous()} if kw else {}
        res = ctx.refine(img[:3].contiguous(), cls[:3].contiguous(), dev(scene["poses"][:3]), K, 1, pixel_means_rgb=MEANS,
                         precision=capi.PREC_BF16X3, **kw3)
        torch.cuda.synchronize()
        assert_front(ctx, res, e, 3, net + " B=3")
        assert_conv1(ctx, e["x"][:3], "bf16x3", net + " B=3")
        after = conv1_canvas(ctx, B, "bf16x3")
        for a, b0 in zip(after[:2], before[:2]):
            assert np.array_equal(a[3:], b0[3:]), "%s: B = 3 wrote past image 2" % net


def test_frames_from_several_cameras(meshes, weights, scene):
    """one dim_refine call with K_frames: 3 frames from 3 cameras, a non-identity frame map; each instance's expectation is built
    with its frame and its frame's camera"""
    Kf = np.stack([K, K.copy(), K.copy()]).astype(np.float32)
    Kf[1, 0, 0] *= 1.1
    Kf[1, 0, 2] += 7.25
    Kf[2, 1, 1] *= 0.9
    Kf[2, 1, 2] -= 5.5
    src = [IDX["cut corner"], IDX["centred blob"], IDX["near, crop wider than the frame"]]
    fidx = np.array([(2 * b + 1) % 3 for b in range(B)], np.int32)
    sc = dict(scene, img={n: v[src] for n, v in scene["img"].items()}, depth=scene["depth"][src])
    for net in ("mask", "image"):
        e = expect(meshes, sc, net, False, Ks=Kf[fidx], frames=fidx)
        ctx = make_ctx(meshes, weights, net)
        try:
            res = ctx.refine_frames(dev(sc["img"][net]), dev(fidx), dev(scene["cls"]), dev(scene["poses"]), dev(Kf), 1,
                                    pixel_means_rgb=MEANS, precision=capi.PREC_FP16)
            torch.cuda.synchronize()
            assert_front(ctx, res, e, B, net + " frames")
            assert_conv1(ctx, e["x"], "fp16", net + " frames")
        finally:
            ctx.close()


@pytest.mark.parametrize("prec", sorted(PREC))
@pytest.mark.parametrize("net", NETS)
def test_net_fwd_packs_conv1_input(ctxs, expected, net, prec):
    """dim_net_fwd's conv1 input (pack_nhwc8_kernel with and without masks, pack_nhwc10_kernel) at B = 1, 3, 16 equals the
    rounded conv1_input of the blobs passed in, bit for bit"""
    ctx, e = ctxs[net], expected(net, False)
    for n in (1, 3, B):
        args = [dev(e[k][:n]) for k in ("zio", "zir")]
        kw = {}
        if net != "image":
            args += [dev(e["zmo"][:n]), dev(e["zmr"][:n])]
        if net == "rgbd":
            kw = {"zoom_depth_observed": dev(e["zdo"][:n]), "zoom_depth_rendered": dev(e["zdr"][:n])}
        ctx.net_forward(*args, precision=PREC[prec], **kw)
        torch.cuda.synchronize()
        assert_conv1(ctx, e["x"][:n], prec, "%s net_fwd %s B=%d" % (net, prec, n))


@pytest.mark.parametrize("net", NETS)
def test_training_step_conv1_input(meshes, expected, scene, net):
    """after one forward_backward of 3 zoomed instances, the training context's conv1 input is the same rounding of the
    zoomed batch it was given, bf16 and bf16x3"""
    e, n = expected(net, False), 3
    w = synth.make_train_weights(0, input_depth=net == "rgbd", input_mask=net != "image")
    ctx = Context(0, max_batch=n, max_classes=1, max_verts=6000, max_faces=11000, input_depth=net == "rgbd",
                  input_mask=net != "image")
    try:
        tr = Trainer(ctx, w, max_points=100)
        rng = np.random.default_rng(4)
        f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV)
        z = {"zoom_image_observed": f32(e["zio"][:n]), "zoom_image_rendered": f32(e["zir"][:n]),
             "zoom_mask_observed": f32(e["zmo"][:n] if net != "image" else np.zeros((n, 1, H, W))),
             "zoom_mask_rendered": f32(e["zmr"][:n] if net != "image" else np.zeros((n, 1, H, W))),
             "zoom_factor": f32(e["zf"][:n]), "zoom_flow": f32(np.zeros((n, 2, H, W))),
             "zoom_flow_weights": f32(np.zeros((n, 2, H, W))), "zoom_mask_gt_observed": f32(np.zeros((n, 1, H, W))),
             "src_pose": f32(scene["poses"][:n]), "point_cloud_model": f32(rng.normal(0, 0.05, (n, 3, 100))),
             "point_cloud_weights": f32(np.ones((n, 3, 100))), "point_cloud_observed": f32(rng.normal(0, 0.05, (n, 3, 100)))}
        if net == "rgbd":
            z["zoom_depth_observed"], z["zoom_depth_rendered"] = f32(e["zdo"][:n]), f32(e["zdr"][:n])
        for prec in ("bf16", "bf16x3"):
            tr.set_precision(prec)
            tr.forward_backward(z, want_maps=False)
            torch.cuda.synchronize()
            assert_conv1(ctx, e["x"][:n], prec, "%s training step %s" % (net, prec))
    finally:
        ctx.close()
