"""GPU: the zoom stage against the float64 reference of tests/zoom_ref.py, under its tolerance rule, teacher-forced: the
sampling checks take the device's own float32 zoom factor and boxes, and the factor and boxes are checked on their own.

The op surface (ZoomMask, ZoomImage, ZoomImageWithFactor, ZoomMaskWithFactor and ZoomFlow both ways, ZoomDepth, ZoomTrans
forward and backward) on contexts of 480 x 640, 61 x 84 (odd H, H W not a multiple of the 256-thread block) and 130 x 172,
one instance at a time and every scene (or every affine) in one batch, each instance checked; then conv1's input written by the fused refinement loop for the mask, RGB-D and image-only networks
in fp16, bf16 and bf16x3, against the reference fed the loop's render (held bit-equal to the oracle's by
test_gpu_loop_front.py).  Prints the largest ambiguous share of each test."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

import zoom_ref as Z  # noqa: E402
import zoom_scenes as S  # noqa: E402
from kernel_ref import s2d_decode  # noqa: E402
from oracle import oracle as O  # noqa: E402
from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402

DEV = torch.device("cuda", 0)
F32 = np.float32
BATCHES = ("one", "all")
MAX_B = 8  # len(S.mask_scenes(...)) == len(S.affines(...))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


@pytest.fixture(scope="module", params=S.SIZES, ids=["%dx%d" % s for s in S.SIZES])
def ctx(request):
    H, W = request.param
    c = Context(0, max_batch=MAX_B, height=H, width=W, max_classes=1, max_verts=100, max_faces=100)
    yield c
    c.close()


def batch_of(items, B, one):
    """the item `one` alone, or every item in one batch (past the first grid row)"""
    assert len(items) <= MAX_B
    return [items[one]] if B == "one" else items


@pytest.mark.parametrize("B", BATCHES)
def test_zoom_mask(ctx, B):
    """ZoomMask: boxes exact, factor in its float32 range (empty observed mask: (1, 1, 0, 0) and status bit 0), the
    three planes at the device's factor; every scene's claim holds, and the batch of all scenes takes every branch"""
    H, W, K = ctx.H, ctx.W, S.camera(ctx.H, ctx.W)
    S.assert_mask_scene_claims(H, W)
    sc = batch_of(S.mask_scenes(H, W), B, 2)
    mo, mg, mr, pose = [np.stack([s[k] for s in sc]) for k in (1, 2, 3, 4)]
    zo, zg, zr, zf, bbox, st = ctx.zoom_mask(dev(mo[:, None]), dev(mg[:, None]), dev(mr[:, None]), dev(pose), K)
    zo, zg, zr, zf, bbox, st = [host(t) for t in (zo, zg, zr, zf, bbox, st)]
    share, empty, wide = 0.0, 0, 0
    for b, s in enumerate(sc):
        vr, _ = Z.mask_valid(mg[b][None], False)
        vn, _ = Z.mask_valid(mr[b][None], True)
        assert np.array_equal(bbox[b], np.concatenate([Z.box(vr), Z.box(vn)])), (s[0], bbox[b])
        rng = Z.zoom_factor_range(bbox[b, :4], bbox[b, 4:], pose[b, :, 3], K, H, W)
        if rng is None:
            assert (zf[b] == (1, 1, 0, 0)).all() and st[b] & 1, s[0]
            empty += 1
        else:
            assert Z.factor_ok(zf[b], rng) and not st[b] & 1, (s[0], zf[b], rng)
            wide += bool(zf[b, 0] > 2 and abs(zf[b, 2]) > 1)
        for got, img, mode in ((zo, mo, 1), (zg, mg, 1), (zr, mr, 2)):
            share = max(share, Z.check_plane(got[b, 0], Z.zoom_expect(img[b], zf[b], mode), "%s mode %d" % (s[0], mode)))
    if B == "all":  # the empty-observed fallback and a crop over 2x centred off the frame were taken
        assert empty == 1 and wide >= 1, (empty, wide)
    print("zoom_mask %dx%d B=%s: largest ambiguous share %.2e" % (H, W, B, share))


@pytest.mark.parametrize("B", BATCHES)
def test_zoom_image_and_with_factor(ctx, B):
    """ZoomImage (boxes from sum_c(image + mean) > 0.01, ambiguity asserted small), its factor, and the mode-3 planes of
    it and of ZoomImageWithFactor at every affine, one per instance, each instance with its own planes: out of the frame
    the planes read -mean"""
    H, W, K = ctx.H, ctx.W, S.camera(ctx.H, ctx.W)
    S.assert_image_scene_claims(H, W)
    sc = batch_of(S.image_scenes(H, W), B, 1)
    io, ir, pose = [np.stack([s[k] for s in sc]) for k in (1, 2, 3)]
    zio, zir, zf, bbox, st = [host(t) for t in ctx.zoom_image(dev(io), dev(ir), dev(pose), K, S.MEANS)]
    share = 0.0
    for b, s in enumerate(sc):
        for got, im in ((bbox[b, :4], io[b]), (bbox[b, 4:], ir[b])):
            v, amb = Z.image_valid(im, S.MEANS)
            share = max(share, float(amb.mean()))
            assert amb.mean() < Z.MAX_AMBIGUOUS and Z.box_ok(got, v, amb), (s[0], got)
        assert Z.factor_ok(zf[b], Z.zoom_factor_range(bbox[b, :4], bbox[b, 4:], pose[b, :, 3], K, H, W)), s[0]
        for got, im in ((zio, io), (zir, ir)):
            for c in range(3):
                Z.check_plane(got[b, c], Z.zoom_expect(im[b, c], zf[b], 3, mean=S.MEANS[c]), "%s channel %d" % (s[0], c))
    ims = S.images(H, W)
    planes = np.stack([ims["noise"], ims["steps"], ims["constant"]]) - S.MEANS[:, None, None]
    aff = batch_of(S.affines(H, W), B, 6)
    po = np.stack([np.roll(planes, 3 * b, axis=2) for b in range(len(aff))])  # each instance its own planes
    pr = po[:, ::-1].copy()
    zo, zr = [host(t) for t in ctx.zoom_image_with_factor(dev(np.stack([a for _, a in aff])), dev(po), dev(pr), S.MEANS)]
    for b, (an, a) in enumerate(aff):
        for c in range(3):
            Z.check_plane(zo[b, c], Z.zoom_expect(po[b, c], a, 3, mean=S.MEANS[c]), "%s with_factor observed %d" % (an, c))
            Z.check_plane(zr[b, c], Z.zoom_expect(pr[b, c], a, 3, mean=S.MEANS[c]), "%s with_factor rendered %d" % (an, c))
    print("zoom_image %dx%d B=%s: largest ambiguous share %.2e" % (H, W, B, share))


@pytest.mark.parametrize("B", BATCHES)
def test_with_factor_ops(ctx, B):
    """ZoomMaskWithFactor and ZoomFlow in both directions (1- and 2-channel flow weights), ZoomDepth, ZoomTrans forward and
    backward: every affine, one per instance, each instance with its own planes; the inverse ones sampled at the
    reference's float32 inverse affine"""
    H, W = ctx.H, ctx.W
    rng = np.random.default_rng(6)
    yy, xx = np.mgrid[0:H, 0:W]
    blob = ((xx - 0.4 * W) ** 2 / (0.3 * W) ** 2 + (yy - 0.6 * H) ** 2 / (0.3 * H) ** 2 < 1)
    depth = np.where(blob, rng.uniform(0.0, 1.2, (H, W)), 0).astype(F32)
    depth[rng.random((H, W)) < 0.05] = F32(0.2)
    sensor = np.where(blob, 0.8 + 0.1 * np.sin(xx / 9.0) + rng.normal(0, 0.002, (H, W)), rng.uniform(1, 2, (H, W)))
    sensor = O.depth_from_u16(np.clip(np.rint(sensor * 1000), 0, 65535).astype(np.uint16))
    ims = S.images(H, W)
    flow = np.stack([(ims["smooth"] - 127.5) / F32(7.0), ims["noise"] - F32(127.5)]).astype(F32)
    fw = np.stack([blob, blob[::-1]]).astype(F32)
    aff = batch_of(S.affines(H, W), B, 6)
    n = len(aff)
    roll = lambda p, b: np.roll(p, 5 * b, axis=-1)  # instance b's own plane
    depth_b = np.stack([roll(depth, b)[None] for b in range(n)])
    sensor_b = np.stack([roll(sensor, b)[None] for b in range(n)])
    flow_b, fw_b = np.stack([roll(flow, b) for b in range(n)]), np.stack([roll(fw, b) for b in range(n)])
    Zf = dev(np.stack([a for _, a in aff]))
    share = 0.0
    for inv in (False, True):
        mwf = host(ctx.zoom_mask_with_factor(Zf, dev(depth_b), inv))
        zfl, zfw = ctx.zoom_flow(Zf, dev(flow_b), None if inv else dev(fw_b), inv)
        zfl, zfw = host(zfl), None if inv else host(zfw)
        for b, (an, zf) in enumerate(aff):
            a, da = Z.inv_affine_for_sampling(zf, H, W) if inv else (zf, np.zeros(4))
            tie = an == "half-pixel shift"  # 0 / 1 planes blended half and half: exact 0.5 ties, excluded
            if not tie:
                share = max(share, Z.check_plane(mwf[b, 0], Z.zoom_expect(depth_b[b, 0], a, 2, da=da),
                                                 "%s mwf %s" % (an, inv)))
            for c in range(2):
                Z.check_plane(zfl[b, c], Z.zoom_expect(flow_b[b, c], a, 4 if inv else 6, wx=zf[0], da=da),
                              "%s flow %d inv=%s" % (an, c, inv))
                if not inv and not tie:
                    share = max(share, Z.check_plane(zfw[b, c], Z.zoom_expect(fw_b[b, c], a, 5), "%s weights %d" % (an, c)))
    zdo, zdr = [host(t) for t in ctx.zoom_depth(Zf, dev(sensor_b), dev(depth_b))]
    for b, (an, zf) in enumerate(aff):
        Z.check_plane(zdo[b, 0], Z.zoom_expect(sensor_b[b, 0], zf, 0), "%s depth observed" % an)
        Z.check_plane(zdr[b, 0], Z.zoom_expect(depth_b[b, 0], zf, 0), "%s depth rendered" % an)
    zfs = np.stack([a for _, a in aff])
    t = np.random.default_rng(7).normal(0, 0.3, (len(zfs), 3)).astype(F32)
    for inv in (False, True):
        assert np.array_equal(host(ctx.zoom_trans(dev(zfs), dev(t), inv)), Z.zoom_trans(zfs, t, inv))
        for zg in (False, True):
            assert np.array_equal(host(ctx.zoom_trans_backward(dev(zfs), dev(t), inv, zg)), Z.zoom_trans(zfs, t, inv, zg))
    print("with_factor %dx%d B=%s: largest ambiguous share %.2e" % (H, W, B, share))


# ------------------------------------------------------------------------------------------------------ fused loop
K = synth.K_LINEMOD
MEANS = synth.PIXEL_MEANS_RGB
H0, W0 = 480, 640
NETS = ("mask", "rgbd", "image")
PRECS = {"fp16": capi.PREC_FP16, "bf16": capi.PREC_BF16, "bf16x3": capi.PREC_BF16X3}
CUBE, SMALL, BIG = 0, 1, 2


def _pose(R3, t):
    p = np.zeros((3, 4))
    p[:, :3], p[:, 3] = R3, t
    return p


LOOP = [("centred cube", CUBE, _pose(synth.euler_to_mat(0.3, 0.5, 0.2), (0.0, 0.0, 0.8))),
        ("tiny and far: magnification >= 20", SMALL, _pose(np.eye(3), (0.01, 0.0, 2.5))),
        ("near: crop over 2x the frame", BIG, _pose(synth.euler_to_mat(0.3, 0.4, 0.2), (-0.15, -0.1, 0.40))),
        ("cut by the right border", CUBE, _pose(synth.euler_to_mat(0.2, 0.1, 0.5), (0.44, 0.02, 0.8))),
        ("centre off the frame", BIG, _pose(synth.euler_to_mat(0.1, 0.2, 0.3), (0.47, 0.0, 0.8)))]


@pytest.fixture(scope="module")
def loop():
    ms = {CUBE: synth.make_cube(), SMALL: synth.make_cube(side=0.01, nu=1, nv=1, tex_size=16, seed=3),
          BIG: synth.make_cube(side=0.3, nu=2, nv=2, tex_size=64, seed=4)}
    poses = np.stack([p for _, _, p in LOOP])
    cls = np.array([c for _, c, _ in LOOP], np.int32)
    rng = np.random.default_rng(9)
    noise, black, depth, ren = [], [], [], []
    for b, (_, c, p) in enumerate(LOOP):
        r = O.render(ms[c], p, K, means_rgb=MEANS)
        noise.append(synth.transform_image(synth.composite_observed(r["bgr"], r["mask"], b)))
        black.append(synth.transform_image(np.where(r["mask"][..., None] > 0, r["bgr"].astype(np.uint8), 0).astype(np.uint8)))
        d = np.where(r["depth"] > 0, r["depth"] + rng.normal(0, 0.002, r["depth"].shape), rng.uniform(1.0, 2.0, r["depth"].shape))
        depth.append(O.depth_from_u16(np.clip(np.rint(d * 1000.0), 0, 65535).astype(np.uint16), 1000.0))
        ren.append(O.render(ms[c], _pose(synth.euler_to_mat(0.02, -0.03, 0.01) @ p[:, :3], p[:, 3] * (1, 1, 1.02)), K,
                            means_rgb=MEANS))
    return dict(meshes=ms, poses=np.stack([_pose(synth.euler_to_mat(0.02, -0.03, 0.01) @ p[:, :3], p[:, 3] * (1, 1, 1.02))
                                           for p in poses]),
                cls=cls, img={"mask": np.stack(noise), "rgbd": np.stack(noise), "image": np.stack(black)},
                depth=np.stack(depth), ren=ren)


def test_loop_scene_covers_the_edges(loop):
    """the loop's scene is what it claims: a render of a few pixels (magnification >= 20), a crop over twice the frame,
    one cut by the right border and a zoom centre off the frame"""
    bb = [r["bbox"] for r in loop["ren"]]
    lo, hi = [], []
    for b, r in enumerate(loop["ren"]):
        real = Z.box(Z.observed_rectangle(r["bbox"], H0, W0) > 0)
        rng = Z.zoom_factor_range(real, r["bbox"], loop["poses"][b].astype(F32)[:, 3], K, H0, W0)
        lo.append(rng[0])
        hi.append(rng[1])
    assert 1 / hi[1][0] >= 20 and lo[2][0] > 2 and lo[4][2] > 1
    assert bb[2][0] == 0 and bb[2][2] == 0
    assert bb[3][1] == W0 - 1 and bb[0][0] > 0


@pytest.mark.parametrize("prec", sorted(PRECS))
@pytest.mark.parametrize("net", NETS)
def test_loop_conv1_input(loop, net, prec):
    """conv1's input from one dim_refine iteration: image and depth lanes inside the 16-bit rounding of the continuous
    interval / 255, mask lanes exact where unambiguous; the factor in its float32 range and the boxes exact (image-only
    network: between the readings of the ambiguous pixels)"""
    B = len(LOOP)
    w = synth.make_train_weights(0, input_mask=False) if net == "image" else synth.make_weights(0, input_depth=net == "rgbd")
    ctx = Context(0, max_batch=B, max_classes=3, max_verts=6000, max_faces=11000, input_depth=net == "rgbd",
                  input_mask=net != "image")
    try:
        for i, m in loop["meshes"].items():
            ctx.upload_mesh(i, m)
        ctx.load_weights(w)
        kw = {"depth_observed": dev(loop["depth"][:, None])} if net == "rgbd" else {}
        res = ctx.refine(dev(loop["img"][net]), dev(loop["cls"]), dev(loop["poses"]), K, 1, pixel_means_rgb=MEANS,
                         precision=PRECS[prec], **kw)
        torch.cuda.synchronize()
        zf, bbox = res["zoom_factor"][0].cpu().numpy(), res["bbox"][0].cpu().numpy()
        hi, g = ctx.debug_activation(0, B, fp16=prec == "fp16")
        hi, pad = s2d_decode(hi), g[3]
        lo = s2d_decode(ctx.debug_activation(0, B, lo=True)[0]) if prec == "bf16x3" else None
    finally:
        ctx.close()
    share = 0.0
    for b in range(B):
        r, img = loop["ren"][b], loop["img"][net][b]
        tag = "%s %s %s" % (net, prec, LOOP[b][0])
        if net == "image":
            for got, im in ((bbox[b, :4], img), (bbox[b, 4:], r["image"])):
                v, amb = Z.image_valid(im, MEANS)
                assert amb.mean() < Z.MAX_AMBIGUOUS and Z.box_ok(got, v, amb), (tag, got)
        else:
            assert np.array_equal(bbox[b, 4:], r["bbox"]), tag
            assert np.array_equal(bbox[b, :4], Z.box(Z.observed_rectangle(r["bbox"], H0, W0) > 0)), tag
        rng = Z.zoom_factor_range(bbox[b, :4], bbox[b, 4:], loop["poses"][b].astype(F32)[:, 3], K, H0, W0)
        assert rng is not None and Z.factor_ok(zf[b], rng), (tag, zf[b], rng)
        blobs = {"zio": [Z.zoom_expect(img[c], zf[b], 3, mean=MEANS[c]) for c in range(3)],
                 "zir": [Z.zoom_expect(r["image"][c], zf[b], 3, mean=MEANS[c]) for c in range(3)],
                 "zdo": [Z.zoom_expect(loop["depth"][b], zf[b], 0)], "zdr": [Z.zoom_expect(r["depth"], zf[b], 0)],
                 "zmo": [Z.zoom_expect(Z.observed_rectangle(bbox[b, [0, 1, 2, 3]] + (0, 1, 0, 1), H0, W0), zf[b], 1)],
                 "zmr": [Z.zoom_expect(r["depth"] if net == "rgbd" else r["mask"], zf[b], 2)]}
        lane = 0
        for name, n, div in Z.conv1_lanes(net):
            for e in blobs[name]:
                h = hi[b, lane, pad:pad + H0, pad:pad + W0].astype(np.float64)
                ll = None if lo is None else lo[b, lane, pad:pad + H0, pad:pad + W0].astype(np.float64)
                if e[0] == "interval":
                    qlo, qhi = Z.scaled_interval(e[1], e[2], div)
                    ok = Z.stored16_ok(h, ll, qlo, qhi, prec)
                    bad = np.argwhere(~ok)
                    assert not len(bad), "%s lane %d: %d pixels outside; first %s: got %r (+ %r), interval [%r, %r]" % (
                        tag, lane, len(bad), tuple(bad[0]), h[tuple(bad[0])], None if ll is None else ll[tuple(bad[0])],
                        qlo[tuple(bad[0])], qhi[tuple(bad[0])])
                else:
                    share = max(share, Z.check_plane(h + (0 if ll is None else ll), e, "%s lane %d" % (tag, lane)))
                lane += 1
        assert lane == w["flow_conv1_weight"].shape[1]
        assert not hi[b, lane:].any(), tag
    print("loop %s %s: largest ambiguous share %.2e" % (net, prec, share))
