"""CPU: the float64 zoom reference (tests/zoom_ref.py) on known answers, its coordinate bound against the float32 chain, and
the oracle's zoom primitives against it under the reference's tolerance rule: every sampler mode forward and inverse,
ZoomMask, ZoomImage, ZoomMaskWithFactor, ZoomFlow, ZoomTrans, the box mask and conv1's input, at three frame sizes."""
import numpy as np
import pytest

import zoom_ref as Z
import zoom_scenes as S
from oracle import oracle as O

F32 = np.float32


# ------------------------------------------------------------------------------------------ known answers of the reference
@pytest.mark.parametrize("H,W", S.SIZES)
def test_reference_known_answers(H, W):
    """identity returns the image; an integer shift the shifted image with zero fill; a half-pixel shift neighbour means"""
    img = S.images(H, W)["noise"].astype(np.float64)
    # the float64 grid is j to within a few ulp: the identity returns the image to float64 rounding
    assert np.abs(Z.zoom(img, (1, 1, 0, 0)) - img).max() <= 1e-12 * 255
    # x = j + 3, y = i - 2, in float64 exactly when the translation is a float64 multiple of 2 / (N - 1)
    X = Z.grid(1.0, 3 * 2.0 / (W - 1), W)
    Y = Z.grid(1.0, -2 * 2.0 / (H - 1), H)
    assert np.abs(X - (np.arange(W) + 3)).max() < 1e-9 and np.abs(Y - (np.arange(H) - 2)).max() < 1e-9
    want = np.zeros_like(img)
    want[2:, :W - 3] = img[:H - 2, 3:]
    got = Z.sample(img, np.round(X)[None, :], np.round(Y)[:, None])
    assert np.array_equal(got, want)
    half = Z.sample(img, (np.arange(W) + 0.5)[None, :], np.arange(H, dtype=np.float64)[:, None])
    nxt = np.concatenate([img[:, 1:], np.zeros((H, 1))], axis=1)
    assert np.abs(half - 0.5 * (img + nxt)).max() <= 1e-13 * 255


@pytest.mark.parametrize("H,W", S.SIZES)
def test_reference_matches_torch_grid_sample_float64(H, W):
    """mode 0 == affine_grid + grid_sample (align_corners=True, zeros) in float64, to 1e-12, on every affine"""
    import torch
    import torch.nn.functional as F

    for name, img in S.images(H, W).items():
        for an, a in S.affines(H, W):
            theta = torch.tensor([[[float(a[0]), 0, float(a[2])], [0, float(a[1]), float(a[3])]]], dtype=torch.float64)
            g = F.affine_grid(theta, (1, 1, H, W), align_corners=True)
            zt = F.grid_sample(torch.from_numpy(img.astype(np.float64))[None, None], g, mode="bilinear",
                               padding_mode="zeros", align_corners=True)[0, 0].numpy()
            assert np.abs(Z.zoom(img, a) - zt).max() <= 1e-12 * max(1.0, np.abs(img).max()), (name, an)


@pytest.mark.parametrize("H,W", S.SIZES)
def test_coordinate_bound_holds_the_float32_chain(H, W):
    """|x_f32 - x| <= d_x for every output index of every affine used, forward and inverse, on both axes; and the bound
    is not loose by orders of magnitude (the largest error is a fair share of it somewhere)"""
    S.assert_affine_claims(H, W)
    used = [(a, np.zeros(4)) for _, a in S.affines(H, W)]
    used += [Z.inv_affine_for_sampling(a, H, W) for a, _ in used]
    share = 0.0
    for a, da in used:
        for w, t, N, dw, dt in ((a[0], a[2], W, da[0], da[2]), (a[1], a[3], H, da[1], da[3])):
            err = np.abs(S.chain_f32(w, t, N).astype(np.float64) - Z.grid(w, t, N))
            d = Z.coord_bound(w, t, N, dw, dt)
            assert (err <= d).all(), (a, N, np.max(err - d))
            share = max(share, float((err / (d - Z.WEIGHT_SHIFT)).max()))
    assert share > 0.1, share


# -------------------------------------------------------------------------------------------- the oracle's primitives


def mode_inputs(H, W, seed=3):
    """per mode, [H, W] float32 planes of the kind the op is given"""
    rng = np.random.default_rng(seed)
    ims = S.images(H, W)
    yy, xx = np.mgrid[0:H, 0:W]
    blob = ((xx - 0.4 * W) ** 2 / (0.3 * W) ** 2 + (yy - 0.6 * H) ** 2 / (0.3 * H) ** 2 < 1)
    soft = (blob * np.clip(rng.normal(0.7, 0.3, (H, W)), 0, 1)).astype(F32)
    depth = np.where(blob, rng.uniform(0.0, 1.2, (H, W)), 0).astype(F32)
    depth[rng.random((H, W)) < 0.05] = F32(0.2)
    flow = (ims["smooth"] - 127.5).astype(F32) / F32(7.0)
    weights = np.where(blob, 1.0, 0.0).astype(F32)
    return {0: list(ims.values()) + [depth], 1: [soft, blob.astype(F32)], 2: [depth], 3: list(ims.values()),
            4: [flow, ims["steps"]], 5: [weights], 6: [flow, ims["noise"]]}


@pytest.mark.parametrize("H,W", S.SIZES)
@pytest.mark.parametrize("inv", [False, True], ids=["forward", "inverse"])
def test_oracle_zoom_plane_every_mode(H, W, inv):
    """O.zoom_plane in modes 0 ... 5 and O.zoom_flow's / wx (mode 6) under every affine, forward and inverse"""
    mean = float(S.MEANS[2])
    shares = []
    for an, zf in S.affines(H, W):
        a, da = Z.inv_affine_for_sampling(zf, H, W) if inv else (zf, np.zeros(4))
        if inv:
            lo, hi = Z.inv_affine_f32(zf, H, W)
            got = O.inv_zoom_affine(zf, H, W)
            assert ((got >= lo) & (got <= hi)).all(), (an, got, lo, hi)
        for mode, planes in mode_inputs(H, W).items():
            if an == "half-pixel shift" and mode in (1, 2, 5):
                continue  # 0 / 1 planes blended half and half: exact 0.5 ties on a large share, which no bound settles
            for k, img in enumerate(planes):
                tag = "%dx%d %s %s mode %d input %d" % (H, W, an, "inverse" if inv else "forward", mode, k)
                if mode == 6:
                    if inv:
                        continue  # the inverse ZoomFlow multiplies (mode 4)
                    got = O.zoom_flow(zf[None], np.stack([img, img])[None])[0][0, 0]
                else:
                    got = O.zoom_plane(img, a, mode, {3: mean, 4: float(zf[0])}.get(mode, 0.0))
                shares.append(Z.check_plane(got, Z.zoom_expect(img, a, mode, mean=mean, wx=zf[0], da=da), tag))
    assert max(shares) < Z.MAX_AMBIGUOUS


def test_mode3_pads_with_minus_mean():
    """a constant image zoomed out past the frame: inside, the constant; outside, exactly -mean"""
    H, W = 61, 84
    img = S.images(H, W)["constant"]
    zf = dict(S.affines(H, W))["crop 5x, centre off the frame"]
    kind, lo, hi = Z.zoom_expect(img, zf, 3, mean=103.939)
    got = O.zoom_plane(img, zf, 3, 103.939)
    Z.check_plane(got, (kind, lo, hi), "constant")
    out = (hi < -103.0)
    assert out.mean() > 0.3 and np.all(got[out] == -F32(103.939))
    assert (lo > 76).any()


@pytest.mark.parametrize("H,W", S.SIZES)
def test_oracle_zoom_mask(H, W):
    """O.zoom_mask (each scene the case it claims): boxes exact, the zoom factor within its float32 range, the three planes (modes 1, 1, 2) against the
    reference at the oracle's own factor"""
    K = S.camera(H, W)
    S.assert_mask_scene_claims(H, W)
    for name, mo, mg, mr, pose in S.mask_scenes(H, W):
        vr, ar = Z.mask_valid(mg[None], False)
        vn, an = Z.mask_valid(mr[None], True)
        assert not ar.any() and not an.any()
        if not vr.any():
            with pytest.raises(ValueError):
                O.zoom_mask(mo[None, None], mg[None, None], mr[None, None], pose[None], K)
            continue
        zo, zg, zr, zf, bbox = O.zoom_mask(mo[None, None], mg[None, None], mr[None, None], pose[None], K)
        assert np.array_equal(bbox[0], np.concatenate([Z.box(vr), Z.box(vn)])), name
        rng = Z.zoom_factor_range(bbox[0, :4], bbox[0, 4:], pose[:, 3], K, H, W)
        assert Z.factor_ok(zf[0], rng), (name, zf[0], rng)
        for got, img, mode in ((zo, mo, 1), (zg, mg, 1), (zr, mr, 2)):
            Z.check_plane(got[0, 0], Z.zoom_expect(img, zf[0], mode), "%s mode %d" % (name, mode))


@pytest.mark.parametrize("H,W", S.SIZES)
def test_oracle_zoom_image(H, W):
    """O.zoom_image: boxes from sum_c(image + mean) > 0.01 (ambiguity asserted small), the factor, the mode-3 planes"""
    K = S.camera(H, W)
    S.assert_image_scene_claims(H, W)
    for name, io, ir, pose in S.image_scenes(H, W):
        zio, zir, zf, bbox = O.zoom_image(io[None], ir[None], pose[None], K, S.MEANS)
        for got, im in ((bbox[0, :4], io), (bbox[0, 4:], ir)):
            v, amb = Z.image_valid(im, S.MEANS)
            assert amb.mean() < Z.MAX_AMBIGUOUS and Z.box_ok(got, v, amb), (name, got)
        assert Z.factor_ok(zf[0], Z.zoom_factor_range(bbox[0, :4], bbox[0, 4:], pose[:, 3], K, H, W)), name
        for got, im in ((zio, io), (zir, ir)):
            for c in range(3):
                Z.check_plane(got[0, c], Z.zoom_expect(im[c], zf[0], 3, mean=S.MEANS[c]), "%s channel %d" % (name, c))


@pytest.mark.parametrize("H,W", S.SIZES)
def test_oracle_with_factor_ops(H, W):
    """ZoomMaskWithFactor (both directions) and ZoomFlow (forward with 1- and 2-channel weights, inverse) at every affine"""
    inp = mode_inputs(H, W)
    depth, flow, fw = inp[2][0], np.stack(inp[4]), inp[5][0]
    fws = np.stack([fw, fw[::-1].copy()])
    for an, zf in S.affines(H, W):
        for inv in (False, True):
            a, da = Z.inv_affine_for_sampling(zf, H, W) if inv else (zf, np.zeros(4))
            got = O.zoom_mask_with_factor(zf[None], depth[None, None], inv)[0, 0]
            if an != "half-pixel shift":  # exact 0.5 ties, as above
                Z.check_plane(got, Z.zoom_expect(depth, a, 2, da=da), "%s mask_with_factor inv=%s" % (an, inv))
            zfl, zfw = O.zoom_flow(zf[None], flow[None], None if inv else fws[None], b_inv_zoom=inv)
            for c in range(2):
                Z.check_plane(zfl[0, c], Z.zoom_expect(flow[c], a, 4 if inv else 6, wx=zf[0], da=da), "%s flow %d" % (an, c))
                if not inv and an != "half-pixel shift":
                    Z.check_plane(zfw[0, c], Z.zoom_expect(fws[c], a, 5, da=da), "%s flow weights %d" % (an, c))


def test_oracle_box_mask_zoom_trans_and_conv1_input():
    """the end-exclusive rectangle (border, one-column and empty boxes), ZoomTrans both ways (exact float32) and conv1's
    input channels (the / 255 is the correctly rounded float32 division)"""
    H, W = 61, 84
    for bb in ([0, W, 0, H], [5, 6, 7, 30], [10, 10, 3, 9], [-1, -1, -1, -1], [W - 1, W, H - 1, H]):
        assert np.array_equal(O.box_mask(np.array(bb, np.int32), H, W), Z.observed_rectangle(bb, H, W)), bb
    rng = np.random.default_rng(5)
    zf = np.array([a for _, a in S.affines(H, W)], F32)
    t = rng.normal(0, 0.3, (len(zf), 3)).astype(F32)
    for inv in (False, True):
        assert np.array_equal(O.zoom_trans(zf, t, inv), Z.zoom_trans(zf, t, inv)), inv
    ims = S.images(H, W)
    zio = np.stack([ims["noise"], ims["smooth"], ims["steps"]])[None] - S.MEANS[None, :, None, None]
    zir = zio[:, ::-1].copy()
    zd = (ims["smooth"] / F32(97.0))[None, None]
    zm = (ims["steps"] / F32(255.0))[None, None]
    for net, args in (("mask", (zio, zir, None, None, zm, zm)), ("rgbd", (zio, zir, zd, zd, zm, zm)),
                      ("image", (zio, zir, None, None, None, None))):
        x = O.conv1_input(*args)
        blobs = dict(zip(("zio", "zir", "zdo", "zdr", "zmo", "zmr"), args))
        want = np.concatenate([blobs[n][0].astype(np.float64) / d for n, _, d in Z.conv1_lanes(net)])
        lo, hi = Z.scaled_interval(want, want, 1.0)
        assert x.shape[1] == sum(c for _, c, _ in Z.conv1_lanes(net))
        assert np.array_equal(x[0], want.astype(F32)) and ((x[0] >= lo) & (x[0] <= hi)).all(), net
