"""GPU parity tests (run with -m gpu on an H100): every CUDA kernel family is called through the C ABI
(deepim_b200.context -> ctypes -> libdeepim_b200.so) and compared with the CPU oracle on the same
seeded inputs.  Bar: bit-exact for integer / index / mask work and for the fp32 geometry kernels
(compiled -fmad=false against an -ffp-contract=off oracle); float tolerances are written in each test.
Nothing here reads /root/reference."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # collected on the CPU box too; every test below needs the GPU
    pytest.skip("no CUDA device", allow_module_level=True)

from oracle import oracle as O  # noqa: E402
from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402

K = synth.K_LINEMOD
MEANS = synth.PIXEL_MEANS_RGB
MEANS32 = MEANS.astype(np.float32)
DEV = torch.device("cuda", 0)
H, W = 480, 640


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.fixture(scope="module")
def meshes():
    return [synth.make_cube(), synth.make_blob()]


@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(0)


@pytest.fixture(scope="module")
def ctx(meshes, weights):
    c = Context(0, max_batch=4, max_classes=4, max_verts=6000, max_faces=11000)
    for i, m in enumerate(meshes):
        c.upload_mesh(i, m)
    c.load_weights(weights)
    yield c
    c.close()


def observed_images(meshes, cls, obs):
    out = []
    for b in range(len(cls)):
        r = O.render(meshes[cls[b]], obs[b], K)
        out.append(synth.transform_image(synth.composite_observed(r["bgr"], r["mask"], b)))
    return np.stack(out)


# ------------------------------------------------------------------------------------------ raster
@pytest.mark.parametrize("trunc", [True, False])
def test_render_bit_exact(ctx, meshes, trunc):
    B = 4
    obs, ini = synth.sample_pose_pairs(B, 11)
    cls = np.array([0, 1, 1, 0], np.int32)
    out = ctx.render(dev(cls), dev(ini.astype(np.float32)), K, pixel_means_rgb=MEANS, trunc_u8=trunc,
                     want=("image", "depth", "mask", "bgr"))
    for b in range(B):
        r = O.render(meshes[cls[b]], ini[b], K, means_rgb=MEANS, trunc_u8=trunc)
        assert np.array_equal(out["bbox"][b].cpu().numpy(), r["bbox"])
        assert np.array_equal(out["mask"][b, 0].cpu().numpy(), r["mask"])
        assert np.array_equal(out["depth"][b, 0].cpu().numpy(), r["depth"])
        assert np.array_equal(out["image"][b].cpu().numpy(), r["image"])
        assert np.array_equal(out["bgr"][b].cpu().numpy(), r["bgr"])
        assert r["mask"].sum() > 500


def test_render_edge_cases(ctx, meshes):
    # partially outside the frame, fully outside (empty -> bbox -1), behind the near plane, and a
    # second render after it (visibility buffer must have been handed back empty)
    poses = np.zeros((4, 3, 4))
    poses[:, :, :3] = np.eye(3)
    poses[0, :, 3] = [0.42, 0.0, 0.8]     # cut by the right border
    poses[1, :, 3] = [3.0, 0.0, 0.8]      # out of view
    poses[2, :, 3] = [0.0, 0.0, 0.1]      # closer than ZNEAR (cube straddles z>0)
    poses[3, :, 3] = [0.0, -0.3, 0.8]     # cut by the top border
    cls = np.zeros(4, np.int32)
    for rep in range(2):
        out = ctx.render(dev(cls), dev(poses.astype(np.float32)), K, pixel_means_rgb=MEANS)
        for b in range(4):
            r = O.render(meshes[0], poses[b], K, means_rgb=MEANS)
            assert np.array_equal(out["bbox"][b].cpu().numpy(), r["bbox"])
            assert np.array_equal(out["mask"][b, 0].cpu().numpy(), r["mask"])
            assert np.array_equal(out["image"][b].cpu().numpy(), r["image"])
    assert list(out["bbox"][1].cpu().numpy()) == [-1, -1, -1, -1]
    assert out["mask"][0, 0, :, W - 1].sum() > 0 and out["mask"][3, 0, 0, :].sum() > 0


def test_render_large_triangles_warp_path(ctx):
    # a 12-triangle cube filling a third of the frame: every triangle takes the warp-cooperative path
    c2 = Context(0, max_batch=1, max_classes=1, max_verts=64, max_faces=64)
    m = synth.make_cube(side=0.3, nu=1, nv=1)
    c2.upload_mesh(0, m)
    obs, _ = synth.sample_pose_pairs(1, 5, z_mean=0.6)
    out = c2.render(dev(np.zeros(1, np.int32)), dev(obs.astype(np.float32)), K, pixel_means_rgb=MEANS)
    r = O.render(m, obs[0], K, means_rgb=MEANS)
    assert r["mask"].sum() > 30000
    assert np.array_equal(out["mask"][0, 0].cpu().numpy(), r["mask"])
    assert np.array_equal(out["depth"][0, 0].cpu().numpy(), r["depth"])
    assert np.array_equal(out["image"][0].cpu().numpy(), r["image"])
    c2.close()


# -------------------------------------------------------------------------------------------- zoom
@pytest.fixture(scope="module")
def zoom_inputs(ctx, meshes):
    B = 3
    obs, ini = synth.sample_pose_pairs(B, 21)
    cls = np.array([1, 0, 1], np.int32)
    ren = [O.render(meshes[cls[b]], ini[b], K, means_rgb=MEANS) for b in range(B)]
    mr = np.stack([r["mask"] for r in ren])[:, None]
    mo = np.stack([O.box_mask(r["bbox"], H, W) for r in ren])[:, None]
    img_r = np.stack([r["image"] for r in ren])
    img_o = observed_images(meshes, cls, obs)
    depth = np.stack([r["depth"] for r in ren])[:, None]
    return dict(B=B, obs=obs, ini=ini, cls=cls, mr=mr, mo=mo, img_r=img_r, img_o=img_o, depth=depth,
                pose32=ini.astype(np.float32))


def test_zoom_mask_bit_exact(ctx, zoom_inputs):
    z = zoom_inputs
    zo, zg, zr, zf, bbox, status = ctx.zoom_mask(dev(z["mo"]), dev(z["mo"]), dev(z["mr"]), dev(z["pose32"]), K)
    ozo, ozg, ozr, ozf, obb = O.zoom_mask(z["mo"], z["mo"], z["mr"], z["pose32"], K)
    assert np.array_equal(bbox.cpu().numpy(), obb)            # the 8 integer zoom bbox indices
    assert np.array_equal(zf.cpu().numpy(), ozf)              # float32 bit pattern
    assert np.array_equal(zo.cpu().numpy(), ozo) and np.array_equal(zg.cpu().numpy(), ozg)
    assert np.array_equal(zr.cpu().numpy(), ozr)
    assert status.cpu().numpy().tolist() == [0] * z["B"]


def test_zoom_mask_depth_as_mask_and_fallbacks(ctx, zoom_inputs):
    z = zoom_inputs
    # rendered "mask" given as a depth image (values in (0.2, 1]) is re-thresholded (zoom_mask.py:39-41)
    depth_as_mask = np.where(z["mr"] > 0, 0.73, 0.1).astype(np.float32)
    zo, zg, zr, zf, bbox, status = ctx.zoom_mask(dev(z["mo"]), dev(z["mo"]), dev(depth_as_mask), dev(z["pose32"]), K)
    ozo, ozg, ozr, ozf, obb = O.zoom_mask(z["mo"], z["mo"], depth_as_mask, z["pose32"], K)
    assert np.array_equal(bbox.cpu().numpy(), obb) and np.array_equal(zf.cpu().numpy(), ozf)
    assert np.array_equal(zr.cpu().numpy(), ozr)
    # empty rendered mask -> observed-box centre branch (zoom_mask.py:70-77)
    empty = np.zeros_like(z["mr"])
    _, _, zr2, zf2, bbox2, st2 = ctx.zoom_mask(dev(z["mo"]), dev(z["mo"]), dev(empty), dev(z["pose32"]), K)
    _, _, ozr2, ozf2, obb2 = O.zoom_mask(z["mo"], z["mo"], empty, z["pose32"], K)
    assert np.array_equal(bbox2.cpu().numpy(), obb2) and np.array_equal(zf2.cpu().numpy(), ozf2)
    assert zr2.abs().sum().item() == 0
    # empty observed mask: the reference raises; the device path flags it per instance
    _, _, _, _, bbox3, st3 = ctx.zoom_mask(dev(empty), dev(empty), dev(z["mr"]), dev(z["pose32"]), K)
    assert st3.cpu().numpy().tolist() == [1] * z["B"]
    assert np.all(bbox3.cpu().numpy()[:, :4] == -1)


def test_zoom_image_flow_depth_mask_ops_bit_exact(ctx, zoom_inputs):
    z = zoom_inputs
    _, _, _, ozf, _ = O.zoom_mask(z["mo"], z["mo"], z["mr"], z["pose32"], K)
    zf = dev(ozf)
    zio, zir = ctx.zoom_image_with_factor(zf, dev(z["img_o"]), dev(z["img_r"]), MEANS32)
    ozio, ozir = O.zoom_image_with_factor(ozf, z["img_o"], z["img_r"], MEANS32)
    assert np.array_equal(zio.cpu().numpy(), ozio) and np.array_equal(zir.cpu().numpy(), ozir)
    # out-of-frame samples come back as -mean (black), quirk App.B-6: with a crop wider than the frame (wx = 2) every output
    # whose four taps lie outside the frame is the sampler's 0 minus the float32 mean, exactly
    wide = np.array([[2.0, 2.0, 0.1, -0.05], [2.0, 2.0, -0.3, 0.2], [2.0, 2.0, 0.0, 0.0]], np.float32)
    zio2, zir2 = ctx.zoom_image_with_factor(dev(wide), dev(z["img_o"]), dev(z["img_r"]), MEANS32)
    one = np.float32(1)

    def taps_out(n, w, t):
        """outputs of one axis whose two taps c0, c0 + 1 both lie outside [0, n - 1] (src_coord's float32 sequence)"""
        ct = -one + np.arange(n, dtype=np.float32) * np.float32(2.0 / (n - 1))
        cr = ((w * ct + t + one) * np.float32(n - 1)) / np.float32(2)
        f0 = np.floor(cr)
        return (f0 + 1 < 0) | (f0 > n - 1)
    for b in range(z["B"]):
        out = taps_out(H, wide[b, 1], wide[b, 3])[:, None] | taps_out(W, wide[b, 0], wide[b, 2])[None, :]
        assert 0.2 * H * W < out.sum() < H * W
        for img in (zio2, zir2):
            for c in range(3):
                assert (img[b, c].cpu().numpy()[out] == -MEANS32[c]).all(), (b, c)
    for inv in (False, True):
        got = ctx.zoom_mask_with_factor(zf, dev(z["depth"]), inv)
        assert np.array_equal(got.cpu().numpy(), O.zoom_mask_with_factor(ozf, z["depth"], inv))
    rng = np.random.default_rng(3)
    flow = rng.normal(size=(z["B"], 2, H, W)).astype(np.float32) * 5
    fw = (rng.uniform(size=(z["B"], 1, H, W)) > 0.5).astype(np.float32)
    zfl, zfw = ctx.zoom_flow(zf, dev(flow), dev(fw), False)
    ofl, ofw = O.zoom_flow(ozf, flow, fw, False)
    assert np.array_equal(zfl.cpu().numpy(), ofl) and np.array_equal(zfw.cpu().numpy(), ofw)
    zfl2, none = ctx.zoom_flow(zf, dev(flow), None, True)
    ofl2, _ = O.zoom_flow(ozf, flow, None, True)
    assert none is None and np.array_equal(zfl2.cpu().numpy(), ofl2)
    zd1, zd2 = ctx.zoom_depth(zf, dev(z["depth"]), dev(z["depth"]))
    assert np.array_equal(zd1.cpu().numpy(), O.zoom_depth(ozf, z["depth"]))
    assert np.array_equal(zd1.cpu().numpy(), zd2.cpu().numpy())


def test_zoom_trans_and_box_mask(ctx):
    zf = np.array([[0.31, 0.31, 0.1, 0.0], [0.77, 0.77, -0.2, 0.3]], np.float32)
    t = np.array([[0.1, -0.2, 0.3], [0.013, 0.021, -0.034]], np.float32)
    for inv in (False, True):
        assert np.array_equal(ctx.zoom_trans(dev(zf), dev(t), inv).cpu().numpy(), O.zoom_trans(zf, t, inv))
    g = ctx.zoom_trans_backward(dev(zf), dev(t), True, True).cpu().numpy()
    assert np.array_equal(g, O.zoom_trans(zf, t, True))      # b_zoom_grad: same scaling as forward
    g = ctx.zoom_trans_backward(dev(zf), dev(t), True, False).cpu().numpy()
    assert np.array_equal(g, t)                              # b_zoom_grad False: pass-through
    bb = np.array([[10, 20, 5, 9], [-1, -1, -1, -1], [0, 639, 0, 479], [7, 7, 3, 30]], np.int32)
    m = ctx.update_mask_box(dev(bb)).cpu().numpy()
    for b in range(4):
        assert np.array_equal(m[b, 0], O.box_mask(bb[b], H, W))
    assert m[3].sum() == 0  # single-column mask -> empty end-exclusive rectangle


# --------------------------------------------------------------------------------------- geometry
def test_se3_compose_matches_reference_golden(ctx, golden_dir):
    g = np.load(os.path.join(golden_dir, "ref_se3.npz"))
    se3 = np.concatenate([g["quat"], g["trans"]], 1).astype(np.float32)
    for lo in range(0, 64, 4):
        ps = g["pose_src"][lo:lo + 4]
        for coord in ("MODEL", "CAMERA", "CAMERA_NEW"):
            out = ctx.se3_compose(dev(ps), dev(se3[lo:lo + 4]), g["T_means"], g["T_stds"], coord).cpu().numpy()
            for k in range(4):
                # the golden was produced from float64 quat/trans; feed the oracle the same float32 se3
                ref = O.rt_transform(ps[k], se3[lo + k, :4], se3[lo + k, 4:], g["T_means"], g["T_stds"], coord)
                np.testing.assert_allclose(out[k], ref, rtol=0, atol=1e-13)
                np.testing.assert_allclose(out[k], g["pose_out_norm_" + coord][lo + k], rtol=0, atol=1e-6)


def test_flow_bit_exact_and_reference_golden(ctx, meshes, golden_dir):
    B = 2
    obs, ini = synth.sample_pose_pairs(B, 31)
    d_src = np.stack([O.render(meshes[1], ini[b], K)["depth"] for b in range(B)])[:, None]
    d_tgt = np.stack([O.render(meshes[1], obs[b], K)["depth"] for b in range(B)])[:, None]
    K64 = K.astype(np.float64)
    KT = np.zeros((B, 3, 4), np.float32)
    for b in range(B):
        Rrel = obs[b, :, :3] @ ini[b, :, :3].T
        T = np.hstack([Rrel, (obs[b, :, 3] - Rrel @ ini[b, :, 3])[:, None]])
        KT[b] = (K64 @ T).astype(np.float32)
    Kinv = np.linalg.inv(K64).astype(np.float32)
    fl, va = ctx.flow(dev(d_src), dev(d_tgt), dev(KT), Kinv)
    ofl, ova = O.flow(d_src, d_tgt, KT, Kinv)
    assert ova.sum() > 1000
    assert np.array_equal(va.cpu().numpy(), ova) and np.array_equal(fl.cpu().numpy(), ofl)
    # small golden case generated from the reference's calc_flow (lib/pair_matching/flow.py)
    f = np.load(os.path.join(golden_dir, "ref_flow.npz"))
    c2 = Context(0, max_batch=1, height=60, width=80, max_classes=1, max_verts=8, max_faces=8)
    Rs, ts, Rt, tt = f["pose_src"][:, :3], f["pose_src"][:, 3], f["pose_tgt"][:, :3], f["pose_tgt"][:, 3]
    T = np.hstack([Rt @ Rs.T, (tt - Rt @ Rs.T @ ts)[:, None]])
    KTs = (f["K"] @ T).astype(np.float32)[None]
    fl2, va2 = c2.flow(dev(f["depth_src"][None, None]), dev(f["depth_tgt"][None, None]), dev(KTs),
                       np.linalg.inv(f["K"]).astype(np.float32))
    vis = f["visible"]
    assert int((va2.cpu().numpy()[0, 0] != vis).sum()) == 0
    assert np.abs(fl2.cpu().numpy()[0][:, vis == 1] - f["flow"].transpose(2, 0, 1)[:, vis == 1]).max() < 5e-5
    c2.close()
    # the reference's own CUDA kernel (lib/flow_c/gpu_flow_kernel.cu compiled unmodified, oracle/build_ref.py) on a rendered
    # 480 x 640 pair: identical validity mask, flow within 2 ulp of the pixel coordinate (FMA contraction of its build)
    g = np.load(os.path.join(golden_dir, "ref_flow_cuda.npz"))
    fl3, va3 = ctx.flow(dev(g["depth_src"]), dev(g["depth_tgt"]), dev(g["KT"]), g["Kinv"])
    assert np.array_equal(va3.cpu().numpy(), g["valid"]) and g["valid"].sum() > 5000
    assert np.abs(fl3.cpu().numpy() - g["flow"]).max() < 2.5e-4


def test_transform3d_forward_backward(ctx):
    # tolerances are the reference's own (transform3d.py:407 forward < 1e-4; l.421-539 grad thresh 5e-3)
    rng = np.random.default_rng(1)
    B, N = 3, 3000
    pts = (rng.normal(size=(B, 3, N)) * 0.05).astype(np.float32)
    q = rng.normal(size=(B, 4)) * 0.1 + np.array([1.0, 0, 0, 0])
    q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    t = (rng.normal(size=(B, 3)) * 0.05).astype(np.float32)
    _, ps = synth.sample_pose_pairs(B, 41)
    ps32 = ps.astype(np.float32)
    Tm, Ts = np.zeros(3, np.float32), np.ones(3, np.float32)
    og = rng.normal(size=(B, 3, N)).astype(np.float32)
    for coord in ("model", "camera"):
        out = ctx.transform3d(dev(pts), dev(q), dev(t), dev(ps32), Tm, Ts, coord).cpu().numpy()
        ref = O.transform3d_forward(pts, q, t, ps32, Tm, Ts, coord)
        assert np.abs(out - ref).max() < 1e-5
        for b in range(B):  # and against RT_transform itself, as the reference's self-test does
            P = O.rt_transform(ps[b], q[b], t[b], (0, 0, 0), (1, 1, 1), coord)
            assert np.abs(out[b] - (P[:, :3] @ pts[b] + P[:, 3:4])).max() < 1e-4
        rg, tg = ctx.transform3d_backward(dev(og), dev(pts), dev(q), dev(t), dev(ps32), Tm, Ts, coord)
        org, otg = O.transform3d_backward(og, pts, q, t, ps32, Tm, Ts, coord)
        scale = max(1.0, np.abs(org).max())
        assert np.abs(rg.cpu().numpy() - org).max() < 5e-3 * scale
        assert np.abs(tg.cpu().numpy() - otg).max() < 5e-3 * max(1.0, np.abs(otg).max())


def test_transform_image_u8(ctx):
    rng = np.random.default_rng(0)
    u8 = rng.integers(0, 256, size=(2, H, W, 3), dtype=np.uint8)
    out = ctx.transform_image_u8(dev(u8), MEANS).cpu().numpy()
    for b in range(2):
        assert np.array_equal(out[b], synth.transform_image(u8[b]))


# --------------------------------------------------------------------------------------------- net
def _net_inputs(zoom_inputs):
    z = zoom_inputs
    ozo, _, ozr, ozf, _ = O.zoom_mask(z["mo"], z["mo"], z["mr"], z["pose32"], K)
    ozio, ozir = O.zoom_image_with_factor(ozf, z["img_o"], z["img_r"], MEANS32)
    return ozio, ozir, ozo, ozr, ozf


def test_net_forward_parity_bf16x3(ctx, weights, zoom_inputs):
    """north_star tolerance on the regressed SE(3) delta: 1e-4 rot / 1e-3 trans (fp32-faithful mode:
    hi/lo bf16 split, three wgmma passes, fp32 accumulation in registers)."""
    zio, zir, zmo, zmr, _ = _net_inputs(zoom_inputs)
    rot, trans = ctx.net_forward(dev(zio), dev(zir), dev(zmo), dev(zmr), capi.PREC_BF16X3)
    orot, otrans, feats = O.net_forward(weights, zio, zir, zmo, zmr, return_features=True)
    assert np.abs(rot.cpu().numpy() - orot).max() < 1e-4
    assert np.abs(trans.cpu().numpy() - otrans).max() < 1e-3
    # and every layer of the tower (bf16 hi+lo activation pair vs fp32 torch), relative to its range
    names = ["flow_conv1", "conv2", "conv3", "conv3_1", "conv4", "conv4_1", "conv5", "conv5_1", "conv6", "conv6_1"]
    B = zio.shape[0]
    for i, n in enumerate(names):
        hi, g = ctx.debug_activation(i + 1, B, lo=False)
        lo, _ = ctx.debug_activation(i + 1, B, lo=True)
        py, px = g[3], g[4]
        f = feats[n]
        act = (hi + lo)[:, py:py + f.shape[2], px:px + f.shape[3], :].transpose(0, 3, 1, 2)
        assert np.abs(act - f).max() < 2e-4 * max(1.0, np.abs(f).max()), n
        border = hi.copy()
        border[:, py:py + f.shape[2], px:px + f.shape[3], :] = 0
        assert not border.any(), "zero border of %s input buffer was overwritten" % n


def test_net_forward_parity_fp16_headline_mode(ctx, weights, zoom_inputs):
    """DIM_PREC_FP16 = the mode bench.py reports: ONE wgmma pass with IEEE-half operands (11 significant bits),
    fp32 accumulation in registers.  Same north_star tolerance as the 3-pass mode: 1e-4 rot / 1e-3 trans.  Every layer is
    checked against the fp32 oracle relative to its range (half storage: 2^-11 per element, accumulated over the tower),
    the activations must stay far inside the half range (the stores saturate at 65504 instead of overflowing), and the
    zero borders of the shared 16-bit buffers must survive."""
    zio, zir, zmo, zmr, _ = _net_inputs(zoom_inputs)
    rot, trans = ctx.net_forward(dev(zio), dev(zir), dev(zmo), dev(zmr), capi.PREC_FP16)
    orot, otrans, feats = O.net_forward(weights, zio, zir, zmo, zmr, return_features=True)
    assert np.abs(rot.cpu().numpy() - orot).max() < 1e-4
    assert np.abs(trans.cpu().numpy() - otrans).max() < 1e-3
    names = ["flow_conv1", "conv2", "conv3", "conv3_1", "conv4", "conv4_1", "conv5", "conv5_1", "conv6", "conv6_1"]
    B = zio.shape[0]
    for i, n in enumerate(names):
        act, g = ctx.debug_activation(i + 1, B, fp16=True)
        py, px = g[3], g[4]
        f = feats[n]
        inner = act[:, py:py + f.shape[2], px:px + f.shape[3], :].transpose(0, 3, 1, 2)
        assert np.abs(f).max() < 65504.0 / 64, n                      # range headroom of the half format
        assert np.abs(inner - f).max() < 2.5e-3 * max(1.0, np.abs(f).max()), n
        border = act.copy()
        border[:, py:py + f.shape[2], px:px + f.shape[3], :] = 0
        assert not border.any(), "zero border of %s input buffer was overwritten" % n
    # the emulation of this storage format on the CPU oracle predicts the deviation (same order of magnitude)
    erot, etrans = O.net_forward(weights, zio, zir, zmo, zmr, emulate_fp16=True)
    assert np.abs(rot.cpu().numpy() - erot).max() < 1e-4 and np.abs(trans.cpu().numpy() - etrans).max() < 1e-4


def test_net_forward_bf16_fast_mode(ctx, weights, zoom_inputs):
    """Fast mode (single bf16 pass): cannot meet 1e-4 by construction (bf16 inputs carry 2^-9
    relative error per operand); bounded here at 2e-3 rot / 2e-3 trans.  NOT the mode bench.py's headline reports."""
    zio, zir, zmo, zmr, _ = _net_inputs(zoom_inputs)
    rot, trans = ctx.net_forward(dev(zio), dev(zir), dev(zmo), dev(zmr), capi.PREC_BF16)
    orot, otrans = O.net_forward(weights, zio, zir, zmo, zmr)
    assert np.abs(rot.cpu().numpy() - orot).max() < 2e-3
    assert np.abs(trans.cpu().numpy() - otrans).max() < 2e-3


def test_net_reload_weights_in_place(ctx, weights, zoom_inputs):
    """dim_net_load on a loaded context overwrites the operand packs in place (same storage, cached tensor maps stay valid)."""
    zio, zir, zmo, zmr, _ = _net_inputs(zoom_inputs)
    a = ctx.net_forward(dev(zio), dev(zir), dev(zmo), dev(zmr), capi.PREC_FP16)
    w2 = synth.make_weights(5)
    ctx.load_weights(w2)
    b = ctx.net_forward(dev(zio), dev(zir), dev(zmo), dev(zmr), capi.PREC_FP16)
    orot, otrans = O.net_forward(w2, zio, zir, zmo, zmr)
    assert np.abs(b[0].cpu().numpy() - orot).max() < 1e-4 and np.abs(b[1].cpu().numpy() - otrans).max() < 1e-3
    ctx.load_weights(weights)
    c = ctx.net_forward(dev(zio), dev(zir), dev(zmo), dev(zmr), capi.PREC_FP16)
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])


# ---------------------------------------------------------------------------------------- the loop
@pytest.fixture(scope="module")
def loop_case(meshes, weights):
    B = 4
    obs, ini = synth.sample_pose_pairs(B, 51)
    cls = np.array([0, 1, 1, 0], np.int32)
    img = observed_images(meshes, cls, obs)
    ref = O.refine(weights, meshes, cls, img, ini, K, 4, MEANS32)
    return dict(B=B, obs=obs, ini=ini, cls=cls, img=img, ref=ref)


@pytest.mark.parametrize("prec", [capi.PREC_FP16, capi.PREC_BF16X3], ids=["fp16", "bf16x3"])
def test_refine_teacher_forced_per_iteration(ctx, meshes, weights, loop_case, prec):
    """Each iteration started from the oracle's pose: integer bbox indices bit-exact, zoom_factor
    bit-exact, se3 within 1e-4 / 1e-3, composed pose within 1e-4 -- for the headline mode (fp16) and the 3-pass mode."""
    c = loop_case
    ref = c["ref"]
    override = np.concatenate([c["ini"][None], ref["poses"][:3]], 0)
    res = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, 4, pixel_means_rgb=MEANS,
                     precision=prec, pose_override=dev(override))
    assert np.array_equal(res["bbox"].cpu().numpy(), ref["bbox"])
    assert np.array_equal(res["zoom_factor"].cpu().numpy(), ref["zoom_factor"])
    se3 = res["se3"].cpu().numpy()
    assert np.abs(se3[..., :4] - ref["se3"][..., :4]).max() < 1e-4
    assert np.abs(se3[..., 4:] - ref["se3"][..., 4:]).max() < 1e-3
    assert np.abs(res["poses"].cpu().numpy() - ref["poses"]).max() < 1e-4


def test_refine_free_running_and_add(ctx, meshes, weights, loop_case):
    """Free-running 4 iterations.  bf16x3 and fp16 (headline): poses within 1e-3 of the oracle.  bf16 (fast mode):
    ADD / ADD-S of the final pose within 0.1 % of the object diameter of the oracle's, and the
    accuracy at 0.1 d identical (BASELINE.json: ADD(-S) within +-0.1 of the reference)."""
    c = loop_case
    ref = c["ref"]
    for prec, tol in ((capi.PREC_BF16X3, 1e-3), (capi.PREC_FP16, 1e-3), (capi.PREC_BF16, 1e-2)):
        res = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, 4, pixel_means_rgb=MEANS, precision=prec)
        poses = res["poses"].cpu().numpy()
        assert np.isfinite(poses).all()
        assert np.abs(poses - ref["poses"]).max() < tol
        acc_g, acc_o = [], []
        for b in range(c["B"]):
            m = meshes[c["cls"][b]]
            pts = m.verts.astype(np.float64)
            metric = O.adi_metric if c["cls"][b] == 0 else O.add_metric  # cube is symmetric -> ADD-S
            eg = metric(poses[3, b, :, :3], poses[3, b, :, 3], c["obs"][b, :, :3], c["obs"][b, :, 3], pts)
            eo = metric(ref["poses"][3, b, :, :3], ref["poses"][3, b, :, 3], c["obs"][b, :, :3], c["obs"][b, :, 3], pts)
            assert abs(eg - eo) < 1e-3 * m.diameter
            acc_g.append(eg < 0.1 * m.diameter)
            acc_o.append(eo < 0.1 * m.diameter)
        assert abs(100.0 * np.mean(acc_g) - 100.0 * np.mean(acc_o)) <= 0.1


def test_refine_is_deterministic_and_batch_consistent(ctx, loop_case):
    c = loop_case
    args = (dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, 4)
    a = ctx.refine(*args, pixel_means_rgb=MEANS, precision=capi.PREC_FP16)
    b = ctx.refine(*args, pixel_means_rgb=MEANS, precision=capi.PREC_FP16)
    for k in ("poses", "se3", "bbox", "zoom_factor"):
        assert torch.equal(a[k], b[k]), k                      # idempotent: no atomics on float data
    # instances are independent: a permuted batch gives permuted results (same tiling -> same bits)
    perm = [2, 0, 3, 1]
    p = ctx.refine(dev(c["img"][perm]), dev(c["cls"][perm]), dev(c["ini"][perm]), K, 4, pixel_means_rgb=MEANS,
                   precision=capi.PREC_FP16)
    assert torch.equal(p["bbox"], a["bbox"][:, perm])
    assert (p["poses"] - a["poses"][:, perm]).abs().max().item() < 1e-5
    # a single instance alone: every output of the chain is reduced in an order fixed per instance (the conv tiles' K steps,
    # fc6's mma rows and its split partials summed in order), whatever the batch size and the launch shapes it picks, so
    # the instance's results are the same bits (tests/test_gpu_schedule.py holds this across SM counts and past B = 16)
    for prec in (capi.PREC_BF16X3, capi.PREC_FP16, capi.PREC_BF16):
        full = ctx.refine(*args, pixel_means_rgb=MEANS, precision=prec)
        s = ctx.refine(dev(c["img"][1:2]), dev(c["cls"][1:2]), dev(c["ini"][1:2]), K, 4, pixel_means_rgb=MEANS,
                       precision=prec)
        for k in ("poses", "se3", "bbox", "zoom_factor"):
            assert torch.equal(s[k][:, 0], full[k][:, 1]), (prec, k)


def test_refine_cuda_graph_replay_equals_eager(ctx, loop_case):
    """With the caller's buffers reused (`out=`) on a non-default stream the library captures the 4-iteration chain into a
    CUDA graph on the second call and replays it afterwards: results must be bit-identical to the eagerly enqueued chain,
    and new inputs written into the same buffers must be honoured by the replay."""
    from deepim_b200._capi import check, lib
    c = loop_case
    img, cls, ini = dev(c["img"]), dev(c["cls"]), dev(c["ini"])
    check(lib.dim_debug_set_option(ctx._h, b"graph", 0))
    eager = ctx.refine(img, cls, ini, K, 4, pixel_means_rgb=MEANS)
    eager_bf = ctx.refine(img, cls, ini, K, 4, pixel_means_rgb=MEANS, precision=capi.PREC_BF16X3)
    assert not torch.equal(eager_bf["se3"], eager["se3"])
    ini2 = dev(c["ini"][[1, 0, 3, 2]])
    cls2 = dev(c["cls"][[1, 0, 3, 2]])
    img2 = dev(c["img"][[1, 0, 3, 2]])
    eager2 = ctx.refine(img2, cls2, ini2, K, 4, pixel_means_rgb=MEANS)
    torch.cuda.synchronize()       # a context is driven from ONE stream at a time: finish the default-stream work first
    check(lib.dim_debug_set_option(ctx._h, b"graph", 1))
    side = torch.cuda.Stream(device=DEV)
    out = None
    for it in range(4):            # eager warm-up, capture + launch, replay, replay -- for each chain
        # the same buffers with only a by-value argument (the precision) changed must get a graph of their own
        for want, kw in ((eager, {}), (eager_bf, {"precision": capi.PREC_BF16X3})):
            with torch.cuda.stream(side):
                out = ctx.refine(img, cls, ini, K, 4, pixel_means_rgb=MEANS, out=out, **kw)
            side.synchronize()
            for k in ("poses", "se3", "zoom_factor", "bbox"):
                assert torch.equal(out[k], want[k]), (it, k, kw)
    with torch.cuda.stream(side):  # same addresses, new contents: the replayed graph reads the buffers, not captured values
        img.copy_(img2); cls.copy_(cls2); ini.copy_(ini2)
        out = ctx.refine(img, cls, ini, K, 4, pixel_means_rgb=MEANS, out=out)
    side.synchronize()
    for k in ("poses", "se3", "zoom_factor", "bbox"):
        assert torch.equal(out[k], eager2[k]), k
    torch.cuda.synchronize()


def test_refine_follows_config_pose_parameterisation(ctx, loop_case):
    """dim_refine composes each iteration's pose under the context's trans_means / trans_stds / rot_coord: poses[i+1] =
    rt_transform(poses[i], se3[i]) in float64 with the values set, eagerly and on graph replay; a second set_config with the
    same buffers reaches the replay (set_config drops the captured chains)."""
    from deepim_b200._capi import check, lib
    c = loop_case
    img, cls, ini = dev(c["img"]), dev(c["cls"]), dev(c["ini"])
    cfg0 = ctx.get_config()

    def holds(out, cfg, what):
        poses, se3 = out["poses"].cpu().numpy(), out["se3"].cpu().numpy()
        src = c["ini"]
        for it in range(poses.shape[0]):
            for b in range(c["B"]):
                ref = O.rt_transform(src[b], se3[it, b, :4], se3[it, b, 4:], cfg["trans_means"], cfg["trans_stds"], cfg["rot_coord"])
                assert np.abs(poses[it, b] - ref).max() <= 1e-12 * np.abs(ref).max(), (what, it, b)
            src = poses[it]

    side = torch.cuda.Stream(device=DEV)
    try:
        default = ctx.refine(img, cls, ini, K, 4, pixel_means_rgb=MEANS)
        out = None
        for new in ({"trans_means": (0.0625, -0.125, 0.03125), "trans_stds": (0.5, 2.0, 0.75), "rot_coord": "MODEL"},
                    {"trans_means": (-0.03125, 0.0625, -0.0625), "trans_stds": (1.5, 0.25, 2.0), "rot_coord": "MODEL"}):
            torch.cuda.synchronize()
            ctx.set_config(**new)
            cfg = ctx.get_config()
            check(lib.dim_debug_set_option(ctx._h, b"graph", 0))
            eager = ctx.refine(img, cls, ini, K, 4, pixel_means_rgb=MEANS)
            holds(eager, cfg, "eager")
            assert not torch.equal(eager["poses"], default["poses"])
            torch.cuda.synchronize()
            check(lib.dim_debug_set_option(ctx._h, b"graph", 1))
            for it in range(3):  # eager warm-up, capture + launch, replay -- on the buffers of the previous config's graph
                with torch.cuda.stream(side):
                    out = ctx.refine(img, cls, ini, K, 4, pixel_means_rgb=MEANS, out=out)
                side.synchronize()
                holds(out, cfg, "graph %d" % it)
                assert torch.equal(out["poses"], eager["poses"]), it
    finally:
        torch.cuda.synchronize()
        check(lib.dim_debug_set_option(ctx._h, b"graph", 1))
        ctx.set_config(**cfg0)


def test_refine_host_matches_device_path(ctx, meshes, loop_case):
    c = loop_case
    B = c["B"]
    u8 = []
    for b in range(B):
        r = O.render(meshes[c["cls"][b]], c["obs"][b], K)
        u8.append(synth.composite_observed(r["bgr"], r["mask"], b))
    u8 = np.stack(u8)
    poses, se3 = ctx.refine_host(u8, c["cls"], c["ini"], K, 4, pixel_means_rgb=MEANS, precision=capi.PREC_FP16)
    d = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, 4, pixel_means_rgb=MEANS, precision=capi.PREC_FP16)
    assert np.array_equal(poses, d["poses"].cpu().numpy())
    assert np.array_equal(se3, d["se3"].cpu().numpy())


def test_errors_are_loud(ctx):
    with pytest.raises(capi.DeepIMError):
        ctx.refine(torch.zeros(5, 3, H, W, device=DEV), torch.zeros(5, dtype=torch.int32, device=DEV),
                   torch.zeros(5, 3, 4, dtype=torch.float64, device=DEV), K, 4)  # batch > max_batch
    with pytest.raises((TypeError, ValueError)):
        ctx.zoom_trans(torch.zeros(2, 4, device=DEV), torch.zeros(2, 3, dtype=torch.float64, device=DEV), True)


def test_bad_class_index_and_lost_object_are_flagged(ctx, meshes, weights, loop_case):
    """Class indices are range-checked (the reference indexes a python list and raises): on the host entry point the call
    fails; on the device entry point the instance renders nothing and is flagged (status bit 1).  An object that leaves the
    view frustum gives an empty rendered mask: the reference crashes in ZoomMask (np.min of an empty array), here the
    iteration is flagged (bit 0) and PoseRefiner.result() raises."""
    from deepim_b200.refiner import PoseRefiner
    c = loop_case
    u8 = np.zeros((c["B"], H, W, 3), np.uint8)
    bad = c["cls"].copy()
    bad[2] = 7                                         # ctx has max_classes = 4
    with pytest.raises(capi.DeepIMError):
        ctx.refine_host(u8, bad, c["ini"], K, 2, pixel_means_rgb=MEANS)
    bad[2] = 3                                         # in range, but no mesh uploaded for class 3
    with pytest.raises(capi.DeepIMError):
        ctx.refine_host(u8, bad, c["ini"], K, 2, pixel_means_rgb=MEANS)
    res = ctx.refine(dev(c["img"]), dev(bad), dev(c["ini"]), K, 2, pixel_means_rgb=MEANS)
    st = ctx.refine_status(c["B"], 2).numpy()
    assert np.isfinite(res["poses"].cpu().numpy()[:, [0, 1, 3]]).all()
    assert (st[:, 2] & 2).all() and not (st[:, [0, 1, 3]] & 2).any()
    # the good instances are untouched by their bad neighbour
    good = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, 2, pixel_means_rgb=MEANS)
    assert torch.equal(good["poses"][:, [0, 1, 3]], res["poses"][:, [0, 1, 3]])
    assert not ctx.refine_status(c["B"], 2).numpy().any()
    # object far outside the frame
    lost = c["ini"].copy()
    lost[1, 0, 3] = 5.0
    ref = PoseRefiner(meshes, weights, K, device=0, max_batch=4, n_iter=2, n_slots=1)
    t = ref.submit(u8, c["cls"], lost)
    with pytest.raises(capi.DeepIMError):
        ref.result(t)
    t = ref.submit(u8, c["cls"], lost)
    ref.result(t, strict=False)
    assert (ref.last_status[:, 1] & 1).all() and not ref.last_status[:, [0, 2, 3]].any()
    ref.close()


# ------------------------------------------------------------------- BASELINE.json configs C3 / C5
def test_config_c3_thirteen_meshes_sharded_batch(weights):
    """C3: 13 LINEMOD-scale meshes, instances round-robin over classes, batch split into device batches
    (the 8-GPU sharding itself is covered by tests/test_sharding_gloo.py; instances are independent, so a
    rank's slice is just such a batch).  Integer bboxes bit-exact, poses within tolerance."""
    from deepim_b200.refiner import PoseRefiner
    meshes13 = synth.make_linemod_like_set(13, seed=2)
    n = 13
    obs, ini = synth.sample_pose_pairs(n, 61)
    cls = np.arange(n, dtype=np.int32) % 13
    u8 = []
    for b in range(n):
        r = O.render(meshes13[cls[b]], obs[b], K)
        u8.append(synth.composite_observed(r["bgr"], r["mask"], b))
    u8 = np.stack(u8)
    ref = PoseRefiner(meshes13, weights, K, device=0, max_batch=8, n_iter=2, precision="bf16x3", n_slots=2)
    poses = ref.refine(u8, cls, ini)                       # 2 device batches (8 + 5), pipelined
    ref.close()
    img = np.stack([synth.transform_image(u8[b]) for b in range(n)])
    oref = O.refine(weights, meshes13, cls, img, ini, K, 2, MEANS32)
    assert poses.shape == (2, n, 3, 4)
    assert np.abs(poses - oref["poses"]).max() < 1e-3
    # first-iteration poses depend only on exact integer/bbox work + the net: tight tolerance
    assert np.abs(poses[0] - oref["poses"][0]).max() < 1e-4


def test_config_c5_50k_vertex_mesh_render_and_refine(weights):
    """C5 stress mesh (~50k verts / 100k tris, diameter 0.25 m at 0.6 m): rasteriser bit-exact on
    sub-pixel triangles, one refinement iteration within tolerance."""
    big = synth.make_blob(158, 316, diameter=0.25, tex_size=512, seed=4, name="stress")
    assert len(big.verts) > 50000 and len(big.faces) > 99000
    c5 = Context(0, max_batch=2, max_classes=1, max_verts=len(big.verts), max_faces=len(big.faces))
    c5.upload_mesh(0, big)
    c5.load_weights(weights)
    obs, ini = synth.sample_pose_pairs(2, 71, z_mean=0.6)
    cls = np.zeros(2, np.int32)
    out = c5.render(dev(cls), dev(ini.astype(np.float32)), K, pixel_means_rgb=MEANS, want=("image", "depth", "mask"))
    for b in range(2):
        r = O.render(big, ini[b], K, means_rgb=MEANS)
        assert r["mask"].sum() > 20000
        assert np.array_equal(out["bbox"][b].cpu().numpy(), r["bbox"])
        assert np.array_equal(out["mask"][b, 0].cpu().numpy(), r["mask"])
        assert np.array_equal(out["depth"][b, 0].cpu().numpy(), r["depth"])
        assert np.array_equal(out["image"][b].cpu().numpy(), r["image"])
    img = observed_images([big], cls, obs)
    res = c5.refine(dev(img), dev(cls), dev(ini), K, 1, pixel_means_rgb=MEANS, precision=capi.PREC_BF16X3)
    oref = O.refine(weights, [big], cls, img, ini, K, 1, MEANS32)
    assert np.array_equal(res["bbox"].cpu().numpy(), oref["bbox"])
    assert np.abs(res["se3"].cpu().numpy()[..., :4] - oref["se3"][..., :4]).max() < 1e-4
    assert np.abs(res["se3"].cpu().numpy()[..., 4:] - oref["se3"][..., 4:]).max() < 1e-3
    c5.close()


# ------------------------------------------------------------------------- train-time update (a14)
def test_train_update_matches_oracle(ctx, meshes, golden_dir):
    """batchUpdaterPyMulti.forward on the device: refined pose, train-path render (no uint8 truncation,
    float32 mean subtraction), labels rot (mat2quat) / trans, reprojection flow + tiled weights."""
    B = 3
    obs, ini = synth.sample_pose_pairs(B, 81)
    cls = np.array([1, 0, 1], np.int32)
    rng = np.random.default_rng(7)
    rot_est = (np.array([1.0, 0, 0, 0]) + rng.normal(size=(B, 4)) * 0.03).astype(np.float32)
    trans_est = (rng.normal(size=(B, 3)) * 0.01).astype(np.float32)
    src32, tgt32 = ini.astype(np.float32), obs.astype(np.float32)
    depth_gt = np.stack([O.render(meshes[cls[b]], obs[b], K)["depth"] for b in range(B)])[:, None]
    out = ctx.train_update(dev(cls), dev(src32), dev(rot_est), dev(trans_est), dev(tgt32), dev(depth_gt), K,
                           pixel_means_rgb=MEANS)
    ref = O.train_update(meshes, cls, src32, rot_est, trans_est, tgt32, depth_gt, K, MEANS)
    assert np.abs(out["src_pose"].cpu().numpy() - ref["src_pose"]).max() < 1e-6
    assert np.abs(out["rot"].cpu().numpy() - ref["rot"]).max() < 1e-6     # Jacobi vs LAPACK eigh, float32 store
    assert np.abs(out["trans"].cpu().numpy() - ref["trans"]).max() < 1e-6
    # the refined pose is float64 on both sides and rounds to the same float32 -> renders are bit-exact
    if np.array_equal(out["src_pose"].cpu().numpy(), ref["src_pose"]):
        assert np.array_equal(out["mask_rendered"].cpu().numpy(), ref["mask_rendered"])
        assert np.array_equal(out["depth_rendered"].cpu().numpy(), ref["depth_rendered"])
        assert np.array_equal(out["image_rendered"].cpu().numpy(), ref["image_rendered"])
    else:
        assert (out["mask_rendered"].cpu().numpy() != ref["mask_rendered"]).mean() < 1e-4
    fw, ofw = out["flow_weights"].cpu().numpy(), ref["flow_weights"]
    assert np.array_equal(fw[:, 0], fw[:, 1]) and ofw.sum() > 1000
    assert (fw != ofw).mean() < 2e-4       # KT differs at float32 rounding level -> a few threshold pixels
    both = (fw[:, :1] == 1) & (ofw[:, :1] == 1)
    assert np.abs(out["flow"].cpu().numpy() - ref["flow"])[np.repeat(both, 2, 1)].max() < 2e-3
    # labels are consistent: composing the label delta onto the refined pose gives the target pose
    for b in range(B):
        back = O.rt_transform(ref["src_pose"][b].astype(np.float64), out["rot"][b].cpu().numpy(),
                              out["trans"][b].cpu().numpy(), (0, 0, 0), (1, 1, 1), "camera")
        assert np.abs(back - tgt32[b]).max() < 1e-5
