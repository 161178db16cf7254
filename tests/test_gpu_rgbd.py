"""GPU: the RGB-D network (config.network.INPUT_DEPTH) in the fused refinement loop and on the op surface -- dim_refine,
dim_refine_host_async and dim_net_fwd of an RGB-D context against the oracle's RGB-D loop (oracle.refine with depth_observed), against
the RGB context
where the depth weights are zero, and the error paths of the mode switch."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from oracle import oracle as O  # noqa: E402
from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import lighting, synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402

K = synth.K_LINEMOD
MEANS = synth.PIXEL_MEANS_RGB
DEV = torch.device("cuda", 0)
H, W = 480, 640
N_ITER = 4
B = 16


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.fixture(scope="module")
def meshes():
    ms = [synth.make_cube(), synth.make_blob()]
    for m in ms:
        m.normals = synth.vertex_normals(m)
    return ms


@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(0, input_depth=True)


def make_ctx(meshes, weights, input_depth=True):
    c = Context(0, max_batch=B, max_classes=4, max_verts=6000, max_faces=11000, input_depth=input_depth)
    for i, m in enumerate(meshes):
        c.upload_mesh(i, m)
    c.load_weights(weights)
    return c


@pytest.fixture(scope="module")
def ctx(meshes, weights):
    c = make_ctx(meshes, weights)
    yield c
    c.close()


@pytest.fixture(scope="module")
def case(meshes, weights):
    """B = 16 observed frames: the render at the observed pose composited over noise, and a sensor-like depth (the render's
    depth plus 2 mm noise on the object, a 1-2 m background elsewhere) stored as millimetre uint16 like LINEMOD's files."""
    obs, ini = synth.sample_pose_pairs(B, 23)
    cls = np.array([b % 2 for b in range(B)], np.int32)
    rng = np.random.default_rng(5)
    u8, dep = [], []
    for b in range(B):
        r = O.render(meshes[cls[b]], obs[b], K, means_rgb=MEANS)
        u8.append(synth.composite_observed(r["bgr"], r["mask"], b))
        d = np.where(r["depth"] > 0, r["depth"] + rng.normal(0, 0.002, r["depth"].shape), rng.uniform(1.0, 2.0, r["depth"].shape))
        dep.append(np.clip(np.rint(d * 1000.0), 0, 65535).astype(np.uint16))
    u8, u16 = np.stack(u8), np.stack(dep)
    img = np.stack([synth.transform_image(u8[b]) for b in range(B)])
    depth = O.depth_from_u16(u16, 1000.0)[:, None]
    # float64 means, as the device gets them: the checker's render subtracts them in float64 like the device's
    ref = O.refine(weights, meshes, cls, img, ini, K, N_ITER, MEANS, depth_observed=depth, return_inputs=True)
    return dict(obs=obs, ini=ini, cls=cls, u8=u8, u16=u16, img=img, depth=depth, ref=ref)


def teacher(case):
    return dev(np.concatenate([case["ini"][None], case["ref"]["poses"][:N_ITER - 1]], 0))


@pytest.mark.parametrize("prec", [capi.PREC_FP16, capi.PREC_BF16X3], ids=["fp16", "bf16x3"])
def test_conv1_input_equals_the_checker_blob(ctx, case, prec):
    """The zoomed 10-channel conv1 input of iteration 0, read back from the space-to-depth buffer, equals the checker's blob
    after 16-bit rounding, bit for bit, depth channels included (bf16x3: both halves)."""
    c = case
    ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, 1, pixel_means_rgb=MEANS, precision=prec,
               depth_observed=dev(c["depth"]))
    torch.cuda.synchronize()
    z = c["ref"]["inputs"][0]
    x = O.conv1_input(z["zio"], z["zir"], z["zdo"], z["zdr"], z["zmo"], z["zmr"])  # [B,10,H,W]
    f16 = prec == capi.PREC_FP16
    hi, g = ctx.debug_activation(0, B, fp16=f16)
    rows, cols, ch, pad = g[0], g[1], g[2], g[3]
    assert ch == 64
    hi = hi.reshape(B, rows, 8, cols, 8)
    xp = np.zeros((B, 16, 2 * rows, 2 * cols), np.float32)
    xp[:, :10, pad:pad + H, pad:pad + W] = x
    # plane (ph*2 + pw)*2 + half holds channels half*8 .. +7 of pixel (2r + ph, 2c + pw)
    exp = xp.reshape(B, 2, 8, rows, 2, cols, 2).transpose(0, 3, 4, 6, 1, 5, 2).reshape(B, rows, 8, cols, 8)
    rnd = (lambda a: a.astype(np.float16).astype(np.float32)) if f16 else \
        (lambda a: torch.from_numpy(a).bfloat16().float().numpy())
    def same(got, want):
        bad = got != want
        where = {"plane %d ch %d" % (pl, c): (int(bad[:, :, pl, :, c].sum()),
                                             float(np.abs(got - want)[:, :, pl, :, c].max()))
                 for pl in range(8) for c in range(8) if bad[:, :, pl, :, c].any()}
        assert not where, where

    same(hi, rnd(exp))
    assert np.abs(exp[:, :, [0, 2, 4, 6], :, 6:8]).max() > 0  # the depth channels are populated
    if prec == capi.PREC_BF16X3:
        lo, _ = ctx.debug_activation(0, B, lo=True)
        same(lo.reshape(B, rows, 8, cols, 8), rnd(exp - rnd(exp)))


@pytest.mark.parametrize("prec", [capi.PREC_FP16, capi.PREC_BF16X3], ids=["fp16", "bf16x3"])
def test_rgbd_refine_teacher_forced_per_iteration(ctx, case, prec):
    c, ref = case, case["ref"]
    res = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS, precision=prec,
                     pose_override=teacher(c), depth_observed=dev(c["depth"]))
    assert np.array_equal(res["bbox"].cpu().numpy(), ref["bbox"])
    assert np.array_equal(res["zoom_factor"].cpu().numpy(), ref["zoom_factor"])
    se3 = res["se3"].cpu().numpy()
    assert np.abs(se3[..., :4] - ref["se3"][..., :4]).max() < 1e-4
    assert np.abs(se3[..., 4:] - ref["se3"][..., 4:]).max() < 1e-3
    assert np.abs(res["poses"].cpu().numpy() - ref["poses"]).max() < 1e-4
    assert not ctx.refine_status(B, N_ITER).numpy().any()


def test_rgbd_refine_free_running_fp16(ctx, case):
    c = case
    res = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS,
                     precision=capi.PREC_FP16, depth_observed=dev(c["depth"]))
    poses = res["poses"].cpu().numpy()
    assert np.isfinite(poses).all()
    assert np.abs(poses - c["ref"]["poses"]).max() < 1e-3


def test_zero_depth_weights_give_the_rgb_context(meshes, case):
    """The RGB-D network with all-zero depth columns is the RGB network: bbox and zoom factor bit for bit, se3 within 1e-5."""
    c = case
    w8 = synth.make_weights(0)
    rgb, rgbd = make_ctx(meshes, w8, False), make_ctx(meshes, synth.with_depth_channels(w8))
    try:
        for prec in (capi.PREC_FP16, capi.PREC_BF16X3):
            a = rgb.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS, precision=prec,
                           pose_override=teacher(c))
            b = rgbd.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS, precision=prec,
                            pose_override=teacher(c), depth_observed=dev(c["depth"]))
            assert torch.equal(a["bbox"], b["bbox"]) and torch.equal(a["zoom_factor"], b["zoom_factor"])
            assert (a["se3"] - b["se3"]).abs().max().item() < 1e-5, prec
    finally:
        rgb.close()
        rgbd.close()


def test_depth_is_wired_in(ctx, case):
    """Raising depth_observed inside instance 0's zoom window changes its se3, and only its."""
    c = case
    args = (dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, 1)
    base = ctx.refine(*args, pixel_means_rgb=MEANS, depth_observed=dev(c["depth"]))["se3"].clone()
    d2 = c["depth"].copy()
    x0, x1, y0, y1 = c["ref"]["bbox"][0, 0, 4:]
    d2[0, 0, y0:y1 + 1, x0:x1 + 1] += np.float32(0.05)
    moved = ctx.refine(*args, pixel_means_rgb=MEANS, depth_observed=dev(d2))["se3"]
    assert (moved[0, 0] - base[0, 0]).abs().max().item() > 1e-6
    assert torch.equal(moved[0, 1:], base[0, 1:])


def test_rgbd_graph_replay_equals_eager(ctx, case):
    """Warm-up, capture and replay of the RGB-D chain give the eager bits; another depth buffer is another graph."""
    c = case
    img, cls, ini = dev(c["img"]), dev(c["cls"]), dev(c["ini"])
    d1 = dev(c["depth"])
    d2 = d1 + 0.03
    ctx_eager = []
    check = capi.check
    check(capi.lib.dim_debug_set_option(ctx._h, b"graph", 0))
    for d in (d1, d2):
        ctx_eager.append({k: v.clone() for k, v in
                          ctx.refine(img, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, depth_observed=d).items()})
    check(capi.lib.dim_debug_set_option(ctx._h, b"graph", 1))
    out = None
    for rep in range(3):
        for i, d in enumerate((d1, d2)):
            out = ctx.refine(img, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, depth_observed=d, out=out)
            for k in ("poses", "se3", "zoom_factor", "bbox"):
                assert torch.equal(out[k], ctx_eager[i][k]), (rep, i, k)
    assert not torch.equal(ctx_eager[0]["se3"], ctx_eager[1]["se3"])


def test_host_entry_equals_device_entry(ctx, case):
    c = case
    dres = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS,
                      depth_observed=dev(c["depth"]))
    poses, se3 = ctx.refine_host(c["u8"], c["cls"], c["ini"], K, N_ITER, pixel_means_rgb=MEANS,
                                 depth_observed_u16=c["u16"], depth_factor=1000.0)
    assert np.array_equal(poses, dres["poses"].cpu().numpy())
    assert np.array_equal(se3, dres["se3"].cpu().numpy())


def test_lit_and_depth_together(ctx, meshes, weights, case):
    c = case
    inten = lighting.sample_intensity(np.random.default_rng(3), (N_ITER, B))
    lit = {"intensity": inten, "offset": lighting.OFFSET, "brightness_ratio": 0.7}
    ref = O.refine(weights, meshes, c["cls"], c["img"], c["ini"], K, N_ITER, MEANS,
                   poses_override=[c["ini"]] + [c["ref"]["poses"][i] for i in range(N_ITER - 1)], lighting=lit,
                   depth_observed=c["depth"])
    res = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS, precision=capi.PREC_FP16,
                     pose_override=teacher(c), depth_observed=dev(c["depth"]), lighting=dict(lit, intensity=dev(inten)))
    assert np.array_equal(res["bbox"].cpu().numpy(), ref["bbox"])
    assert np.array_equal(res["zoom_factor"].cpu().numpy(), ref["zoom_factor"])
    se3 = res["se3"].cpu().numpy()
    assert np.abs(se3[..., :4] - ref["se3"][..., :4]).max() < 1e-4
    assert np.abs(se3[..., 4:] - ref["se3"][..., 4:]).max() < 1e-3
    assert np.abs(res["poses"].cpu().numpy() - ref["poses"]).max() < 1e-4


@pytest.mark.parametrize("prec", [capi.PREC_FP16, capi.PREC_BF16X3], ids=["fp16", "bf16x3"])
def test_net_fwd_rgbd_matches_the_checker(ctx, weights, case, prec):
    z = case["ref"]["inputs"][0]
    rot, trans = ctx.net_forward(dev(z["zio"]), dev(z["zir"]), dev(z["zmo"]), dev(z["zmr"]), precision=prec,
                                 zoom_depth_observed=dev(z["zdo"]), zoom_depth_rendered=dev(z["zdr"]))
    rr, tr = O.net_forward(weights, z["zio"], z["zir"], z["zmo"], z["zmr"], zdo=z["zdo"], zdr=z["zdr"])
    assert np.abs(rot.cpu().numpy() - rr).max() < 1e-4
    assert np.abs(trans.cpu().numpy() - tr).max() < 1e-3


def test_depth_arguments_follow_the_network_error_paths(meshes, weights, case):
    c = case
    w8 = synth.make_weights(0)
    rgb = make_ctx(meshes, w8, False)
    rgbd = make_ctx(meshes, weights)
    try:
        args = (dev(c["img"][:2]), dev(c["cls"][:2]), dev(c["ini"][:2]), K, 1)
        with pytest.raises(capi.DeepIMError, match="takes depth input.*depth_frames must not be NULL"):
            rgbd.refine(*args, pixel_means_rgb=MEANS)
        with pytest.raises(capi.DeepIMError, match="takes no depth input"):
            rgb.refine(*args, pixel_means_rgb=MEANS, depth_observed=dev(c["depth"][:2]))
        with pytest.raises(capi.DeepIMError, match="takes depth input.*depth_frames_u16_host"):
            rgbd.refine_host(c["u8"][:2], c["cls"][:2], c["ini"][:2], K, 1, pixel_means_rgb=MEANS)
        with pytest.raises(capi.DeepIMError, match="takes no depth input"):
            rgb.refine_host(c["u8"][:2], c["cls"][:2], c["ini"][:2], K, 1, pixel_means_rgb=MEANS,
                            depth_observed_u16=c["u16"][:2])
        z = c["ref"]["inputs"][0]
        with pytest.raises(capi.DeepIMError, match="takes depth input.*zoom_depth_observed"):
            rgbd.net_forward(dev(z["zio"][:2]), dev(z["zir"][:2]), dev(z["zmo"][:2]), dev(z["zmr"][:2]))
        with pytest.raises(capi.DeepIMError, match="takes no depth input"):
            rgb.net_forward(dev(z["zio"][:2]), dev(z["zir"][:2]), dev(z["zmo"][:2]), dev(z["zmr"][:2]),
                            zoom_depth_observed=dev(z["zdo"][:2]), zoom_depth_rendered=dev(z["zdr"][:2]))
        # NULL depth
        poses = torch.empty((1, 2, 3, 4), dtype=torch.float64, device=DEV)
        rc = capi.lib.dim_refine(rgbd._h, C.c_void_p(args[0].data_ptr()), 2, None,
                                 capi.farr(np.asarray(K, np.float32).reshape(9), 9), None, C.c_void_p(args[1].data_ptr()),
                                 C.c_void_p(args[2].data_ptr()), 2, 1, 0.25, 6.0, capi.farr(MEANS, 3, C.c_double),
                                 capi.PREC_FP16, None, C.c_void_p(poses.data_ptr()), None, None, None, None, None, None)
        assert rc != 0 and b"NULL" in capi.lib.dim_last_error()
        # the switch is refused once weights are loaded, and a weight of the other network is refused
        with pytest.raises(capi.DeepIMError, match="before dim_net_load"):
            capi.check(capi.lib.dim_ctx_set_input_depth(rgb._h, 1))
        with pytest.raises(ValueError, match="input_depth"):
            rgb.load_weights(weights)
        with pytest.raises(ValueError, match="input_depth"):
            rgbd.load_weights(w8)
        # the RGB-D training step refuses an RGB context (the other direction: test_gpu_rgbd_train.py)
        zb = torch.zeros((2, 3, H, W), device=DEV)
        z1 = torch.zeros((2, 1, H, W), device=DEV)
        zf = torch.tensor([[1.0, 1.0, 0.0, 0.0]] * 2, device=DEV)
        p = lambda t: C.c_void_p(t.data_ptr())
        rc = capi.lib.dim_train_forward_backward(rgb._h, p(zb), p(zb), p(z1), p(z1), p(zf), *([None] * 7), 2, 0,
                                                 *([None] * 7), None, None, 0, p(z1), p(z1), None)
        assert rc != 0 and b"takes no depth input" in capi.lib.dim_last_error()
        # and the switch is refused once the context trains
        t = Context(0, max_batch=2, max_classes=1, max_verts=6000, max_faces=11000)
        try:
            capi.check(capi.lib.dim_train_create(t._h, 100))
            with pytest.raises(capi.DeepIMError, match="dim_train_create"):
                capi.check(capi.lib.dim_ctx_set_input_depth(t._h, 1))
        finally:
            t.close()
        # the RGB context still refines after all that
        rgb.refine(*args, pixel_means_rgb=MEANS)
        torch.cuda.synchronize()
    finally:
        rgb.close()
        rgbd.close()


def test_pose_refiner_rgbd_matches_context_refine(meshes, weights, case):
    """PoseRefiner(input_depth=True) with the observed uint16 depth gives Context.refine_host's poses."""
    from deepim_b200.refiner import PoseRefiner
    c = case
    ref = PoseRefiner(meshes, weights, K, device=0, max_batch=B, n_iter=N_ITER, n_slots=1, input_depth=True)
    try:
        got = ref.refine(c["u8"], c["cls"], c["ini"], depths_u16=c["u16"])
        want, _ = ref.ctx.refine_host(c["u8"], c["cls"], c["ini"], K, N_ITER, pixel_means_rgb=MEANS,
                                      depth_observed_u16=c["u16"], depth_factor=1000.0)
        assert np.array_equal(got, want)
        with pytest.raises(ValueError, match="depths_u16"):
            ref.submit(c["u8"], c["cls"], c["ini"])
    finally:
        ref.close()
