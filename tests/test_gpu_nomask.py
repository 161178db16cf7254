"""GPU: the image-only network (config.network.INPUT_MASK: False) in the fused refinement loop and on the op surface --
dim_refine(_lit), dim_refine_host_async and dim_net_fwd of a dim_ctx_set_input_mask(ctx, 0) context against the oracle's
image-only loop (oracle.refine with input_mask=False), against the 8-channel context with zero mask columns, and the error
paths of the switch.

B = 16 observed frames: eight renders on a black background (the observed box is the object's) and eight composited over
noise (the observed box is the full frame).  Instance 5 refines a black-textured cube: its render has no colour-valid pixel,
so ZoomImage centres the zoom on the observed box and the loop flags it with status bit 2."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from kernel_ref import s2d_decode  # noqa: E402
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
BLACK = 5  # instance refined with the black cube (class 2)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.fixture(scope="module")
def meshes():
    black = synth.make_cube()
    black.tex = np.zeros_like(black.tex)
    ms = [synth.make_cube(), synth.make_blob(), black]
    for m in ms:
        m.normals = synth.vertex_normals(m)
    return ms


@pytest.fixture(scope="module")
def weights():
    return synth.make_train_weights(0, input_mask=False)


def make_ctx(meshes, weights, input_mask=False):
    c = Context(0, max_batch=B, max_classes=4, max_verts=6000, max_faces=11000, input_mask=input_mask)
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
    obs, ini = synth.sample_pose_pairs(B, 29)
    obs_cls = np.array([b % 2 for b in range(B)], np.int32)
    cls = obs_cls.copy()
    cls[BLACK] = 2
    u8 = []
    for b in range(B):
        r = O.render(meshes[obs_cls[b]], obs[b], K, means_rgb=MEANS)
        if b < B // 2:
            u8.append(np.where(r["mask"][..., None] > 0, r["bgr"].astype(np.uint8), 0).astype(np.uint8))
        else:
            u8.append(synth.composite_observed(r["bgr"], r["mask"], b))
    u8 = np.stack(u8)
    img = np.stack([synth.transform_image(u8[b]) for b in range(B)])
    ref = O.refine(weights, meshes, cls, img, ini, K, N_ITER, MEANS, input_mask=False, return_inputs=True)
    return dict(obs=obs, ini=ini, cls=cls, u8=u8, img=img, ref=ref)


def teacher(case, ref=None):
    ref = case["ref"] if ref is None else ref
    return dev(np.concatenate([case["ini"][None], ref["poses"][:N_ITER - 1]], 0))


def test_case_covers_both_observed_boxes_and_the_fallback(case):
    bb = case["ref"]["bbox"]
    full = np.array([0, W - 1, 0, H - 1])
    assert (bb[:, B // 2:, :4] == full).all()
    assert ((bb[:, :B // 2, 1] - bb[:, :B // 2, 0]) < W // 2).all()
    assert (bb[:, BLACK, 4:] == -1).all() and (np.delete(bb[:, :, 5], BLACK, axis=1) >= 0).all()


@pytest.mark.parametrize("prec", [capi.PREC_FP16, capi.PREC_BF16X3], ids=["fp16", "bf16x3"])
def test_conv1_input_is_the_zoomed_images(ctx, case, prec):
    """The conv1 input of iteration 0, read back from the space-to-depth buffer: lanes 0-5 equal zoom_image / 255 after
    16-bit rounding, bit for bit (bf16x3: both halves); lanes 6-7 are exact zeros everywhere."""
    c = case
    ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, 1, pixel_means_rgb=MEANS, precision=prec)
    torch.cuda.synchronize()
    z = c["ref"]["inputs"][0]
    x = O.conv1_input(z["zio"], z["zir"])  # [B,6,H,W]
    f16 = prec == capi.PREC_FP16
    hi, g = ctx.debug_activation(0, B, fp16=f16)
    rows, cols, ch, pad = g[0], g[1], g[2], g[3]
    assert ch == 32
    exp = np.zeros((B, 8, 2 * rows, 2 * cols), np.float32)
    exp[:, :6, pad:pad + H, pad:pad + W] = x
    rnd = (lambda a: a.astype(np.float16).astype(np.float32)) if f16 else \
        (lambda a: torch.from_numpy(a).bfloat16().float().numpy())
    got = s2d_decode(hi)
    assert np.array_equal(got, rnd(exp)), np.argwhere(got != rnd(exp))[:5]
    assert not got[:, 6:].any()
    if prec == capi.PREC_BF16X3:
        lo = s2d_decode(ctx.debug_activation(0, B, lo=True)[0])
        assert np.array_equal(lo, rnd(exp - rnd(exp))) and not lo[:, 6:].any()


def test_nomask_refine_teacher_forced_per_iteration(ctx, case):
    c, ref = case, case["ref"]
    res = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS, precision=capi.PREC_FP16,
                     pose_override=teacher(c))
    assert np.array_equal(res["bbox"].cpu().numpy(), ref["bbox"])
    assert np.array_equal(res["zoom_factor"].cpu().numpy(), ref["zoom_factor"])
    se3 = res["se3"].cpu().numpy()
    assert np.abs(se3[..., :4] - ref["se3"][..., :4]).max() < 1e-4
    assert np.abs(se3[..., 4:] - ref["se3"][..., 4:]).max() < 1e-3
    assert np.abs(res["poses"].cpu().numpy() - ref["poses"]).max() < 1e-4
    st = ctx.refine_status(B, N_ITER).numpy()
    assert (st[:, BLACK] == 4).all() and not np.delete(st, BLACK, axis=1).any(), st


def test_nomask_refine_lit_teacher_forced(ctx, meshes, weights, case):
    c = case
    inten = lighting.sample_intensity(np.random.default_rng(3), (N_ITER, B))
    lit = {"intensity": inten, "offset": lighting.OFFSET, "brightness_ratio": 0.7}
    po = [c["ini"]] + [c["ref"]["poses"][i] for i in range(N_ITER - 1)]
    ref = O.refine(weights, meshes, c["cls"], c["img"], c["ini"], K, N_ITER, MEANS, poses_override=po, lighting=lit,
                   input_mask=False)
    res = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS, precision=capi.PREC_FP16,
                     pose_override=teacher(c), lighting=dict(lit, intensity=dev(inten)))
    assert np.array_equal(res["bbox"].cpu().numpy(), ref["bbox"])
    assert np.array_equal(res["zoom_factor"].cpu().numpy(), ref["zoom_factor"])
    se3 = res["se3"].cpu().numpy()
    assert np.abs(se3[..., :4] - ref["se3"][..., :4]).max() < 1e-4
    assert np.abs(se3[..., 4:] - ref["se3"][..., 4:]).max() < 1e-3
    assert np.abs(res["poses"].cpu().numpy() - ref["poses"]).max() < 1e-4
    assert (ctx.refine_status(B, N_ITER).numpy()[:, BLACK] == 4).all()


@pytest.mark.parametrize("prec", [capi.PREC_FP16, capi.PREC_BF16, capi.PREC_BF16X3], ids=["fp16", "bf16", "bf16x3"])
def test_net_fwd_equals_the_eight_channel_network_with_zero_mask_columns(meshes, weights, case, prec):
    """dim_net_fwd of the mask-free context with W6 and of the 8-channel context with W6 plus zero mask columns, on the same
    zoomed images: bit-identical outputs (the zero columns add exact zeros to the fp32 accumulators)."""
    w8 = dict(weights, flow_conv1_weight=np.concatenate([weights["flow_conv1_weight"], np.zeros((64, 2, 7, 7), np.float32)], 1))
    z = case["ref"]["inputs"][0]
    m = (np.random.default_rng(2).uniform(size=(B, 1, H, W)) > 0.5).astype(np.float32)
    c6, c8 = make_ctx(meshes, weights), make_ctx(meshes, w8, True)
    try:
        r6, t6 = c6.net_forward(dev(z["zio"]), dev(z["zir"]), precision=prec)
        r8, t8 = c8.net_forward(dev(z["zio"]), dev(z["zir"]), dev(m), dev(1 - m), precision=prec)
        assert torch.equal(r6, r8) and torch.equal(t6, t8)
        if prec == capi.PREC_FP16:
            rr, tr = O.net_forward(weights, z["zio"], z["zir"])
            assert np.abs(r6.cpu().numpy() - rr).max() < 1e-4 and np.abs(t6.cpu().numpy() - tr).max() < 1e-3
    finally:
        c6.close()
        c8.close()


def test_nomask_graph_replay_equals_eager_and_host_equals_device(ctx, case):
    c = case
    img, cls, ini = dev(c["img"]), dev(c["cls"]), dev(c["ini"])
    capi.check(capi.lib.dim_debug_set_option(ctx._h, b"graph", 0))
    eager = {k: v.clone() for k, v in ctx.refine(img, cls, ini, K, N_ITER, pixel_means_rgb=MEANS).items()}
    capi.check(capi.lib.dim_debug_set_option(ctx._h, b"graph", 1))
    out = None
    for rep in range(3):
        out = ctx.refine(img, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, out=out)
        for k in ("poses", "se3", "zoom_factor", "bbox"):
            assert torch.equal(out[k], eager[k]), (rep, k)
    poses, se3 = ctx.refine_host(c["u8"], c["cls"], c["ini"], K, N_ITER, pixel_means_rgb=MEANS)
    assert np.array_equal(poses, eager["poses"].cpu().numpy())
    assert np.array_equal(se3, eager["se3"].cpu().numpy())


def test_pose_refiner_nomask(meshes, weights, case):
    """PoseRefiner(input_mask=False) gives Context.refine_host's poses; the black-render instance's bit 2 is reported in
    last_status without raising."""
    from deepim_b200.refiner import PoseRefiner
    c = case
    ref = PoseRefiner(meshes, weights, K, device=0, max_batch=B, n_iter=N_ITER, n_slots=1, input_mask=False)
    try:
        got = ref.refine(c["u8"], c["cls"], c["ini"])
        assert (ref.last_status[:, BLACK] == 4).all()
        want, _ = ref.ctx.refine_host(c["u8"], c["cls"], c["ini"], K, N_ITER, pixel_means_rgb=MEANS)
        assert np.array_equal(got, want)
    finally:
        ref.close()


def test_empty_observed_image_sets_status_bit_0(ctx, case):
    c = case
    img = c["img"][:2].copy()
    img[1] = -MEANS.astype(np.float32)[:, None, None]  # image + mean = 0 everywhere
    res = ctx.refine(dev(img), dev(c["cls"][:2]), dev(c["ini"][:2]), K, 1, pixel_means_rgb=MEANS)
    st = ctx.refine_status(2, 1).numpy()
    assert st[0, 0] == 0 and st[0, 1] & 1
    assert res["zoom_factor"][0, 1].cpu().numpy().tolist() == [1.0, 1.0, 0.0, 0.0]


def test_error_paths(meshes, weights, case):
    c = case
    w8 = synth.make_weights(0)
    rgb = make_ctx(meshes, w8, True)
    nm = make_ctx(meshes, weights)
    try:
        with pytest.raises(capi.DeepIMError, match="before dim_net_load"):
            capi.check(capi.lib.dim_ctx_set_input_mask(rgb._h, 0))
        with pytest.raises(capi.DeepIMError, match="before dim_net_load"):
            capi.check(capi.lib.dim_ctx_set_input_mask(nm._h, 1))
        with pytest.raises(capi.DeepIMError, match="INPUT_DEPTH without INPUT_MASK"):
            Context(0, max_batch=2, max_classes=1, max_verts=6000, max_faces=11000, input_depth=True, input_mask=False)
        d = Context(0, max_batch=2, max_classes=1, max_verts=6000, max_faces=11000, input_mask=False)
        try:
            with pytest.raises(capi.DeepIMError, match="INPUT_DEPTH without INPUT_MASK"):
                capi.check(capi.lib.dim_ctx_set_input_depth(d._h, 1))
        finally:
            d.close()
        with pytest.raises(ValueError, match=r"Context\(input_mask=False\)"):
            rgb.load_weights(weights)
        with pytest.raises(ValueError, match=r"\(64, 8, 7, 7\) belongs to Context\(\)"):
            nm.load_weights(w8)
        z = c["ref"]["inputs"][0]
        m = torch.zeros((2, 1, H, W), device=DEV)
        with pytest.raises(capi.DeepIMError, match="takes no mask input"):
            nm.net_forward(dev(z["zio"][:2]), dev(z["zir"][:2]), m, m)
        with pytest.raises(capi.DeepIMError, match="NULL argument"):
            rgb.net_forward(dev(z["zio"][:2]), dev(z["zir"][:2]))
        t = Context(0, max_batch=2, max_classes=1, max_verts=6000, max_faces=11000)
        try:
            capi.check(capi.lib.dim_train_create(t._h, 100))
            with pytest.raises(capi.DeepIMError, match="dim_train_create"):
                capi.check(capi.lib.dim_ctx_set_input_mask(t._h, 0))
        finally:
            t.close()
        nm.refine(dev(c["img"][:2]), dev(c["cls"][:2]), dev(c["ini"][:2]), K, 1, pixel_means_rgb=MEANS)
        torch.cuda.synchronize()
    finally:
        rgb.close()
        nm.close()
