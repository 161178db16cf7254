"""GPU: the ModelNet (unseen-object) branch of the test and train loops -- the fused refinement loop and the train-time
batch update with the Lambert-lit renderer (dim_refine, dim_refine_host_async, dim_train_update with a dim_lighting) against the
oracle's lit loops (oracle.refine / oracle.train_update with lighting), against the unlit calls where the light is neutral,
and through the Python layers (PoseRefiner, trainer)."""
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
MEANS32 = MEANS.astype(np.float32)
DEV = torch.device("cuda", 0)
H, W = 480, 640
N_ITER = 4


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def lit(intensity, ratio=0.7):
    return {"intensity": intensity, "offset": lighting.OFFSET, "brightness_ratio": ratio}


@pytest.fixture(scope="module")
def meshes():
    ms = [synth.make_cube(), synth.make_blob()]
    for m in ms:
        m.normals = synth.vertex_normals(m)
    return ms


@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(0)


@pytest.fixture(scope="module")
def ctx(meshes, weights):
    c = Context(0, max_batch=4, max_classes=4, max_verts=6000, max_faces=11000)
    for i, m in enumerate(meshes):
        c.upload_mesh(i, m)  # uploads m.normals as well
    c.load_weights(weights)
    yield c
    c.close()


@pytest.fixture(scope="module")
def case(meshes, weights):
    B = 4
    obs, ini = synth.sample_pose_pairs(B, 51)
    cls = np.array([0, 1, 1, 0], np.int32)
    u8 = []
    for b in range(B):
        r = O.render_lit(meshes[cls[b]], meshes[cls[b]].normals, obs[b], K, O.light_position(obs[b]),
                         np.array([1.02, 0.97, 1.0], np.float32), 0.7)
        u8.append(synth.composite_observed(r["bgr"], r["mask"], b))
    u8 = np.stack(u8)
    img = np.stack([synth.transform_image(u8[b]) for b in range(B)])
    inten = lighting.sample_intensity(np.random.default_rng(11), (N_ITER, B))
    ref = O.refine(weights, meshes, cls, img, ini, K, N_ITER, MEANS32, lighting=lit(inten))
    return dict(B=B, obs=obs, ini=ini, cls=cls, u8=u8, img=img, inten=inten, ref=ref)


@pytest.mark.parametrize("prec", [capi.PREC_FP16, capi.PREC_BF16X3], ids=["fp16", "bf16x3"])
def test_lit_refine_teacher_forced_per_iteration(ctx, case, prec):
    """Each iteration started from the lit CPU checker's pose: bbox and zoom factor bit-exact (the lit render has the unlit
    geometry), se3 within 1e-4 rot / 1e-3 trans, composed pose within 1e-4."""
    c, ref = case, case["ref"]
    override = np.concatenate([c["ini"][None], ref["poses"][:3]], 0)
    res = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS, precision=prec,
                     pose_override=dev(override), lighting=lit(dev(c["inten"])))
    assert np.array_equal(res["bbox"].cpu().numpy(), ref["bbox"])
    assert np.array_equal(res["zoom_factor"].cpu().numpy(), ref["zoom_factor"])
    se3 = res["se3"].cpu().numpy()
    assert np.abs(se3[..., :4] - ref["se3"][..., :4]).max() < 1e-4
    assert np.abs(se3[..., 4:] - ref["se3"][..., 4:]).max() < 1e-3
    assert np.abs(res["poses"].cpu().numpy() - ref["poses"]).max() < 1e-4
    assert not ctx.refine_status(c["B"], N_ITER).numpy().any()


def test_lit_refine_free_running_fp16(ctx, case):
    c = case
    res = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS, precision=capi.PREC_FP16,
                     lighting=lit(dev(c["inten"])))
    poses = res["poses"].cpu().numpy()
    assert np.isfinite(poses).all()
    assert np.abs(poses - c["ref"]["poses"]).max() < 1e-3


def test_neutral_light_gives_the_unlit_loop_bit_for_bit(ctx, case):
    """brightness_ratio 0 and unit intensity: round(texel) = the uint8-truncated unlit colour, so the lit dim_refine computes what
    the unlit one computes, bit for bit."""
    c = case
    args = (dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER)
    unlit = ctx.refine(*args, pixel_means_rgb=MEANS)
    flat = ctx.refine(*args, pixel_means_rgb=MEANS, lighting=lit(torch.ones(N_ITER, c["B"], 3, device=DEV), 0.0))
    for k in ("poses", "se3", "zoom_factor", "bbox"):
        assert torch.equal(flat[k], unlit[k]), k
    # with the real light the colours, hence the poses, differ
    lit_res = ctx.refine(*args, pixel_means_rgb=MEANS, lighting=lit(dev(c["inten"])))
    assert not torch.equal(lit_res["se3"], unlit["se3"])


def test_each_iteration_uses_its_own_intensity(ctx, case):
    """Iteration `it` renders with intensity[it]: changing only iteration 2's draw leaves iterations 0-1 bit-identical and
    changes iteration 2 onwards."""
    c = case
    args = (dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER)
    a = ctx.refine(*args, pixel_means_rgb=MEANS, lighting=lit(dev(c["inten"])))
    inten2 = c["inten"].copy()
    inten2[2] = np.where(inten2[2] > 1.0, 0.9, 1.1).astype(np.float32)
    b = ctx.refine(*args, pixel_means_rgb=MEANS, lighting=lit(dev(inten2)))
    for k in ("poses", "se3", "zoom_factor", "bbox"):
        assert torch.equal(a[k][:2], b[k][:2]), k
    assert not torch.equal(a["se3"][2], b["se3"][2])
    assert not torch.equal(a["poses"][2], b["poses"][2]) and not torch.equal(a["poses"][3], b["poses"][3])


def test_lit_graph_replay_equals_eager_and_never_mixes_with_unlit(ctx, case):
    """The lit chain is captured and replayed as a CUDA graph like the unlit one.  Lit and unlit calls alternating on one
    context with the SAME output buffers stay bit-identical to their eager runs (the graph key separates them), and new
    intensities written into the same buffer are honoured by the replay."""
    from deepim_b200._capi import check, lib
    c = case
    img, cls, ini = dev(c["img"]), dev(c["cls"]), dev(c["ini"])
    inten = dev(c["inten"])
    inten_b = dev(lighting.sample_intensity(np.random.default_rng(12), (N_ITER, c["B"])))
    check(lib.dim_debug_set_option(ctx._h, b"graph", 0))
    eager_lit = ctx.refine(img, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, lighting=lit(inten))
    eager_lit_b = ctx.refine(img, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, lighting=lit(inten_b))
    eager_unlit = ctx.refine(img, cls, ini, K, N_ITER, pixel_means_rgb=MEANS)
    eager_ratio = ctx.refine(img, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, lighting=lit(inten, 0.5))
    torch.cuda.synchronize()
    check(lib.dim_debug_set_option(ctx._h, b"graph", 1))
    side = torch.cuda.Stream(device=DEV)
    out = None
    keys = ("poses", "se3", "zoom_factor", "bbox")
    for it in range(4):  # eager warm-up, capture + launch, replay, replay -- for each of the three chains
        for want, kw in ((eager_lit, {"lighting": lit(inten)}), (eager_unlit, {}), (eager_ratio, {"lighting": lit(inten, 0.5)})):
            with torch.cuda.stream(side):
                out = ctx.refine(img, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, out=out, **kw)
            side.synchronize()
            for k in keys:
                assert torch.equal(out[k], want[k]), (it, k, kw.get("lighting", {}).get("brightness_ratio"))
    with torch.cuda.stream(side):  # same intensity buffer, new contents
        inten.copy_(inten_b)
        out = ctx.refine(img, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, out=out, lighting=lit(inten))
    side.synchronize()
    for k in keys:
        assert torch.equal(out[k], eager_lit_b[k]), k
    torch.cuda.synchronize()


def test_lit_host_entry_equals_device_entry(ctx, case):
    c = case
    poses, se3 = ctx.refine_host(c["u8"], c["cls"], c["ini"], K, N_ITER, pixel_means_rgb=MEANS, precision=capi.PREC_FP16,
                                 lighting=lit(c["inten"]))
    d = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS, precision=capi.PREC_FP16,
                   lighting=lit(dev(c["inten"])))
    assert np.array_equal(poses, d["poses"].cpu().numpy())
    assert np.array_equal(se3, d["se3"].cpu().numpy())
    assert not ctx.refine_status(c["B"], N_ITER).numpy().any()


def test_lit_train_update_matches_oracle(ctx, meshes):
    """batchUpdaterPyMulti.forward of the ModelNet branch: the re-render is lit with the light of the float64 refined pose,
    image = float32 quantised colours - float32 means.  Every other output is the unlit update's, bit for bit; the lit image,
    depth and mask are bit-exact against the oracle wherever the refined pose rounds to the same float32."""
    B = 3
    obs, ini = synth.sample_pose_pairs(B, 81)
    cls = np.array([1, 0, 1], np.int32)
    rng = np.random.default_rng(7)
    rot_est = (np.array([1.0, 0, 0, 0]) + rng.normal(size=(B, 4)) * 0.03).astype(np.float32)
    trans_est = (rng.normal(size=(B, 3)) * 0.01).astype(np.float32)
    src32, tgt32 = ini.astype(np.float32), obs.astype(np.float32)
    depth_gt = np.stack([O.render(meshes[cls[b]], obs[b], K)["depth"] for b in range(B)])[:, None]
    inten = lighting.sample_intensity(rng, B)
    args = (dev(cls), dev(src32), dev(rot_est), dev(trans_est), dev(tgt32), dev(depth_gt), K)
    out = ctx.train_update(*args, pixel_means_rgb=MEANS, lighting=lit(dev(inten)))
    unlit = ctx.train_update(*args, pixel_means_rgb=MEANS)
    for k in ("depth_rendered", "mask_rendered", "src_pose", "rot", "trans", "flow", "flow_weights"):
        assert torch.equal(out[k], unlit[k]), k
    assert not torch.equal(out["image_rendered"], unlit["image_rendered"])
    ref = O.train_update(meshes, cls, src32, rot_est, trans_est, tgt32, depth_gt, K, MEANS, lighting=lit(inten))
    sp = out["src_pose"].cpu().numpy()
    assert np.abs(sp - ref["src_pose"]).max() < 1e-6
    assert np.abs(out["rot"].cpu().numpy() - ref["rot"]).max() < 1e-6     # Jacobi vs LAPACK eigh, float32 store
    assert np.abs(out["trans"].cpu().numpy() - ref["trans"]).max() < 1e-6
    same = [b for b in range(B) if np.array_equal(sp[b], ref["src_pose"][b])]
    assert same, "no instance's refined pose rounds to the oracle's float32 pose"
    for b in same:
        for k in ("image_rendered", "depth_rendered", "mask_rendered"):
            assert np.array_equal(out[k][b].cpu().numpy(), ref[k][b]), (b, k)
    fw, ofw = out["flow_weights"].cpu().numpy(), ref["flow_weights"]
    assert np.array_equal(fw[:, 0], fw[:, 1]) and ofw.sum() > 1000
    assert (fw != ofw).mean() < 2e-4       # KT differs at float32 rounding level -> a few threshold pixels (as unlit)
    both = (fw[:, :1] == 1) & (ofw[:, :1] == 1)
    assert np.abs(out["flow"].cpu().numpy() - ref["flow"])[np.repeat(both, 2, 1)].max() < 2e-3


def test_lighting_refuses_missing_normals_and_null_intensity(ctx, case):
    import ctypes as C
    from deepim_b200._capi import lib
    c = case
    bare = Context(0, max_batch=2, max_classes=1, max_verts=6000, max_faces=11000)
    try:
        bare.upload_mesh(0, synth.make_cube())  # no normals
        L = lit(torch.ones(N_ITER, 2, 3, device=DEV))
        with pytest.raises(capi.DeepIMError, match="normals"):
            bare.refine(dev(c["img"][:2]), dev(c["cls"][:2] * 0), dev(c["ini"][:2]), K, N_ITER, lighting=L)
        with pytest.raises(capi.DeepIMError, match="normals"):
            bare.refine_host(c["u8"][:2], c["cls"][:2] * 0, c["ini"][:2], K, N_ITER, lighting=lit(np.ones((N_ITER, 2, 3), np.float32)))
        with pytest.raises(capi.DeepIMError, match="normals"):
            bare.train_update(dev(c["cls"][:2] * 0), dev(c["ini"][:2].astype(np.float32)), torch.zeros(2, 4, device=DEV),
                              torch.zeros(2, 3, device=DEV), dev(c["obs"][:2].astype(np.float32)), None, K, want_flow=False,
                              lighting=lit(torch.ones(2, 3, device=DEV)))
    finally:
        bare.close()
    # NULL intensity through the C ABI (NULL lighting is the unlit loop)
    B = c["B"]
    img, cls, ini = dev(c["img"]), dev(c["cls"]), dev(c["ini"])
    poses = torch.empty(N_ITER, B, 3, 4, dtype=torch.float64, device=DEV)
    K9 = capi.farr(K.reshape(9), 9)
    means = capi.farr(MEANS, 3, C.c_double)
    null_int = capi.Lighting(None, (C.c_double * 3)(0.0, 0.5, 0.5), 0.7)
    rc = lib.dim_refine(ctx._h, C.c_void_p(img.data_ptr()), B, None, K9, None, C.c_void_p(cls.data_ptr()),
                        C.c_void_p(ini.data_ptr()), B, N_ITER, 0.25, 6.0, means, capi.PREC_FP16, None, C.c_void_p(poses.data_ptr()),
                        None, None, None, None, C.byref(null_int), None)
    assert rc != 0 and b"NULL" in lib.dim_last_error()
    with pytest.raises(capi.DeepIMError):
        capi.check(rc)
    with pytest.raises(ValueError):
        ctx.refine(img, cls, ini, K, N_ITER, lighting={"offset": (0, 0.5, 0.5)})  # no intensity


def test_fit_batch_lit_four_inner_iterations(meshes):
    from deepim_b200.trainer import Trainer, fit_batch, make_device_batch
    B = 2
    tctx = Context(0, max_batch=B, max_classes=2, max_verts=6000, max_faces=11000)
    try:
        for i, m in enumerate(meshes):
            tctx.upload_mesh(i, m)
        src = lighting.LightSource(seed=3)
        batch, cls, tgt, depth_gt = make_device_batch(tctx, meshes, B, 11, K, MEANS, lighting=src)
        plain, _, _, _ = make_device_batch(tctx, meshes, B, 11, K, MEANS)
        assert torch.equal(batch["mask_rendered"], plain["mask_rendered"]) and torch.equal(batch["flow"], plain["flow"])
        assert not torch.equal(batch["image_rendered"], plain["image_rendered"])
        assert not torch.equal(batch["image_observed"], plain["image_observed"])
        tr = Trainer(tctx, synth.make_train_weights(0))
        objs = fit_batch(tr, batch, cls, tgt, depth_gt, K, n_inner=4, lighting=src).cpu().numpy()
        assert objs.shape == (4,) and np.isfinite(objs).all()
        torch.cuda.synchronize()
    finally:
        tctx.close()


def test_pose_refiner_lit_matches_context_refine(ctx, meshes, weights, case):
    """PoseRefiner(lighting={"seed": s}) draws intensity[n_iter, n, 3] per submit from default_rng(s): the same draws given to
    Context.refine give the same poses."""
    from deepim_b200.refiner import PoseRefiner
    c = case
    ref = PoseRefiner(meshes, weights, K, device=0, max_batch=4, n_iter=N_ITER, n_slots=1, lighting={"seed": 23})
    try:
        poses = ref.refine(c["u8"], c["cls"], c["ini"])
    finally:
        ref.close()
    inten = lighting.sample_intensity(np.random.default_rng(23), (N_ITER, c["B"]))
    d = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS, precision=capi.PREC_FP16,
                   lighting=lit(dev(inten)))
    assert np.array_equal(poses, d["poses"].cpu().numpy())
    with pytest.raises(ValueError):
        PoseRefiner([synth.make_cube()], weights, K, device=0, max_batch=2, n_iter=2, n_slots=1, lighting={"seed": 1})
