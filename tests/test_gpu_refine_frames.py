"""GPU: the frame-indexed fused loop (dim_refine and dim_refine_host_async with a frame map, PoseRefiner.refine_frames).

Instance b of dim_refine(frames, idx) observes frames[idx[b]]; its results must equal dim_refine(frames[idx]) without a map,
bit for bit -- poses, se3, zoom factors, bboxes and status -- for every network and precision.  dim_refine's own parity with the
oracle is covered elsewhere, so the equality carries it over.

The case: F = 3 frames of the C2 mesh composited over noise, B = 16 instances observing them 10 / 5 / 1 (not contiguous; frame
2 has a single observer), every instance an initial hypothesis near its frame's object, spread over two classes."""
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
from deepim_b200.refiner import PoseRefiner  # noqa: E402

K = synth.K_LINEMOD
MEANS = synth.PIXEL_MEANS_RGB
DEV = torch.device("cuda", 0)
H, W = 480, 640
N_ITER = 4
B, F = 16, 3
IDX = np.array([0, 1, 0, 0, 1, 0, 2, 0, 1, 0, 0, 1, 0, 0, 1, 0], np.int32)  # 10 / 5 / 1 observers
KEYS = ("poses", "se3", "zoom_factor", "bbox")


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def make_frames(meshes, n_frames, n_inst, frame_of, seed, black=()):
    """n_frames observed frames (the blob at a sampled pose, over noise; frames in `black` over black) with u16 sensor-like
    depth, and per instance a class (alternating) and an initial pose: a perturbation of its frame's object pose."""
    fobs, _ = synth.sample_pose_pairs(n_frames, seed)
    pobs, pini = synth.sample_pose_pairs(n_inst, seed + 1)
    rng = np.random.default_rng(seed)
    u8, u16 = [], []
    for f in range(n_frames):
        r = O.render(meshes[0], fobs[f], K, means_rgb=MEANS)
        if f in black:
            u8.append(np.where(r["mask"][..., None] > 0, r["bgr"].astype(np.uint8), 0).astype(np.uint8))
        else:
            u8.append(synth.composite_observed(r["bgr"], r["mask"], seed + f))
        d = np.where(r["depth"] > 0, r["depth"] + rng.normal(0, 0.002, r["depth"].shape), rng.uniform(1.0, 2.0, r["depth"].shape))
        u16.append(np.clip(np.rint(d * 1000.0), 0, 65535).astype(np.uint16))
    u8, u16 = np.stack(u8), np.stack(u16)
    ini = pini.copy()
    ini[:, :, 3] = fobs[frame_of][:, :, 3] + (pini[:, :, 3] - pobs[:, :, 3])
    cls = (np.arange(n_inst) % 2).astype(np.int32)
    img = np.stack([synth.transform_image(u8[f]) for f in range(n_frames)])
    depth = O.depth_from_u16(u16, 1000.0)[:, None].astype(np.float32)
    return dict(u8=u8, u16=u16, img=img, depth=depth, cls=cls, ini=ini)


@pytest.fixture(scope="module")
def meshes():
    ms = [synth.make_blob(), synth.make_cube()]
    for m in ms:
        m.normals = synth.vertex_normals(m)
    return ms


@pytest.fixture(scope="module")
def case(meshes):
    return make_frames(meshes, F, B, IDX, 41, black=(2,))


def make_ctx(meshes, weights, **kw):
    c = Context(0, max_batch=B, max_classes=2, max_verts=6000, max_faces=11000, **kw)
    for i, m in enumerate(meshes):
        c.upload_mesh(i, m)
    c.load_weights(weights)
    return c


@pytest.fixture(scope="module")
def ctx(meshes):
    c = make_ctx(meshes, synth.make_weights(0))
    yield c
    c.close()


def status(ctx, n=B):
    return ctx.refine_status(n, N_ITER).numpy().copy()


def assert_same(a, b, sa=None, sb=None):
    for k in KEYS:
        assert np.array_equal(a[k].cpu().numpy(), b[k].cpu().numpy()), k
    if sa is not None:
        assert np.array_equal(sa, sb)


def frames_vs_gathered(ctx, c, idx, prec=capi.PREC_FP16, lit=None, depth=False):
    """(refine_frames result, status), (refine on the gathered frames result, status)"""
    frames, fidx = dev(c["img"]), dev(idx)
    df = dev(c["depth"]) if depth else None
    lf = None if lit is None else dict(lit, intensity=dev(lit["intensity"]))
    args = (dev(c["cls"][:len(idx)]), dev(c["ini"][:len(idx)]), K, N_ITER)
    a = {k: v.clone() for k, v in ctx.refine_frames(frames, fidx, *args, pixel_means_rgb=MEANS, precision=prec,
                                                    lighting=lf, depth_frames=df).items()}
    sa = status(ctx, len(idx))
    g = frames[fidx.long()].contiguous()
    b = ctx.refine(g, *args, pixel_means_rgb=MEANS, precision=prec, lighting=lf,
                   depth_observed=None if df is None else df[fidx.long()].contiguous())
    return (a, sa), (b, status(ctx, len(idx)))


# ------------------------------------------------------------------------------------ 1. bit-identity with dim_refine
@pytest.mark.parametrize("prec", [capi.PREC_FP16, capi.PREC_BF16, capi.PREC_BF16X3], ids=["fp16", "bf16", "bf16x3"])
def test_mask_network_equals_refine_on_gathered_frames(ctx, case, prec):
    (a, sa), (b, sb) = frames_vs_gathered(ctx, case, IDX, prec)
    assert_same(a, b, sa, sb)
    assert np.isfinite(a["poses"].cpu().numpy()).all()


def test_lit_loop_equals_refine_on_gathered_frames(ctx, case):
    inten = lighting.sample_intensity(np.random.default_rng(3), (N_ITER, B))
    lit = {"intensity": inten, "offset": lighting.OFFSET, "brightness_ratio": 0.7}
    (a, sa), (b, sb) = frames_vs_gathered(ctx, case, IDX, lit=lit)
    assert_same(a, b, sa, sb)


def test_image_only_network_equals_refine_on_gathered_frames(meshes, case):
    c = make_ctx(meshes, synth.make_train_weights(0, input_mask=False), input_mask=False)
    try:
        (a, sa), (b, sb) = frames_vs_gathered(c, case, IDX)
        assert_same(a, b, sa, sb)
        bb = a["bbox"].cpu().numpy()[0, :, :4]
        full = np.array([0, W - 1, 0, H - 1])
        assert (bb[IDX != 2] == full).all()            # frames over noise: the whole image is valid
        assert (bb[IDX == 2, 1] - bb[IDX == 2, 0] < W // 2).all()  # frame 2, over black: the object's box
    finally:
        c.close()


def test_rgbd_network_equals_refine_on_gathered_frames(meshes, case):
    c = make_ctx(meshes, synth.make_weights(0, input_depth=True), input_depth=True)
    try:
        (a, sa), (b, sb) = frames_vs_gathered(c, case, IDX, depth=True)
        assert_same(a, b, sa, sb)
        # host entry with the u16 depth frames = the device entry with their float conversion
        poses, se3 = c.refine_frames_host(case["u8"], IDX, case["cls"], case["ini"], K, N_ITER, pixel_means_rgb=MEANS,
                                          depth_frames_u16=case["u16"], depth_factor=1000.0)
        assert np.array_equal(poses, a["poses"].cpu().numpy()) and np.array_equal(se3, a["se3"].cpu().numpy())
    finally:
        c.close()


# ------------------------------------------------------------------------------------------------- 2. identity map
def test_identity_map_equals_refine(ctx, meshes):
    c = make_frames(meshes, B, B, np.arange(B), 53)
    img, cls, ini = dev(c["img"]), dev(c["cls"]), dev(c["ini"])
    a = {k: v.clone() for k, v in ctx.refine_frames(img, dev(np.arange(B, dtype=np.int32)), cls, ini, K, N_ITER,
                                                    pixel_means_rgb=MEANS).items()}
    sa = status(ctx)
    b = ctx.refine(img, cls, ini, K, N_ITER, pixel_means_rgb=MEANS)
    assert_same(a, b, sa, status(ctx))


def test_one_frame_for_every_instance(ctx, meshes):
    c = make_frames(meshes, 1, B, np.zeros(B, np.int32), 61)
    assert set(c["cls"].tolist()) == {0, 1}
    (a, sa), (b, sb) = frames_vs_gathered(ctx, c, np.zeros(B, np.int32))
    assert_same(a, b, sa, sb)


# -------------------------------------------------------------------------------------------------- 3. graph replay
def test_graph_replay_index_rewrite_and_interleaving(ctx, case):
    """On a side stream (the legacy default stream cannot be captured): eager run, capture and replay of dim_refine with a
    frame map equal the launch-by-launch run, with two index buffers and dim_refine without a map interleaved on one context; new indices written
    into a captured index buffer take effect at the next replay."""
    s = torch.cuda.Stream(device=DEV)
    s.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(s):
        graph_replay_body(ctx, case)
    torch.cuda.synchronize()


def graph_replay_body(ctx, case):
    c = case
    frames, cls, ini = dev(c["img"]), dev(c["cls"]), dev(c["ini"])
    idx2 = np.roll(IDX, 5)
    capi.check(capi.lib.dim_debug_set_option(ctx._h, b"graph", 0))   # eager references, launch by launch
    want = {}
    for name, idx in (("a", IDX), ("b", idx2)):
        want[name] = {k: v.clone() for k, v in ctx.refine_frames(frames, dev(idx), cls, ini, K, N_ITER,
                                                                 pixel_means_rgb=MEANS).items()}
    want_refine = {k: v.clone() for k, v in ctx.refine(frames[dev(IDX).long()].contiguous(), cls, ini, K, N_ITER,
                                                       pixel_means_rgb=MEANS).items()}
    assert not all(torch.equal(want["a"][k], want["b"][k]) for k in KEYS)
    capi.check(capi.lib.dim_debug_set_option(ctx._h, b"graph", 1))
    fidx, fidx2, gathered = dev(IDX), dev(IDX), frames[dev(IDX).long()].contiguous()
    out = out2 = outr = None
    for rep in range(3):  # eager, capture, replay -- interleaved with a second index buffer and with no frame map
        out = ctx.refine_frames(frames, fidx, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, out=out)
        assert_same(out, want["a"])
        out2 = ctx.refine_frames(frames, fidx2, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, out=out2)
        assert_same(out2, want["a"])
        outr = ctx.refine(gathered, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, out=outr)
        assert_same(outr, want_refine)
    # new contents in the same index buffer: the replayed graph reads them
    fidx.copy_(dev(idx2))
    out = ctx.refine_frames(frames, fidx, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, out=out)
    assert_same(out, want["b"])
    out2 = ctx.refine_frames(frames, fidx2, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, out=out2)
    assert_same(out2, want["a"])


# ---------------------------------------------------------------------------------------- 4. host entry = device entry
@pytest.mark.parametrize("sync", [True, False], ids=["sync", "async"])
def test_host_entry_equals_device_entry(ctx, case, sync):
    c = case
    a = ctx.refine_frames(dev(c["img"]), dev(IDX), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS)
    sa = status(ctx)
    poses = torch.empty((N_ITER, B, 3, 4), dtype=torch.float64).pin_memory()
    se3 = torch.empty((N_ITER, B, 7), dtype=torch.float32).pin_memory()
    ctx.refine_frames_host(torch.from_numpy(c["u8"]).pin_memory(), torch.from_numpy(IDX).pin_memory(), c["cls"], c["ini"], K,
                           N_ITER, pixel_means_rgb=MEANS, poses_out=poses, se3_out=se3, sync=sync)
    torch.cuda.synchronize()
    assert np.array_equal(poses.numpy(), a["poses"].cpu().numpy())
    assert np.array_equal(se3.numpy(), a["se3"].cpu().numpy())
    assert np.array_equal(status(ctx), sa)


# ------------------------------------------------------------------------------------ 5. PoseRefiner.refine_frames
def test_pose_refiner_refine_frames_equals_refine_on_gathered_frames(meshes):
    n, nf = 37, 11
    frame_of = np.random.default_rng(7).integers(0, nf, size=n).astype(np.int32)
    frame_of[:8] = 3                                      # the first device batch: one frame for eight instances
    c = make_frames(meshes, nf, n, frame_of, 71)
    r = PoseRefiner(meshes, synth.make_weights(0), K, device=0, max_batch=B, n_iter=N_ITER, n_slots=2)
    try:
        got = r.refine_frames(c["u8"], frame_of, c["cls"], c["ini"])
        want = r.refine(c["u8"][frame_of], c["cls"], c["ini"])
        assert got.shape == (N_ITER, n, 3, 4) and np.isfinite(got).all()
        assert np.array_equal(got, want)
        with pytest.raises(ValueError, match="instance 4 has frame index 11"):
            r.refine_frames(c["u8"], np.array([0, 1, 2, 0, 11]), c["cls"][:5], c["ini"][:5])
    finally:
        r.close()


# ------------------------------------------------------------------------------------------------------ 6. errors
def test_error_paths(ctx, meshes, case):
    c = case
    frames, fidx, cls, ini = dev(c["img"]), dev(IDX), dev(c["cls"]), dev(c["ini"])
    h = ctx._h
    K9 = capi.farr(np.asarray(K, np.float32).reshape(9), 9)
    means = capi.farr(MEANS, 3, capi.C.c_double)
    poses = torch.empty((N_ITER, B, 3, 4), dtype=torch.float64, device=DEV)
    st = ctx._stream()
    p = capi.C.c_void_p

    kf = dev(np.stack([np.asarray(K, np.float32)] * F))
    hu8, hidx, hcls, hini = (np.ascontiguousarray(a) for a in (c["u8"], IDX, c["cls"], c["ini"]))
    hposes = np.full((N_ITER, B, 3, 4), 7.0)

    def dev_call(F_, fptr=p(frames.data_ptr()), iptr=p(fidx.data_ptr()), depth=None, k9=K9, kptr=None):
        return capi.lib.dim_refine(h, fptr, F_, iptr, k9, kptr, p(cls.data_ptr()), p(ini.data_ptr()), B, N_ITER, 0.25, 6.0,
                                   means, capi.PREC_FP16, None, p(poses.data_ptr()), None, None, None, depth, None, st)

    def host_call(F_, iptr=p(hidx.ctypes.data), k9=K9, kptr=None):
        return capi.lib.dim_refine_host_async(h, p(hu8.ctypes.data), F_, iptr, k9, kptr, p(hcls.ctypes.data),
                                              p(hini.ctypes.data), B, N_ITER, 0.25, 6.0, means, capi.PREC_FP16,
                                              p(hposes.ctypes.data), None, None, 1000.0, None, st)
    for call, entry in ((dev_call, b"dim_refine: "), (host_call, b"dim_refine_host_async: ")):
        for F_ in (0, B + 1):
            assert call(F_) == 2 and entry + b"frame count F" in capi.lib.dim_last_error()
        # no frame map: instance b observes frame b, so F must equal B
        assert call(F, iptr=None) == 2 and entry + b"frame_idx is NULL" in capi.lib.dim_last_error()
        assert b"F must equal B" in capi.lib.dim_last_error()
        # exactly one of K9 and K_frames
        for k9, kptr in ((K9, p(kf.data_ptr())), (None, None)):
            assert call(F, k9=k9, kptr=kptr) == 2 and entry + b"exactly one of K9_host and K_frames" in capi.lib.dim_last_error()
    assert dev_call(F, fptr=None) == 2 and b"NULL argument" in capi.lib.dim_last_error()
    assert dev_call(F, depth=p(frames.data_ptr())) == 2 and b"takes no depth input" in capi.lib.dim_last_error()
    torch.cuda.synchronize()
    assert (hposes == 7.0).all()

    host = dict(pixel_means_rgb=MEANS)
    bad = IDX.copy()
    bad[9] = F
    with pytest.raises(capi.DeepIMError, match="instance 9 has frame index 3: out of range"):
        ctx.refine_frames_host(c["u8"], bad, c["cls"], c["ini"], K, N_ITER, **host)
    bad[9] = -1
    with pytest.raises(capi.DeepIMError, match="instance 9 has frame index -1"):
        ctx.refine_frames_host(c["u8"], bad, c["cls"], c["ini"], K, N_ITER, **host)
    with pytest.raises(capi.DeepIMError, match="depth_frames_u16_host"):
        ctx.refine_frames_host(c["u8"], IDX, c["cls"], c["ini"], K, N_ITER, depth_frames_u16=c["u16"], **host)
    u8_17 = np.zeros((B + 1, H, W, 3), np.uint8)
    with pytest.raises(capi.DeepIMError, match="frame count F"):
        ctx.refine_frames_host(u8_17, IDX, c["cls"], c["ini"], K, N_ITER, **host)
    r = make_ctx(meshes, synth.make_weights(0, input_depth=True), input_depth=True)
    try:
        with pytest.raises(capi.DeepIMError, match="depth_frames"):
            r.refine_frames(frames, fidx, cls, ini, K, N_ITER, pixel_means_rgb=MEANS)
        with pytest.raises(capi.DeepIMError, match="depth_frames_u16_host"):
            r.refine_frames_host(c["u8"], IDX, c["cls"], c["ini"], K, N_ITER, **host)
    finally:
        r.close()


def test_device_index_out_of_range_is_clamped_and_flagged(ctx, case):
    """The defined path for a bad device index: instance 4 (index 7 with F = 3) and instance 6 (index -2) observe frame 0
    and carry status bit 3 in every iteration; the others are untouched."""
    c = case
    bad = IDX.copy()
    bad[4], bad[6] = 7, -2
    clamp = bad.copy()
    clamp[4] = clamp[6] = 0
    frames = dev(c["img"])
    args = (dev(c["cls"]), dev(c["ini"]), K, N_ITER)
    a = {k: v.clone() for k, v in ctx.refine_frames(frames, dev(bad), *args, pixel_means_rgb=MEANS).items()}
    sa = status(ctx)
    b = ctx.refine_frames(frames, dev(clamp), *args, pixel_means_rgb=MEANS)
    sb = status(ctx)
    assert_same(a, b)
    assert ((sa[:, [4, 6]] & 8) == 8).all()
    assert np.array_equal(sa & ~8, sb) and not (np.delete(sa, [4, 6], axis=1) & 8).any()
