"""GPU: one camera per frame in the frame-indexed fused loop (dim_refine / dim_refine_host_async with K_frames,
Context.refine_frames(K=[F,3,3]), PoseRefiner.refine_frames(K_frames=...) / refine(K=...), lm6d_io's per-pair `-K.txt`).

Instance b is rendered and zoomed with the camera of its frame, so its results must equal dim_refine's with
K9 = K_frames[frame_idx[b]], bit for bit -- poses, se3, zoom factors, bboxes and status -- for every network and precision.
dim_refine's own parity with the oracle is covered elsewhere; the teacher-forced oracle check below holds each camera
to the float restatement directly.

The case: F = 6 frames at 480x640 from three cameras (LINEMOD, YCB-Video camera 1, and an off-centre one; frames 0 / 3 the
first, 1 / 4 the second, 2 / 5 the third), each frame the C2 blob at a sampled pose rendered with its camera over noise.
B = 16 instances observe them 5 / 1 / 3 / 2 / 4 / 1 (not contiguous), each an initial hypothesis near its frame's object, over
two classes."""
import os
import shutil

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from oracle import oracle as O  # noqa: E402
from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import lighting, lm6d_io, synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.refiner import PoseRefiner  # noqa: E402


def pinhole(fx, fy, cx, cy):
    return np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], np.float32)


CAMS = np.stack([pinhole(572.41, 573.57, 325.26, 242.05),      # LINEMOD
                 pinhole(1066.778, 1067.487, 312.99, 241.31),  # YCB-Video camera 1
                 pinhole(800.0, 790.0, 410.5, 190.25)])        # off-centre
MEANS = synth.PIXEL_MEANS_RGB
DEV = torch.device("cuda", 0)
H, W = 480, 640
N_ITER = 4
B, F = 16, 6
CAM_OF_FRAME = np.array([0, 1, 2, 0, 1, 2])
KF = CAMS[CAM_OF_FRAME]                                          # [F,3,3]
IDX = np.random.default_rng(5).permutation(np.repeat(np.arange(F), [5, 1, 3, 2, 4, 1])).astype(np.int32)
KEYS = ("poses", "se3", "zoom_factor", "bbox")


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def make_frames(meshes, Kf, frame_of, seed):
    """len(Kf) observed frames, frame f the blob at a sampled pose rendered with camera Kf[f] over noise, with u16
    sensor-like depth; per instance a class (alternating) and an initial pose near its frame's object pose."""
    n_frames, n_inst = len(Kf), len(frame_of)
    fobs, _ = synth.sample_pose_pairs(n_frames, seed)
    pobs, pini = synth.sample_pose_pairs(n_inst, seed + 1)
    rng = np.random.default_rng(seed)
    u8, u16 = [], []
    for f in range(n_frames):
        r = O.render(meshes[0], fobs[f], Kf[f], means_rgb=MEANS)
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
    return make_frames(meshes, KF, IDX, 91)


def make_ctx(meshes, weights, max_batch=B, **kw):
    c = Context(0, max_batch=max_batch, max_classes=2, max_verts=6000, max_faces=11000, **kw)
    for i, m in enumerate(meshes):
        c.upload_mesh(i, m)
    c.load_weights(weights)
    return c


@pytest.fixture(scope="module")
def ctx(meshes):
    c = make_ctx(meshes, synth.make_weights(0))
    yield c
    c.close()


def status(ctx, n):
    return ctx.refine_status(n, N_ITER).numpy().copy()


def cpu(r):
    return {k: r[k].cpu().numpy() for k in KEYS}


def mixed_vs_per_camera(ctx, c, idx, prec=capi.PREC_FP16, lit=None, depth=False):
    """refine_frames with one camera per frame against refine_frames (one K9) on each camera's sub-batch: every output of
    every instance bit for bit, status included"""
    n = len(idx)
    frames = dev(c["img"])
    df = dev(c["depth"]) if depth else None
    lf = None if lit is None else dict(lit, intensity=dev(lit["intensity"][:, :n]))
    a = cpu(ctx.refine_frames(frames, dev(idx), dev(c["cls"][:n]), dev(c["ini"][:n]), dev(KF), N_ITER, pixel_means_rgb=MEANS,
                              precision=prec, lighting=lf, depth_frames=df))
    sa = status(ctx, n)
    cam = CAM_OF_FRAME[idx]
    assert len(set(cam.tolist())) == 3
    for k in range(3):
        s = np.nonzero(cam == k)[0]
        lk = None if lit is None else dict(lit, intensity=dev(lit["intensity"][:, s]))
        b = cpu(ctx.refine_frames(frames, dev(idx[s]), dev(c["cls"][s]), dev(c["ini"][s]), CAMS[k], N_ITER,
                                  pixel_means_rgb=MEANS, precision=prec, lighting=lk, depth_frames=df))
        for key in KEYS:
            assert np.array_equal(a[key][:, s], b[key]), (k, key)
        assert np.array_equal(sa[:, s], status(ctx, len(s))), k
    assert np.isfinite(a["poses"]).all()
    return a, sa


# ---------------------------------------------------------------------------- 1. mixed batch = per-camera K9 batches
@pytest.mark.parametrize("prec", [capi.PREC_FP16, capi.PREC_BF16, capi.PREC_BF16X3], ids=["fp16", "bf16", "bf16x3"])
def test_mask_network_mixed_batch_equals_per_camera_batches(ctx, case, prec):
    a, sa = mixed_vs_per_camera(ctx, case, IDX, prec)
    assert not sa.any(), sa
    # the cameras do differ: the same instance under another camera zooms elsewhere
    other = cpu(ctx.refine_frames(dev(case["img"]), dev(IDX), dev(case["cls"]), dev(case["ini"]), CAMS[0], N_ITER,
                                  pixel_means_rgb=MEANS, precision=prec))
    moved = CAM_OF_FRAME[IDX] != 0
    assert (a["zoom_factor"][0, moved] != other["zoom_factor"][0, moved]).any(axis=-1).all()
    assert np.array_equal(a["zoom_factor"][0, ~moved], other["zoom_factor"][0, ~moved])


def test_lit_loop_mixed_batch_equals_per_camera_batches(ctx, case):
    inten = lighting.sample_intensity(np.random.default_rng(3), (N_ITER, B))
    mixed_vs_per_camera(ctx, case, IDX, lit={"intensity": inten, "offset": lighting.OFFSET, "brightness_ratio": 0.7})


def test_image_only_network_mixed_batch_equals_per_camera_batches(meshes, case):
    c = make_ctx(meshes, synth.make_train_weights(0, input_mask=False), input_mask=False)
    try:
        mixed_vs_per_camera(c, case, IDX)
    finally:
        c.close()


def test_rgbd_network_mixed_batch_equals_per_camera_batches(meshes, case):
    c = make_ctx(meshes, synth.make_weights(0, input_depth=True), input_depth=True)
    try:
        a, _ = mixed_vs_per_camera(c, case, IDX, depth=True)
        # the host entry with the u16 depth frames = the device entry with their float conversion
        poses, se3 = c.refine_frames_host(case["u8"], IDX, case["cls"], case["ini"], KF, N_ITER, pixel_means_rgb=MEANS,
                                          depth_frames_u16=case["u16"], depth_factor=1000.0)
        assert np.array_equal(poses, a["poses"]) and np.array_equal(se3, a["se3"])
    finally:
        c.close()


def test_past_sixteen_instances_on_a_forty_instance_context(meshes, case):
    idx = np.random.default_rng(9).integers(0, F, size=33).astype(np.int32)
    idx[:F] = np.arange(F)
    c33 = make_frames(meshes, KF, idx, 97)
    c = make_ctx(meshes, synth.make_weights(0), max_batch=40)
    try:
        mixed_vs_per_camera(c, c33, idx)
    finally:
        c.close()


# ------------------------------------------------------------------------------- 2. one camera everywhere = K9
def test_same_camera_for_every_frame_equals_refine_frames(ctx, case):
    for k in (0, 2):
        a = cpu(ctx.refine_frames(dev(case["img"]), dev(IDX), dev(case["cls"]), dev(case["ini"]),
                                  dev(np.repeat(CAMS[k][None], F, 0)), N_ITER, pixel_means_rgb=MEANS))
        sa = status(ctx, B)
        b = cpu(ctx.refine_frames(dev(case["img"]), dev(IDX), dev(case["cls"]), dev(case["ini"]), CAMS[k], N_ITER,
                                  pixel_means_rgb=MEANS))
        for key in KEYS:
            assert np.array_equal(a[key], b[key]), (k, key)
        assert np.array_equal(sa, status(ctx, B))


# ------------------------------------------------------------------------------------- 3. teacher-forced oracle
def test_teacher_forced_against_the_oracle_per_camera(ctx, meshes, case):
    """Each camera group against oracle.refine(K = its camera), every iteration fed the oracle's source pose: bbox and zoom
    factor bit-exact, se3 within 1e-4 (rotation) / 1e-3 (translation)."""
    n_iter = 2
    weights = synth.make_weights(0)
    c = case
    sel = np.concatenate([np.nonzero(CAM_OF_FRAME[IDX] == k)[0][:2] for k in range(3)])  # two instances per camera
    idx, cls, ini = IDX[sel], c["cls"][sel], c["ini"][sel]
    po = np.empty((n_iter, len(sel), 3, 4))
    ref = {k: np.empty((n_iter, len(sel)) + s, t) for k, s, t in
           (("se3", (7,), np.float32), ("zoom_factor", (4,), np.float32), ("bbox", (8,), np.int32))}
    for k in range(3):
        s = np.nonzero(CAM_OF_FRAME[idx] == k)[0]
        r = O.refine(weights, meshes, cls[s], c["img"][idx[s]], ini[s], CAMS[k], n_iter, MEANS.astype(np.float32))
        po[0, s] = ini[s]
        po[1:, s] = r["poses"][:-1]
        for key in ref:
            ref[key][:, s] = r[key]
    res = cpu(ctx.refine_frames(dev(c["img"]), dev(idx), dev(cls), dev(ini), dev(KF), n_iter, pixel_means_rgb=MEANS,
                                precision=capi.PREC_FP16, pose_override=dev(po)))
    assert np.array_equal(res["bbox"], ref["bbox"])
    assert np.array_equal(res["zoom_factor"], ref["zoom_factor"])
    assert np.abs(res["se3"][..., :4] - ref["se3"][..., :4]).max() < 1e-4
    assert np.abs(res["se3"][..., 4:] - ref["se3"][..., 4:]).max() < 1e-3


# -------------------------------------------------------------------------------------------------- 4. graph replay
def test_graph_replay_intrinsics_rewrite_and_interleaving(ctx, case):
    """On a side stream (the legacy default stream cannot be captured): new intrinsics in a captured K buffer take effect at
    the next replay without a new capture, a second K buffer is a second graph, and a call with K9 interleaves."""
    s = torch.cuda.Stream(device=DEV)
    s.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(s):
        graph_replay_body(ctx, case)
    torch.cuda.synchronize()


def graph_replay_body(ctx, case):
    c = case
    frames, fidx, cls, ini = dev(c["img"]), dev(IDX), dev(c["cls"]), dev(c["ini"])
    kf2 = CAMS[(CAM_OF_FRAME + 1) % 3]                           # every frame under another camera
    args = (fidx, cls, ini)
    count = lambda: capi.lib.dim_debug_graph_count(ctx._h)       # noqa: E731

    def same(r, want):
        for k in KEYS:
            assert torch.equal(r[k], want[k]), k
    capi.check(capi.lib.dim_debug_set_option(ctx._h, b"graph", 0))  # eager references, launch by launch
    want = {name: {k: v.clone() for k, v in ctx.refine_frames(frames, *args, dev(kf), N_ITER, pixel_means_rgb=MEANS).items()}
            for name, kf in (("a", KF), ("b", kf2))}
    want_one = {k: v.clone() for k, v in ctx.refine_frames(frames, *args, CAMS[1], N_ITER, pixel_means_rgb=MEANS).items()}
    assert not torch.equal(want["a"]["zoom_factor"], want["b"]["zoom_factor"])
    capi.check(capi.lib.dim_debug_set_option(ctx._h, b"graph", 1))
    n0 = count()
    kbuf, kbuf2 = dev(KF), dev(KF)
    out = out2 = out1 = None
    for rep in range(3):  # eager, capture, replay -- two K buffers and a K9 call interleaved
        out = ctx.refine_frames(frames, *args, kbuf, N_ITER, pixel_means_rgb=MEANS, out=out)
        same(out, want["a"])
        out2 = ctx.refine_frames(frames, *args, kbuf2, N_ITER, pixel_means_rgb=MEANS, out=out2)
        same(out2, want["a"])
        out1 = ctx.refine_frames(frames, *args, CAMS[1], N_ITER, pixel_means_rgb=MEANS, out=out1)
        same(out1, want_one)
    assert count() == n0 + 3                                     # two K buffers are two graphs; K9 is a third
    kbuf.copy_(dev(kf2))                                         # new intrinsics in the captured buffer: a replay reads them
    out = ctx.refine_frames(frames, *args, kbuf, N_ITER, pixel_means_rgb=MEANS, out=out)
    same(out, want["b"])
    out2 = ctx.refine_frames(frames, *args, kbuf2, N_ITER, pixel_means_rgb=MEANS, out=out2)
    same(out2, want["a"])
    assert count() == n0 + 3


# ---------------------------------------------------------------------------------------- 5. host entry = device entry
@pytest.mark.parametrize("sync", [True, False], ids=["sync", "async"])
def test_host_entry_equals_device_entry(ctx, case, sync):
    c = case
    a = cpu(ctx.refine_frames(dev(c["img"]), dev(IDX), dev(c["cls"]), dev(c["ini"]), dev(KF), N_ITER, pixel_means_rgb=MEANS))
    sa = status(ctx, B)
    poses = torch.empty((N_ITER, B, 3, 4), dtype=torch.float64).pin_memory()
    se3 = torch.empty((N_ITER, B, 7), dtype=torch.float32).pin_memory()
    ctx.refine_frames_host(torch.from_numpy(c["u8"]).pin_memory(), torch.from_numpy(IDX).pin_memory(), c["cls"], c["ini"],
                           torch.from_numpy(KF).pin_memory(), N_ITER, pixel_means_rgb=MEANS, poses_out=poses, se3_out=se3,
                           sync=sync)
    torch.cuda.synchronize()
    assert np.array_equal(poses.numpy(), a["poses"]) and np.array_equal(se3.numpy(), a["se3"])
    assert np.array_equal(status(ctx, B), sa)


# --------------------------------------------------------------------------------------------------- 6. PoseRefiner
def test_pose_refiner_cameras_equal_per_camera_refiners(meshes):
    n, nf = 37, 11
    rng = np.random.default_rng(17)
    frame_of = rng.integers(0, nf, size=n).astype(np.int32)
    frame_of[:8] = 3
    cam = np.arange(nf) % 3
    kf = CAMS[cam]
    c = make_frames(meshes, kf, frame_of, 101)
    weights = synth.make_weights(0)
    r = PoseRefiner(meshes, weights, CAMS[0], device=0, max_batch=B, n_iter=N_ITER, n_slots=2)
    try:
        got = r.refine_frames(c["u8"], frame_of, c["cls"], c["ini"], K_frames=kf)
        per_instance = r.refine(c["u8"][frame_of], c["cls"], c["ini"], K=kf[frame_of])
        assert got.shape == (N_ITER, n, 3, 4) and np.isfinite(got).all()
        assert np.array_equal(got, per_instance)
        with pytest.raises(ValueError, match="K_frames: expected shape"):
            r.refine_frames(c["u8"], frame_of, c["cls"], c["ini"], K_frames=kf[:-1])
        with pytest.raises(ValueError, match="K: expected one camera per instance"):
            r.refine(c["u8"][frame_of], c["cls"], c["ini"], K=kf)
    finally:
        r.close()
    for k in range(3):
        s = np.nonzero(cam[frame_of] == k)[0]
        rk = PoseRefiner(meshes, weights, CAMS[k], device=0, max_batch=B, n_iter=N_ITER, n_slots=1)
        try:
            want = rk.refine_frames(c["u8"], frame_of[s], c["cls"][s], c["ini"][s])
        finally:
            rk.close()
        assert np.array_equal(got[:, s], want), k


# ---------------------------------------------------------------------------------------------- 7. lm6d_io -K.txt
def test_lm6d_evaluate_with_per_pair_intrinsics_equals_camera_groups(tmp_path):
    import cv2
    import lm6d_fixture
    root = str(tmp_path / "mixed")
    classes, ms = lm6d_fixture.build(root, n_per_class=2)
    k2 = CAMS[1]
    with_k = []  # the second pair of each class: observed by the second camera, with its -K.txt
    for ci, cname in enumerate(classes):
        obs, _ = lm6d_io.LM6DRefine(root, classes, "val").pairs(cname)[1]
        d = os.path.join(root, "data", "observed")
        pose = lm6d_io.read_pose(os.path.join(root, "data", "gt_observed", cname, obs.split("/")[1] + "-pose.txt"))
        r = O.render(ms[cname], pose, k2)
        cv2.imwrite(os.path.join(d, obs + "-color.png"), synth.composite_observed(r["bgr"], r["mask"], 5 + ci))
        np.savetxt(os.path.join(d, obs + "-K.txt"), k2.astype(np.float64))
        with_k.append(obs)
    ds = lm6d_io.LM6DRefine(root, classes, "val")
    assert np.array_equal(ds.load_pair(classes[0], ds.pairs(classes[0])[1])["K"], k2.astype(np.float64))
    assert "K" not in ds.load_pair(classes[0], ds.pairs(classes[0])[0])
    weights = synth.make_weights(0)
    res, poses, gt = lm6d_io.evaluate(ds, weights, synth.K_LINEMOD, n_iter=2)
    assert np.isfinite(poses).all() and "arp_2d" in res

    def group(name, keep_k, K):
        g = str(tmp_path / name)
        shutil.copytree(root, g)
        for cname in classes:
            pairs = [p for p in ds.pairs(cname) if (p[0] in with_k) == keep_k]
            with open(os.path.join(g, "image_set", "val_%s.txt" % cname), "w") as f:
                f.write("\n".join("%s %s" % p for p in pairs) + "\n")
        for obs in with_k:
            os.remove(os.path.join(g, "data", "observed", obs + "-K.txt"))
        return lm6d_io.evaluate(lm6d_io.LM6DRefine(g, classes, "val"), weights, K, n_iter=2)
    order = [p[0] in with_k for cname in classes for p in ds.pairs(cname)]
    mask = np.array(order)
    for keep_k, K in ((False, synth.K_LINEMOD), (True, k2)):
        _, p, g_ = group("cam%d" % keep_k, keep_k, K)
        sel = mask if keep_k else ~mask
        assert np.array_equal(poses[:, sel], p) and np.array_equal(gt[sel], g_)


# ------------------------------------------------------------------------------------------------------ 8. errors
def test_error_paths(ctx, case):
    c = case
    frames, fidx, cls, ini = dev(c["img"]), dev(IDX), dev(c["cls"]), dev(c["ini"])
    means = capi.farr(MEANS, 3, capi.C.c_double)
    poses = torch.full((N_ITER, B, 3, 4), 7.0, dtype=torch.float64, device=DEV)
    p = capi.C.c_void_p
    kf, K9 = dev(KF.astype(np.float32)), capi.farr(KF[0].astype(np.float32).reshape(9), 9)
    hposes = np.full((N_ITER, B, 3, 4), 7.0)
    hu8, hidx, hkf, hcls, hini = (np.ascontiguousarray(a) for a in (c["u8"], IDX, KF.astype(np.float32), c["cls"], c["ini"]))

    def dev_call(F_=F, iptr=p(fidx.data_ptr()), k9=None, kptr=p(kf.data_ptr())):
        return capi.lib.dim_refine(ctx._h, p(frames.data_ptr()), F_, iptr, k9, kptr, p(cls.data_ptr()), p(ini.data_ptr()), B,
                                   N_ITER, 0.25, 6.0, means, capi.PREC_FP16, None, p(poses.data_ptr()), None, None, None, None,
                                   None, ctx._stream())

    def host_call(F_=F, iptr=p(hidx.ctypes.data), k9=None, kptr=p(hkf.ctypes.data)):
        return capi.lib.dim_refine_host_async(ctx._h, p(hu8.ctypes.data), F_, iptr, k9, kptr, p(hcls.ctypes.data),
                                              p(hini.ctypes.data), B, N_ITER, 0.25, 6.0, means, capi.PREC_FP16,
                                              p(hposes.ctypes.data), None, None, 1000.0, None, ctx._stream())
    for call, entry, kptr in ((dev_call, b"dim_refine: ", p(kf.data_ptr())),
                              (host_call, b"dim_refine_host_async: ", p(hkf.ctypes.data))):
        for k9, kp in ((None, None), (K9, kptr)):   # neither K, both K
            assert call(k9=k9, kptr=kp) == 2 and entry + b"exactly one of K9_host and K_frames" in capi.lib.dim_last_error()
        assert call(iptr=None) == 2 and entry + b"frame_idx is NULL" in capi.lib.dim_last_error()   # F = 6, B = 16
        assert b"F must equal B" in capi.lib.dim_last_error()
    torch.cuda.synchronize()
    assert (poses == 7.0).all() and (hposes == 7.0).all()

    def bad(f, r, col, v):
        k = KF.copy()
        k[f, r, col] = v
        return k
    for k, frame, why in ((bad(2, 0, 0, np.nan), 2, "not finite"), (bad(4, 1, 2, np.inf), 4, "not finite"),
                          (bad(4, 0, 0, 0.0), 4, "fx and fy must be > 0"), (bad(1, 1, 1, -5.0), 1, "fx and fy must be > 0"),
                          (bad(1, 0, 1, 0.5), 1, "skew"), (bad(3, 1, 0, 0.5), 3, "skew"),
                          (bad(5, 2, 2, 2.0), 5, "last row"), (bad(0, 2, 0, 1e-3), 0, "last row")):
        out_p = np.full((N_ITER, B, 3, 4), 7.0)
        out_s = np.full((N_ITER, B, 7), 7.0, np.float32)
        with pytest.raises(capi.DeepIMError, match=r"dim_refine_host_async: frame %d has intrinsics .*%s" % (frame, why)):
            ctx.refine_frames_host(c["u8"], IDX, c["cls"], c["ini"], k, N_ITER, pixel_means_rgb=MEANS, poses_out=out_p,
                                   se3_out=out_s)
        torch.cuda.synchronize()
        assert (out_p == 7.0).all() and (out_s == 7.0).all()
    with pytest.raises(ValueError, match="one camera per frame"):
        ctx.refine_frames(frames, fidx, cls, ini, dev(KF[:-1]), N_ITER, pixel_means_rgb=MEANS)
    with pytest.raises(ValueError, match="one camera per frame"):
        ctx.refine_frames_host(c["u8"], IDX, c["cls"], c["ini"], np.concatenate([KF, KF[:1]]), N_ITER, pixel_means_rgb=MEANS)
    # the frame index checks hold with per-frame intrinsics too
    wrong = IDX.copy()
    wrong[3] = F
    with pytest.raises(capi.DeepIMError, match="dim_refine_host_async: instance 3 has frame index 6"):
        ctx.refine_frames_host(c["u8"], wrong, c["cls"], c["ini"], KF, N_ITER, pixel_means_rgb=MEANS)
    with pytest.raises(capi.DeepIMError, match="depth_frames_u16_host"):
        ctx.refine_frames_host(c["u8"], IDX, c["cls"], c["ini"], KF, N_ITER, pixel_means_rgb=MEANS,
                               depth_frames_u16=c["u16"])


def test_device_frame_index_out_of_range_uses_frame_zero_camera(ctx, case):
    """A bad device index: the instance observes frame 0 with frame 0's camera and carries status bit 3."""
    c = case
    badi = IDX.copy()
    badi[2], badi[7] = 9, -1
    clamp = badi.copy()
    clamp[2] = clamp[7] = 0
    args = (dev(c["cls"]), dev(c["ini"]), dev(KF), N_ITER)
    a = cpu(ctx.refine_frames(dev(c["img"]), dev(badi), *args, pixel_means_rgb=MEANS))
    sa = status(ctx, B)
    b = cpu(ctx.refine_frames(dev(c["img"]), dev(clamp), *args, pixel_means_rgb=MEANS))
    sb = status(ctx, B)
    for k in KEYS:
        assert np.array_equal(a[k], b[k]), k
    assert ((sa[:, [2, 7]] & 8) == 8).all() and np.array_equal(sa & ~8, sb)
