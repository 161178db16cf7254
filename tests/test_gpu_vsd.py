"""GPU: the Visible Surface Discrepancy (dim_pose_error_vsd, Context.pose_error_vsd, PoseRefiner.vsd, pose_eval.evaluate_pose_vsd,
lm6d_io.evaluate's vsd) held bit for bit to the oracle's contract (oracle/vsd.py).

The scene: B = 16 instances of two classes (the C2 blob and a C3 mesh) observing 6 frames from three cameras through a
frame map.  Each frame's observed depth is the object at its true pose, rounded to mm, with rectangular holes and an
occluder 6 cm in front of part of it; frame 5's object is cut by the right border.  The estimates are 1-10 mm / 1-6 deg
away; instance 13's estimate is out of view and instance 14 has a bad class."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

import lm6d_fixture  # noqa: E402
from test_icp_oracle import mm, perturb  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle import vsd as V  # noqa: E402
from deepim_b200 import lighting, lm6d_io, pose_eval, synth  # noqa: E402
from deepim_b200._capi import farr, lib  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.refiner import PoseRefiner, plan_frame_batches  # noqa: E402

DEV = torch.device("cuda", 0)
K = synth.K_LINEMOD
B, F = 16, 6
DELTA, TAUS = 0.015, (0.005, 0.01, 0.02, 0.05)


def pinhole(fx, fy, cx, cy):
    return np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], np.float32)


CAMS = np.stack([K, pinhole(1066.778, 1067.487, 312.99, 241.31), pinhole(800.0, 790.0, 410.5, 190.25)])


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def observe(mesh, G, Kc, rng):
    """sensor-like depth of the mesh at G: mm-quantised, three holes, an occluder 6 cm in front of its upper left part"""
    d = mm(O.render(mesh, G, Kc, want=("depth",))["depth"])
    ys, xs = np.nonzero(d)
    for _ in range(3):
        k = rng.integers(len(ys))
        d[max(ys[k] - 6, 0):ys[k] + 6, max(xs[k] - 8, 0):xs[k] + 8] = 0.0
    d[max(ys.min() - 4, 0):(ys.min() + ys.max()) // 2, max(xs.min() - 4, 0):(xs.min() + xs.max()) // 2] = np.float32(
        float(G[2, 3]) - 0.06)
    return d


def frames_scene(meshes, counts, seed):
    """len(counts) frames (frame f: camera f % 3, class f % 2), counts[f] instances per frame in a shuffled order"""
    rng = np.random.default_rng(seed)
    nf = len(counts)
    gt = synth.sample_pose_pairs(nf, seed)[0]
    cam = np.arange(nf) % 3
    u16 = np.stack([np.rint(observe(meshes[f % 2], gt[f], CAMS[cam[f]], rng).astype(np.float64) * 1000).astype(np.uint16)
                    for f in range(nf)])
    frame_of = rng.permutation(np.repeat(np.arange(nf), counts)).astype(np.int32)
    est = np.stack([perturb(gt[f], rng, t=rng.uniform(0.001, 0.01), deg=rng.uniform(1.0, 6.0)) for f in frame_of])
    return dict(u16=u16, depth=O.depth_from_u16(u16, 1000.0), frame_of=frame_of, cls=(frame_of % 2).astype(np.int32),
                est=est, gt=gt[frame_of], Kf=CAMS[cam])


def scene(meshes):
    rng = np.random.default_rng(3)
    gt = synth.sample_pose_pairs(F, 3)[0]
    gt[5, 0, 3] = gt[5, 2, 3] * (640 - 410.5) / 800.0  # frame 5 (camera 2): the object centred on the right border
    cam = np.arange(F) % 3
    depth = np.stack([observe(meshes[f % 2], gt[f], CAMS[cam[f]], rng) for f in range(F)]).astype(np.float32)
    frame_of = rng.permutation(np.repeat(np.arange(F), [3, 3, 3, 3, 2, 2])).astype(np.int32)
    cls = (frame_of % 2).astype(np.int32)
    est = np.stack([perturb(gt[f], rng, t=rng.uniform(0.001, 0.01), deg=rng.uniform(1.0, 6.0)) for f in frame_of])
    est[13, :, 3] = [5.0, 0.0, 0.8]  # out of view
    cls[14] = 5                      # no such class
    return dict(depth=depth, frame_of=frame_of, cls=cls, est=est, gt=gt[frame_of], Kf=CAMS[cam])


@pytest.fixture(scope="module")
def meshes():
    ms = [synth.make_blob(), synth.make_linemod_like_set()[4]]
    for m in ms:
        m.normals = synth.vertex_normals(m)
    return ms


def context(meshes, **kw):
    ctx = Context(0, max_batch=B, max_classes=2, max_verts=20000, max_faces=40000, **kw)
    for i, m in enumerate(meshes):
        ctx.upload_mesh(i, m)
    return ctx


@pytest.fixture(scope="module")
def ctx(meshes):
    c = context(meshes)
    yield c
    c.close()


@pytest.fixture(scope="module")
def case(meshes):
    return scene(meshes)


def call(ctx, s, sel=None, frame_map=True, **kw):
    sel = np.arange(len(s["cls"])) if sel is None else sel
    if frame_map:
        args = (dev(s["depth"]), dev(s["cls"][sel]), dev(s["est"][sel]), dev(s["gt"][sel]), s["Kf"])
        kw.setdefault("frame_idx", dev(s["frame_of"][sel]))
    else:  # every instance its own copy of its frame and camera
        f = s["frame_of"][sel]
        args = (dev(s["depth"][f]), dev(s["cls"][sel]), dev(s["est"][sel]), dev(s["gt"][sel]), s["Kf"][f])
    r = ctx.pose_error_vsd(*args, DELTA, TAUS, **kw)
    return {k: v.cpu().numpy() for k, v in r.items()}


@pytest.fixture(scope="module")
def run(ctx, case):
    return call(ctx, case)


def test_err_and_status_equal_the_oracle(run, case, meshes):
    err, st = V.vsd(meshes, case["cls"], case["est"], case["gt"], case["depth"], case["Kf"], DELTA, TAUS,
                    frame_idx=case["frame_of"])
    assert np.array_equal(run["err"], err) and np.array_equal(run["status"], st)
    assert list(st[:13]) == [0] * 13 and st[13] == 0 and st[14] == 3 and st[15] == 0
    assert (run["err"][13] == 1.0).all() and (run["err"][14] == 1.0).all()
    good = np.r_[0:13, 15]
    assert (run["err"][good, 0] > 0).all() and (run["err"][good, -1] < 0.5).all()
    assert (np.diff(run["err"], axis=1) <= 0).all()
    f5 = np.nonzero(case["frame_of"] == 5)[0]
    assert len(f5) and (case["depth"][5][:, -1] > 0).any()  # the object cut by the border is in the scene


def test_bad_frame_index_and_profile_record(ctx, case, run):
    fidx = case["frame_of"].copy()
    fidx[2] = 9  # out of [0, 6): frame 0 and its camera, bit 3
    ctx.profile_enable(True)
    r = call(ctx, case, frame_idx=dev(fidx))
    stages, n = ctx.profile_read()
    ctx.profile_enable(False)
    assert n == 1 and stages["render"] > 0 and stages["zoom"] > 0
    assert r["status"][2] & 8 and not (np.delete(r["status"], 2) & 8).any()
    moved = dict(case, frame_of=np.where(np.arange(B) == 2, 0, case["frame_of"]).astype(np.int32))
    assert np.array_equal(r["err"], call(ctx, moved)["err"])


def test_cameras_frame_map_and_batch_sizes_equal_their_reference_calls(ctx, case, run):
    """K_frames against K9 calls per camera, the frame map against gathered frames, B = 1 against B = max_batch"""
    cam_of = case["frame_of"] % 3
    for cam in range(3):
        sel = np.nonzero(cam_of == cam)[0]
        f = case["frame_of"][sel]
        r = ctx.pose_error_vsd(dev(case["depth"][f]), dev(case["cls"][sel]), dev(case["est"][sel]), dev(case["gt"][sel]),
                               CAMS[cam], DELTA, TAUS)
        for k in run:
            assert np.array_equal(r[k].cpu().numpy(), run[k][sel]), (cam, k)
    gathered = call(ctx, case, frame_map=False)
    for b in range(B):
        one = call(ctx, case, sel=np.array([b]), frame_map=False)
        for k in run:
            assert np.array_equal(one[k], run[k][b:b + 1]), (b, k)
    for k in run:
        assert np.array_equal(gathered[k], run[k]), k


def test_two_runs_identical_and_every_context_variant(meshes, case, run):
    for kw in ({}, {"input_mask": False}, {"input_depth": True}):
        c = context(meshes, **kw)
        for _ in range(2):
            r = call(c, case)
            for k in run:
                assert np.array_equal(r[k], run[k]), (kw, k)
        c.close()


def test_error_paths_leave_outputs_untouched(ctx, case):
    depth, cls, est, gt = dev(case["depth"][case["frame_of"]]), dev(case["cls"]), dev(case["est"]), dev(case["gt"])
    err = torch.full((B, 4), -7.0, dtype=torch.float64, device=DEV)
    st = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    K9 = farr(K.reshape(9), 9)
    taus = farr(TAUS, ctype=C.c_double)
    p = lambda t: C.c_void_p(t.data_ptr())
    base = dict(ctx=ctx._h, depth=p(depth), F=B, fidx=None, K9=K9, Kf=None, cls=p(cls), est=p(est), gt=p(gt), B=B, zn=0.25,
                zf=6.0, delta=DELTA, taus=taus, n_tau=4, err=p(err), st=p(st), stream=None)
    nonpinhole = K.copy()
    nonpinhole[0, 1] = 1.0
    Kf = dev(np.stack([K] * B))
    fidx = dev(np.zeros(B, np.int32))
    bad_tau = lambda v: farr([0.01, v, 0.02, 0.05], ctype=C.c_double)
    for over in ({"ctx": None}, {"depth": None}, {"cls": None}, {"est": None}, {"gt": None}, {"taus": None}, {"err": None},
                 {"B": 0}, {"B": B + 1}, {"F": 0, "fidx": p(fidx)}, {"F": B + 1, "fidx": p(fidx)}, {"F": B - 1},
                 {"n_tau": 0}, {"n_tau": 17}, {"delta": 0.0}, {"delta": -0.01}, {"delta": float("nan")},
                 {"delta": float("inf")}, {"taus": bad_tau(0.0)}, {"taus": bad_tau(-0.01)}, {"taus": bad_tau(float("nan"))},
                 {"taus": bad_tau(float("inf"))}, {"K9": None}, {"Kf": p(Kf)}, {"K9": farr(nonpinhole.reshape(9), 9)},
                 {"K9": farr([float("nan")] + list(K.reshape(9)[1:]), 9)}):
        a = dict(base, **over)
        assert lib.dim_pose_error_vsd(*a.values()) == 2, over
        if over != {"ctx": None}:
            assert b"dim_pose_error_vsd" in lib.dim_last_error(), over
        torch.cuda.synchronize()
        assert (err == -7.0).all() and (st == -7).all(), over
    assert lib.dim_pose_error_vsd(*dict(base, st=None).values()) == 0  # status is optional
    torch.cuda.synchronize()
    assert (err != -7.0).all() and (st == -7).all()
    assert lib.dim_pose_error_vsd(*base.values()) == 0
    torch.cuda.synchronize()
    assert (st != -7).all()


def test_context_equals_the_c_entry(ctx, case, run):
    err = torch.empty((B, 4), dtype=torch.float64, device=DEV)
    st = torch.empty((B,), dtype=torch.int32, device=DEV)
    p = lambda t: C.c_void_p(t.data_ptr())
    Kf = dev(case["Kf"])
    args = [dev(case[k]) for k in ("depth", "frame_of", "cls", "est", "gt")]
    assert lib.dim_pose_error_vsd(ctx._h, p(args[0]), F, p(args[1]), None, p(Kf), p(args[2]), p(args[3]), p(args[4]), B, 0.25,
                                  6.0, DELTA, farr(TAUS, ctype=C.c_double), 4, p(err), p(st), None) == 0
    torch.cuda.synchronize()
    assert np.array_equal(err.cpu().numpy(), run["err"]) and np.array_equal(st.cpu().numpy(), run["status"])


def test_pose_refiner_vsd_equals_context_per_batch(ctx, meshes):
    """37 instances over 11 frames from 3 cameras, u16 depth converted on the device"""
    counts = [4, 3, 5, 2, 4, 3, 5, 3, 4, 2, 2]
    s = frames_scene(meshes, counts, 9)
    n = len(s["cls"])
    assert n == 37
    ref = PoseRefiner(meshes, synth.make_weights(0), max_batch=B, n_iter=2)
    got = ref.vsd(s["u16"], s["cls"], s["est"], s["gt"], K_frames=s["Kf"], frame_of=s["frame_of"], taus=TAUS)
    ref.close()
    batches = plan_frame_batches(s["frame_of"], 11, B, 0, n, s["Kf"])
    assert len(batches) == 3
    for a, b, frames, local, Kb in batches:
        r = ctx.pose_error_vsd(dev(s["depth"][frames]), dev(s["cls"][a:b]), dev(s["est"][a:b]), dev(s["gt"][a:b]), Kb, DELTA,
                               TAUS, frame_idx=dev(local))
        for k in got:
            assert np.array_equal(r[k].cpu().numpy(), got[k][a:b]), (a, k)
    assert (got["status"] == 0).all() and got["err"].shape == (n, 4)


def test_refinement_graphs_replay_unchanged_after_vsd(meshes, case):
    """graphs of the unlit, lit and RGB-D chains captured before a VSD call replay to the same bits after it"""
    Bq, n_iter = 4, 2
    obs, ini = synth.sample_pose_pairs(Bq, 17)
    cls = np.zeros(Bq, np.int32)
    rend = [O.render(meshes[0], obs[b], K, means_rgb=synth.PIXEL_MEANS_RGB) for b in range(Bq)]
    img = dev(np.stack([synth.transform_image(synth.composite_observed(r["bgr"], r["mask"], b)) for b, r in enumerate(rend)]))
    dobs = dev(np.stack([r["depth"] for r in rend])[:, None])
    inten = dev(lighting.sample_intensity(np.random.default_rng(3), (n_iter, Bq)))
    lit = {"intensity": inten, "offset": lighting.OFFSET, "brightness_ratio": 0.7}
    clsd, inid = dev(cls), dev(ini)
    side = torch.cuda.Stream(device=DEV)
    for kw, chains in (({}, ({}, {"lighting": lit})), ({"input_depth": True}, ({"depth_observed": dobs},))):
        c = context(meshes, **kw)
        c.load_weights(synth.make_weights(0, input_depth=bool(kw)))
        for ch in chains:
            out = None
            with torch.cuda.stream(side):
                for _ in range(3):  # eager, capture + launch, replay
                    out = c.refine(img, clsd, inid, K, n_iter, pixel_means_rgb=synth.PIXEL_MEANS_RGB, out=out, **ch)
                want = {k: v.clone() for k, v in out.items()}
                graphs = lib.dim_debug_graph_count(c._h)
                call(c, case)
                out = c.refine(img, clsd, inid, K, n_iter, pixel_means_rgb=synth.PIXEL_MEANS_RGB, out=out, **ch)
            side.synchronize()
            assert graphs >= 1 and lib.dim_debug_graph_count(c._h) == graphs
            for k in want:
                assert torch.equal(out[k], want[k]), (kw, list(ch), k)
        c.close()


def test_evaluate_with_vsd(tmp_path):
    classes, _ = lm6d_fixture.build(str(tmp_path), n_per_class=2)
    ds = lm6d_io.LM6DRefine(str(tmp_path), classes, "val")
    w = synth.make_weights(0)
    base = lm6d_io.evaluate(ds, w, K, n_iter=2, max_batch=3, icp_iters=2)
    off = lm6d_io.evaluate(ds, w, K, n_iter=2, max_batch=3, icp_iters=2, vsd=False)
    assert np.array_equal(base[1], off[1]) and repr(base[0]) == repr(off[0]) and "vsd" not in base[0]
    res, poses, gt = lm6d_io.evaluate(ds, w, K, n_iter=2, max_batch=3, icp_iters=2, vsd=True)
    assert np.array_equal(poses, base[1]) and poses.shape[0] == 3
    assert repr({k: v for k, v in res.items() if k != "vsd"}) == repr(base[0])
    meshes = [ds.mesh(c) for c in classes]
    ref = PoseRefiner(meshes, w, K=K, max_batch=3, n_iter=2)
    pairs = [(ci, p) for ci, c in enumerate(classes) for p in ds.pairs(c)]
    cls = np.array([ci for ci, _ in pairs], np.int32)
    u16 = np.stack([lm6d_io.read_depth_u16(str(tmp_path / "data" / "observed" / (p[0] + "-depth.png"))) for _, p in pairs])
    errs = np.stack([ref.vsd(u16, cls, p, gt)["err"][:, 0] for p in poses])
    ref.close()
    assert np.array_equal(res["vsd"]["errors"], errs)
    exp = pose_eval.evaluate_pose_vsd(errs, cls, len(classes), 0.3)
    assert repr(exp["mean"]) == repr(res["vsd"]["mean"]) and repr(exp["classes"]) == repr(res["vsd"]["classes"])
    assert len(res["vsd"]["mean"]["recall"]) == 3
