"""GPU: projective point-to-plane ICP against observed depth (dim_icp, Context.icp, PoseRefiner.icp, lm6d_io.evaluate's
icp_iters) held to the oracle's contract (oracle/icp.py).

The scene: B = 16 instances of two classes (the C2 blob and a C3 mesh), each observing its own frame: the object rendered
at its true pose, depth rounded to mm with rectangular holes, the initial pose 1 cm / 3 deg away.  Instance 13 is out of
view (bit 0), 14 has a bad class (bits 0 + 1), 15 observes a frame that is all holes (bit 4)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

import lm6d_fixture  # noqa: E402
from test_icp_oracle import ADD_RATIO_BOUND, add, mm, perturb  # noqa: E402
from oracle import icp as I  # noqa: E402
from oracle import oracle as O  # noqa: E402
from deepim_b200 import lighting, lm6d_io, pose_eval, synth  # noqa: E402
from deepim_b200._capi import farr, lib  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.refiner import PoseRefiner, plan_frame_batches  # noqa: E402

DEV = torch.device("cuda", 0)
K = synth.K_LINEMOD
H, W = 480, 640
B, N_ITER = 16, 10
KEYS = ("poses", "inliers", "rms", "status")


def pinhole(fx, fy, cx, cy):
    return np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], np.float32)


CAMS = np.stack([K, pinhole(1066.778, 1067.487, 312.99, 241.31), pinhole(800.0, 790.0, 410.5, 190.25)])


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def make_meshes():
    return [synth.make_blob(), synth.make_linemod_like_set()[4]]


def observe(mesh, G, Kc, rng):
    """the depth a sensor gives of the mesh at G: mm-quantised, with three rectangular holes over the object"""
    d = mm(O.render(mesh, G, Kc, want=("depth",))["depth"])
    ys, xs = np.nonzero(d)
    for _ in range(3):
        if len(ys):
            k = rng.integers(len(ys))
            d[max(ys[k] - 8, 0):ys[k] + 8, max(xs[k] - 12, 0):xs[k] + 12] = 0.0
    return d


def scene(meshes, seed=3):
    rng = np.random.default_rng(seed)
    gt = synth.sample_pose_pairs(B, seed)[0]
    cls = (np.arange(B) % 2).astype(np.int32)
    depth = np.stack([observe(meshes[cls[b]], gt[b], K, rng) for b in range(B)])
    P0 = np.stack([perturb(gt[b], rng) for b in range(B)])
    P0[13, :, 3] = [5.0, 0.0, 0.8]   # out of view
    cls[14] = 5                      # no such class
    depth[15] = 0.0                  # all holes
    return dict(gt=gt, cls=cls, depth=depth.astype(np.float32), P0=P0)


def frames_scene(meshes, counts, seed):
    """len(counts) frames from the three cameras (frame f: camera f % 3, class f % 2), counts[f] instances per frame in a
    shuffled order, each near its frame's object"""
    rng = np.random.default_rng(seed)
    F = len(counts)
    gt = synth.sample_pose_pairs(F, seed)[0]
    cam = np.arange(F) % 3
    u16 = np.stack([np.rint(observe(meshes[f % 2], gt[f], CAMS[cam[f]], rng).astype(np.float64) * 1000).astype(np.uint16)
                    for f in range(F)])
    frame_of = rng.permutation(np.repeat(np.arange(F), counts)).astype(np.int32)
    P0 = np.stack([perturb(gt[f], rng) for f in frame_of])
    return dict(u16=u16, depth=O.depth_from_u16(u16, 1000.0), frame_of=frame_of, cls=(frame_of % 2).astype(np.int32), P0=P0,
                Kf=CAMS[cam])


@pytest.fixture(scope="module")
def meshes():
    ms = make_meshes()
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


@pytest.fixture(scope="module")
def run(ctx, case):
    r = ctx.icp(dev(case["depth"]), dev(case["cls"]), dev(case["P0"]), K, N_ITER)
    return {k: v.cpu().numpy() for k, v in r.items()}


def test_status_bits(run):
    st = run["status"]
    assert (st[:, :13] == 0).all(), st
    assert (st[:, 13] == 1).all() and (st[:, 14] == 3).all() and (st[:, 15] == 16).all()
    assert (run["inliers"][:, 13:15] == 0).all() and (run["inliers"][:, 15] == 0).all()


def test_teacher_forced_parity_every_iteration(run, case, meshes):
    """the oracle's single step fed the device's P_k: the same inlier count, P_{k+1} within 1e-10, rms within 1e-6"""
    for b in range(B):
        if case["cls"][b] >= len(meshes):
            assert np.array_equal(run["poses"][:, b], np.broadcast_to(case["P0"][b], (N_ITER, 3, 4)))
            continue
        ren = O.render(meshes[case["cls"][b]], case["P0"][b], K, want=("depth",))["depth"]
        surf = I.model_surface(ren, K, 0.02)
        for k in range(N_ITER):
            Pk = case["P0"][b] if k == 0 else run["poses"][k - 1, b]
            P1, c, e, _, _ = I.step(ren, case["P0"][b], Pk, case["depth"][b], K, surface=surf)
            assert c == run["inliers"][k, b], (b, k)
            assert np.abs(P1 - run["poses"][k, b]).max() < 1e-10, (b, k)
            rms = np.sqrt(e / c) if c else 0.0
            assert abs(run["rms"][k, b] - rms) <= 1e-6 * max(rms, 1e-30), (b, k)


def test_free_running_matches_oracle_and_converges(run, case, meshes):
    ref = I.icp(meshes, case["cls"], case["P0"], case["depth"], K, N_ITER)
    assert np.array_equal(ref["status"], run["status"])
    assert np.abs(ref["poses"][-1] - run["poses"][-1]).max() < 1e-6
    for b in range(13):
        pts = meshes[case["cls"][b]].verts.astype(np.float64)
        ratio = add(run["poses"][-1, b], case["gt"][b], pts) / add(case["P0"][b], case["gt"][b], pts)
        assert ratio <= ADD_RATIO_BOUND, (b, ratio)


def test_two_runs_identical_and_every_context_variant(meshes, case, run):
    args = (dev(case["depth"]), dev(case["cls"]), dev(case["P0"]), K, N_ITER)
    for kw in ({}, {"input_mask": False}, {"input_depth": True}):
        c = context(meshes, **kw)
        for _ in range(2):
            r = c.icp(*args)
            for k in KEYS:
                assert np.array_equal(r[k].cpu().numpy(), run[k]), (kw, k)
        c.close()


def test_frame_map_with_cameras_equals_per_camera_calls(ctx, meshes):
    """F = 6 frames from 3 cameras, 1-5 instances per frame, against K9 calls on each camera's sub-batch over its
    instances' gathered frames"""
    s = frames_scene(meshes, [5, 1, 3, 2, 4, 1], 8)
    full = ctx.icp(dev(s["depth"]), dev(s["cls"]), dev(s["P0"]), s["Kf"], N_ITER, frame_idx=dev(s["frame_of"]))
    cam_of = np.arange(6)[s["frame_of"]] % 3
    for cam in range(3):
        sel = np.nonzero(cam_of == cam)[0]
        sub = ctx.icp(dev(s["depth"][s["frame_of"][sel]]), dev(s["cls"][sel]), dev(s["P0"][sel]), CAMS[cam], N_ITER)
        for k in KEYS:
            assert torch.equal(sub[k], full[k][:, torch.from_numpy(sel).to(DEV)]), (cam, k)
    assert (full["status"] == 0).all()
    bad = s["frame_of"].copy()
    bad[2] = 9  # out of [0, 6): frame 0 (and its camera), bit 3
    r = ctx.icp(dev(s["depth"]), dev(s["cls"]), dev(s["P0"]), s["Kf"], 2, frame_idx=dev(bad))
    assert (r["status"][:, 2].cpu().numpy() & 8).all() and not (r["status"][:, 3:].cpu().numpy() & 8).any()


def test_error_paths_leave_outputs_untouched(ctx, case):
    depth, cls, P0 = dev(case["depth"]), dev(case["cls"]), dev(case["P0"])
    outs = [torch.full((2, B, 3, 4), -7.0, dtype=torch.float64, device=DEV), torch.full((2, B), -7, dtype=torch.int32, device=DEV),
            torch.full((2, B), -7.0, device=DEV), torch.full((2, B), -7, dtype=torch.int32, device=DEV)]
    K9 = farr(K.reshape(9), 9)
    p = lambda t: C.c_void_p(t.data_ptr())
    base = dict(ctx=ctx._h, depth=p(depth), F=B, fidx=None, K9=K9, Kf=None, cls=p(cls), pose=p(P0), B=B, n_iter=2, zn=0.25,
                zf=6.0, md=0.02, mp=64, poses=p(outs[0]), inl=p(outs[1]), rms=p(outs[2]), st=p(outs[3]), stream=None)
    nonpinhole = K.copy()
    nonpinhole[0, 1] = 1.0
    Kf = dev(np.stack([K] * B))
    fidx = dev(np.zeros(B, np.int32))
    for over in ({"ctx": None}, {"depth": None}, {"cls": None}, {"pose": None}, {"poses": None}, {"inl": None},
                 {"rms": None}, {"st": None}, {"B": 0}, {"B": B + 1}, {"F": 0, "fidx": p(fidx)}, {"F": B + 1, "fidx": p(fidx)},
                 {"F": B - 1}, {"n_iter": 0}, {"md": 0.0}, {"md": -0.01}, {"md": float("nan")}, {"md": float("inf")},
                 {"mp": 5}, {"K9": None}, {"Kf": p(Kf)}, {"K9": farr(nonpinhole.reshape(9), 9)},
                 {"K9": farr([float("nan")] + list(K.reshape(9)[1:]), 9)}):
        a = dict(base, **over)
        assert lib.dim_icp(*a.values()) == 2, over
        if over != {"ctx": None}:
            assert b"dim_icp" in lib.dim_last_error(), over
        torch.cuda.synchronize()
        assert (outs[0] == -7.0).all() and (outs[1] == -7).all() and (outs[2] == -7.0).all() and (outs[3] == -7).all(), over
    assert lib.dim_icp(*base.values()) == 0
    torch.cuda.synchronize()
    assert (outs[3] != -7).all()


def test_context_icp_equals_the_c_entry(ctx, case, run):
    outs = [torch.empty((N_ITER, B, 3, 4), dtype=torch.float64, device=DEV), torch.empty((N_ITER, B), dtype=torch.int32, device=DEV),
            torch.empty((N_ITER, B), device=DEV), torch.empty((N_ITER, B), dtype=torch.int32, device=DEV)]
    depth, cls, P0 = dev(case["depth"]), dev(case["cls"]), dev(case["P0"])
    p = lambda t: C.c_void_p(t.data_ptr())
    assert lib.dim_icp(ctx._h, p(depth), B, None, farr(K.reshape(9), 9), None, p(cls), p(P0), B, N_ITER, 0.25, 6.0, 0.02, 64,
                       *[p(t) for t in outs], None) == 0
    torch.cuda.synchronize()
    for k, t in zip(KEYS, outs):
        assert np.array_equal(t.cpu().numpy(), run[k]), k


def test_pose_refiner_icp_equals_context_icp_per_batch(ctx, meshes):
    """37 instances over 11 frames from 3 cameras, u16 depth converted on the device"""
    counts = [4, 3, 5, 2, 4, 3, 5, 3, 4, 2, 2]
    s = frames_scene(meshes, counts, 9)
    n = len(s["cls"])
    assert n == 37
    ref = PoseRefiner(meshes, synth.make_weights(0), max_batch=B, n_iter=2)
    got = ref.icp(s["u16"], s["cls"], s["P0"], K_frames=s["Kf"], frame_of=s["frame_of"], n_iter=4)
    ref.close()
    batches = plan_frame_batches(s["frame_of"], 11, B, 0, n, s["Kf"])
    assert len(batches) == 3
    for a, b, frames, local, Kb in batches:
        r = ctx.icp(dev(s["depth"][frames]), dev(s["cls"][a:b]), dev(s["P0"][a:b]), Kb, 4, frame_idx=dev(local))
        for k in KEYS:
            assert np.array_equal(r[k].cpu().numpy(), got[k][:, a:b]), (a, k)
    assert (got["status"] == 0).all()
    assert np.array_equal(ctx.depth_from_u16(dev(s["u16"])).cpu().numpy(), s["depth"])


def test_refinement_graphs_replay_unchanged_after_icp(meshes, case):
    """graphs of the unlit, lit and RGB-D chains captured before a dim_icp call replay to the same bits after it"""
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
                c.icp(dev(case["depth"]), dev(case["cls"]), dev(case["P0"]), K, 3)
                out = c.refine(img, clsd, inid, K, n_iter, pixel_means_rgb=synth.PIXEL_MEANS_RGB, out=out, **ch)
            side.synchronize()
            assert graphs >= 1 and lib.dim_debug_graph_count(c._h) == graphs
            for k in want:
                assert torch.equal(out[k], want[k]), (kw, list(ch), k)
        c.close()


def test_evaluate_with_icp(tmp_path):
    classes, _ = lm6d_fixture.build(str(tmp_path), n_per_class=2)
    ds = lm6d_io.LM6DRefine(str(tmp_path), classes, "val")
    w = synth.make_weights(0)
    base = lm6d_io.evaluate(ds, w, K, n_iter=2, max_batch=3)
    zero = lm6d_io.evaluate(ds, w, K, n_iter=2, max_batch=3, icp_iters=0)
    assert np.array_equal(base[1], zero[1]) and repr(base[0]) == repr(zero[0])
    res, poses, gt = lm6d_io.evaluate(ds, w, K, n_iter=2, max_batch=3, icp_iters=5)
    assert poses.shape == (3, 4, 3, 4) and np.array_equal(poses[:2], base[1])
    meshes = [ds.mesh(c) for c in classes]
    ref = PoseRefiner(meshes, w, K=K, max_batch=3, n_iter=2)
    pairs = [(ci, p) for ci, c in enumerate(classes) for p in ds.pairs(c)]
    cls = np.array([ci for ci, _ in pairs], np.int32)
    init = np.stack([ds.load_pair(classes[ci], p)["pose_rendered"] for ci, p in pairs])
    imgs = np.stack([ds.load_pair(classes[ci], p)["image_observed"] for ci, p in pairs])
    u16 = np.stack([lm6d_io.read_depth_u16(str(tmp_path / "data" / "observed" / (p[0] + "-depth.png"))) for _, p in pairs])
    refined = ref.refine(imgs, cls, init)
    polished = ref.icp(u16, cls, refined[-1], n_iter=5)["poses"][-1]
    want = np.concatenate([refined, polished[None]])
    assert np.array_equal(poses, want)
    pts = [ds.points(c) for c in classes]
    exp = pose_eval.evaluate_pose_add(ref.ctx, want, gt, cls, pts, [ds.diameters[c] for c in classes],
                                      [c == "glue" for c in classes])
    ref.close()
    assert repr(exp["mean"]) == repr(res["mean"])
