"""GPU: BOP 2019's pose errors -- MSSD / MSPD over a symmetry set (dim_pose_error_sym, Context.pose_error_sym,
PoseRefiner.pose_error_sym), the BOP 2019 VSD (dim_pose_error_vsd_ex) and lm6d_io.evaluate(bop=True) -- held bit for bit to
the oracle (oracle/bop.py) and to their own reference calls.

MSSD / MSPD: M = 16 estimates 0.5-4 cm / 5-40 deg from their ground truth, three cameras, a point set of 3 000 points and one
of 30 000, and S = 1 (identity), 2 (identity and a half-turn about z) and 630 (a continuous symmetry about z through an
offset, combined with the half-turn).  Instance 3's estimate is behind the camera (MSPD = inf).
VSD: test_gpu_vsd's B = 16 scene (holes, an occluder, an object cut by the border, an estimate out of view, a bad class)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

import json  # noqa: E402

import lm6d_fixture  # noqa: E402
from test_gpu_vsd import CAMS, context, dev, frames_scene, scene  # noqa: E402
from test_icp_oracle import perturb  # noqa: E402
from oracle import bop as OB  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle import vsd as V  # noqa: E402
from deepim_b200 import bop, lighting, lm6d_io, pose_eval, synth  # noqa: E402
from deepim_b200._capi import farr, lib  # noqa: E402
from deepim_b200.context import launch_count  # noqa: E402
from deepim_b200.refiner import PoseRefiner, plan_frame_batches  # noqa: E402

DEV = torch.device("cuda", 0)
K = synth.K_LINEMOD
M = 16
DELTA = pose_eval.BOP19_VSD_DELTA
TAUS = pose_eval.BOP19_VSD_TAUS
DIAM = np.array([0.11, 0.17])  # per class, metres
FLIP_Z = np.diag([-1.0, -1.0, 1.0, 1.0])


def p(t):
    return C.c_void_p(t.data_ptr())


def sym_sets():
    cont = {"axis": np.array([0.0, 0.0, 1.0]), "offset": np.array([0.002, -0.001, 0.0])}
    full = bop.symmetry_transforms({"symmetries_discrete": [FLIP_Z], "symmetries_continuous": [cont]})
    assert full.shape == (630, 3, 4)
    return {1: np.eye(3, 4)[None], 2: bop.symmetry_transforms({"symmetries_discrete": [FLIP_Z]}), 630: full}


SYMS = sym_sets()


@pytest.fixture(scope="module")
def sym_case():
    rng = np.random.default_rng(12)
    gt = synth.sample_pose_pairs(M, 4)[0]
    est = np.stack([perturb(g, rng, t=rng.uniform(0.005, 0.04), deg=rng.uniform(5.0, 40.0)) for g in gt])
    est[3, 2, 3] = -0.5  # behind the camera
    Ks = CAMS[np.arange(M) % 3].astype(np.float64)
    pts = {3000: rng.uniform(-0.05, 0.05, (3000, 3)), 30000: rng.normal(0.0, 0.03, (30011, 3))}
    return dict(gt=gt, est=est, K=Ks, pts=pts)


@pytest.fixture(scope="module")
def ctx(meshes):
    c = context(meshes)
    yield c
    c.close()


@pytest.fixture(scope="module")
def meshes():
    ms = [synth.make_blob(), synth.make_linemod_like_set()[4]]
    for m in ms:
        m.normals = synth.vertex_normals(m)
    return ms


def sym_call(ctx, s, n, S, sel=None):
    sel = np.arange(M) if sel is None else sel
    r = ctx.pose_error_sym(dev(s["est"][sel]), dev(s["gt"][sel]), s["pts"][n], SYMS[S], s["K"][sel])
    return {k: v.cpu().numpy() for k, v in r.items()}


@pytest.fixture(scope="module")
def sym_runs(ctx, sym_case):
    return {(n, S): sym_call(ctx, sym_case, n, S) for n in (3000, 30000) for S in (1, 2, 630)}


@pytest.mark.parametrize("n", [3000, 30000])
@pytest.mark.parametrize("S", [1, 2, 630])
def test_mssd_mspd_equal_the_oracle(sym_runs, sym_case, n, S):
    err, idx = OB.mssd_mspd(sym_case["est"], sym_case["gt"], sym_case["pts"][n], SYMS[S], sym_case["K"])
    got = sym_runs[(n, S)]
    assert np.array_equal(got["err"], err) and np.array_equal(got["sym_idx"], idx)
    assert np.isinf(err[3, 1]) and np.isfinite(np.delete(err, 3, 0)).all() and np.isfinite(err[:, 0]).all()
    if S > 1:
        assert (got["err"] <= sym_runs[(n, 1)]["err"]).all()
    if S == 630:
        assert (got["sym_idx"] > 0).any()


def test_mssd_mspd_independent_of_batch_sms_and_runs(ctx, sym_case, sym_runs):
    for n in (3000, 30000):
        for S in (2, 630):
            want = sym_runs[(n, S)]
            for m in (0, 3, 15):
                one = sym_call(ctx, sym_case, n, S, sel=np.array([m]))
                for k in want:
                    assert np.array_equal(one[k], want[k][m:m + 1]), (n, S, m, k)
            assert all(np.array_equal(sym_call(ctx, sym_case, n, S)[k], want[k]) for k in want)
            for sms in (1, 114):
                assert lib.dim_debug_set_option(ctx._h, b"sms", sms) == 0
                r = sym_call(ctx, sym_case, n, S)
                assert lib.dim_debug_set_option(ctx._h, b"sms", 0) == 0
                for k in want:
                    assert np.array_equal(r[k], want[k]), (n, S, sms, k)


def test_sym_context_equals_the_c_entry_and_batches_past_max_batch(ctx, sym_case, sym_runs):
    s = sym_case
    pts, sy = dev(s["pts"][3000]), dev(SYMS[630])
    err = torch.empty((M, 2), dtype=torch.float64, device=DEV)
    idx = torch.empty((M, 2), dtype=torch.int32, device=DEV)
    assert lib.dim_pose_error_sym(ctx._h, p(dev(s["est"])), p(dev(s["gt"])), M, p(pts), 3000, p(sy), 630,
                                  p(dev(s["K"].reshape(M, 9))), p(err), p(idx), None) == 0
    torch.cuda.synchronize()
    want = sym_runs[(3000, 630)]
    assert np.array_equal(err.cpu().numpy(), want["err"]) and np.array_equal(idx.cpu().numpy(), want["sym_idx"])
    # one K broadcast, and 40 instances (three calls of at most 16)
    r = ctx.pose_error_sym(dev(s["est"][:5]), dev(s["gt"][:5]), s["pts"][3000], SYMS[2], K)
    e, i = OB.mssd_mspd(s["est"][:5], s["gt"][:5], s["pts"][3000], SYMS[2], K)
    assert np.array_equal(r["err"].cpu().numpy(), e) and np.array_equal(r["sym_idx"].cpu().numpy(), i)
    big = np.r_[np.arange(M), np.arange(M), np.arange(8)]
    r = sym_call(ctx, s, 3000, 630, sel=big)
    assert np.array_equal(r["err"], want["err"][big]) and np.array_equal(r["sym_idx"], want["sym_idx"][big])


def test_sym_refusals_leave_outputs_untouched(ctx, sym_case):
    s = sym_case
    est, gt, pts, sy, Kd = dev(s["est"]), dev(s["gt"]), dev(s["pts"][3000]), dev(SYMS[630]), dev(s["K"].reshape(M, 9))
    big = dev(np.tile(SYMS[630], (7, 1, 1)))  # 4410 symmetries
    err = torch.full((M, 2), -7.0, dtype=torch.float64, device=DEV)
    idx = torch.full((M, 2), -7, dtype=torch.int32, device=DEV)
    base = dict(ctx=ctx._h, est=p(est), gt=p(gt), M=M, pts=p(pts), N=3000, syms=p(sy), S=630, K=p(Kd), err=p(err), idx=p(idx),
                stream=None)
    n0 = launch_count()
    for over in ({"ctx": None}, {"est": None}, {"gt": None}, {"pts": None}, {"syms": None}, {"K": None}, {"err": None},
                 {"M": 0}, {"M": M + 1}, {"N": 0}, {"S": 0}, {"S": 4097, "syms": p(big)}):
        assert lib.dim_pose_error_sym(*dict(base, **over).values()) == 2, over
        if over != {"ctx": None}:
            assert b"dim_pose_error_sym" in lib.dim_last_error(), over
        torch.cuda.synchronize()
        assert (err == -7.0).all() and (idx == -7).all(), over
    assert launch_count() == n0
    assert lib.dim_pose_error_sym(*dict(base, idx=None).values()) == 0  # sym_idx2 is optional
    torch.cuda.synchronize()
    assert (err != -7.0).all() and (idx == -7).all()
    assert lib.dim_pose_error_sym(*dict(base, S=4096, syms=p(big)).values()) == 0


def test_pose_refiner_sym_equals_context_per_batch(ctx, meshes, sym_case):
    """37 instances of two classes (interleaved), per-instance cameras"""
    rng = np.random.default_rng(4)
    s = sym_case
    n = 37
    pick = rng.integers(0, M, n)
    cls = (np.arange(n) % 3 == 0).astype(np.int32)
    pts = [s["pts"][3000], s["pts"][30000][:5000]]
    syms = [SYMS[630], SYMS[2]]
    ref = PoseRefiner(meshes, synth.make_weights(0), max_batch=M, n_iter=1)
    got = ref.pose_error_sym(cls, s["est"][pick], s["gt"][pick], pts, syms, s["K"][pick])
    ref.close()
    for c in (0, 1):
        sel = np.nonzero(cls == c)[0]
        for a in range(0, len(sel), M):
            b = sel[a:a + M]
            r = ctx.pose_error_sym(dev(s["est"][pick[b]]), dev(s["gt"][pick[b]]), pts[c], syms[c], s["K"][pick[b]])
            assert np.array_equal(r["err"].cpu().numpy(), got["err"][b]) and np.array_equal(r["sym_idx"].cpu().numpy(),
                                                                                           got["sym_idx"][b])


# ------------------------------------------------------------------------------------------------ BOP 2019 VSD
@pytest.fixture(scope="module")
def case(meshes):
    return scene(meshes)


def diam_of(cls):
    return np.where(cls < 2, DIAM[np.minimum(cls, 1)], 0.05)


def vsd_call(ctx, s, sel=None, frame_map=True, **kw):
    sel = np.arange(len(s["cls"])) if sel is None else sel
    kw.setdefault("visib_mode", "bop19")
    kw.setdefault("diameters", diam_of(s["cls"][sel]))
    if frame_map:
        args = (dev(s["depth"]), dev(s["cls"][sel]), dev(s["est"][sel]), dev(s["gt"][sel]), s["Kf"])
        kw.setdefault("frame_idx", dev(s["frame_of"][sel]))
    else:
        f = s["frame_of"][sel]
        args = (dev(s["depth"][f]), dev(s["cls"][sel]), dev(s["est"][sel]), dev(s["gt"][sel]), s["Kf"][f])
    r = ctx.pose_error_vsd(*args, DELTA, TAUS, **kw)
    return {k: v.cpu().numpy() for k, v in r.items()}


@pytest.fixture(scope="module")
def run(ctx, case):
    return vsd_call(ctx, case)


@pytest.fixture(scope="module")
def oracle_vsd(case, meshes):
    """the oracle's errors and status with BOP 2019 visibility and relative taus, and with each switch alone"""
    f = lambda **kw: OB.vsd(meshes, case["cls"], case["est"], case["gt"], case["depth"], case["Kf"], DELTA, TAUS,
                           frame_idx=case["frame_of"], **kw)
    return {"bop19": f(visib_mode="bop19", diameters=diam_of(case["cls"])), "sixd17_rel": f(visib_mode="sixd17", diameters=diam_of(case["cls"])),
            "bop19_abs": f(visib_mode="bop19")}


def test_bop19_vsd_equals_the_oracle(run, oracle_vsd):
    err, st = oracle_vsd["bop19"]
    assert np.array_equal(run["err"], err) and np.array_equal(run["status"], st)
    assert st[14] == 3 and (run["err"][13] == 1.0).all() and (np.diff(run["err"], axis=1) <= 0).all()
    assert not np.array_equal(oracle_vsd["sixd17_rel"][0], err) and not np.array_equal(oracle_vsd["bop19_abs"][0], err)


def test_each_vsd_switch_alone_equals_the_oracle(ctx, case, oracle_vsd):
    assert np.array_equal(vsd_call(ctx, case, visib_mode="sixd17")["err"], oracle_vsd["sixd17_rel"][0])
    assert np.array_equal(vsd_call(ctx, case, diameters=None)["err"], oracle_vsd["bop19_abs"][0])


def test_mode0_without_diameters_is_dim_pose_error_vsd(ctx, case):
    depth, fidx, cls = dev(case["depth"]), dev(case["frame_of"]), dev(case["cls"])
    est, gt, Kf = dev(case["est"]), dev(case["gt"]), dev(case["Kf"])
    taus = farr(TAUS, ctype=C.c_double)
    outs = []
    for ex in (False, True):
        err = torch.full((16, 10), -7.0, dtype=torch.float64, device=DEV)
        st = torch.full((16,), -7, dtype=torch.int32, device=DEV)
        torch.cuda.synchronize()
        launch_count(True)
        args = (ctx._h, p(depth), 6, p(fidx), None, p(Kf), p(cls), p(est), p(gt), 16, 0.25, 6.0, DELTA, taus, 10)
        if ex:
            assert lib.dim_pose_error_vsd_ex(*args, 0, None, p(err), p(st), None) == 0
        else:
            assert lib.dim_pose_error_vsd(*args, p(err), p(st), None) == 0
        torch.cuda.synchronize()
        outs.append((launch_count(), err.cpu().numpy(), st.cpu().numpy()))
    assert outs[0][0] == outs[1][0] > 0
    assert np.array_equal(outs[0][1], outs[1][1]) and np.array_equal(outs[0][2], outs[1][2])
    r = vsd_call(ctx, case, visib_mode="sixd17", diameters=None)  # Context's default path
    assert np.array_equal(r["err"], outs[0][1])


def test_bop19_cameras_frame_map_and_batch_sizes_equal_their_reference_calls(ctx, case, run):
    cam_of = case["frame_of"] % 3
    d = diam_of(case["cls"])
    for cam in range(3):
        sel = np.nonzero(cam_of == cam)[0]
        f = case["frame_of"][sel]
        r = ctx.pose_error_vsd(dev(case["depth"][f]), dev(case["cls"][sel]), dev(case["est"][sel]), dev(case["gt"][sel]),
                               CAMS[cam], DELTA, TAUS, visib_mode="bop19", diameters=d[sel])
        for k in run:
            assert np.array_equal(r[k].cpu().numpy(), run[k][sel]), (cam, k)
    gathered = vsd_call(ctx, case, frame_map=False)
    for k in run:
        assert np.array_equal(gathered[k], run[k]), k
    for b in (0, 5, 13, 15):
        one = vsd_call(ctx, case, sel=np.array([b]), frame_map=False)
        for k in run:
            assert np.array_equal(one[k], run[k][b:b + 1]), (b, k)


def test_vsd_ex_refusals_leave_outputs_untouched(ctx, case):
    depth, cls, est, gt = dev(case["depth"][case["frame_of"]]), dev(case["cls"]), dev(case["est"]), dev(case["gt"])
    err = torch.full((16, 10), -7.0, dtype=torch.float64, device=DEV)
    st = torch.full((16,), -7, dtype=torch.int32, device=DEV)
    d = np.ascontiguousarray(diam_of(case["cls"]))
    dptr = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    keep = []

    def with_diam(v):
        a = d.copy()
        a[7] = v
        keep.append(a)
        return dptr(a)

    base = dict(ctx=ctx._h, depth=p(depth), F=16, fidx=None, K9=farr(K.reshape(9), 9), Kf=None, cls=p(cls), est=p(est),
                gt=p(gt), B=16, zn=0.25, zf=6.0, delta=DELTA, taus=farr(TAUS, ctype=C.c_double), n_tau=10, mode=1,
                diam=dptr(d), err=p(err), st=p(st), stream=None)
    n0 = launch_count()
    for over in ({"mode": 2}, {"mode": -1}, {"diam": with_diam(0.0)}, {"diam": with_diam(-0.1)},
                 {"diam": with_diam(float("nan"))}, {"diam": with_diam(float("inf"))}, {"n_tau": 17}, {"B": 17},
                 {"err": None}, {"K9": None}):
        assert lib.dim_pose_error_vsd_ex(*dict(base, **over).values()) == 2, over
        assert b"dim_pose_error_vsd_ex" in lib.dim_last_error(), over
        torch.cuda.synchronize()
        assert (err == -7.0).all() and (st == -7).all(), over
    assert launch_count() == n0
    assert lib.dim_pose_error_vsd_ex(*base.values()) == 0
    torch.cuda.synchronize()
    assert (err != -7.0).all() and (st != -7).all()
    with pytest.raises(ValueError):
        vsd_call(ctx, case, visib_mode="bop20")
    with pytest.raises(ValueError):
        vsd_call(ctx, case, diameters=d[:5])


def test_pose_refiner_bop19_vsd_equals_context_per_batch(ctx, meshes):
    counts = [4, 3, 5, 2, 4, 3, 5, 3, 4, 2, 2]
    s = frames_scene(meshes, counts, 9)
    n = len(s["cls"])
    d = diam_of(s["cls"])
    ref = PoseRefiner(meshes, synth.make_weights(0), max_batch=16, n_iter=2)
    got = ref.vsd(s["u16"], s["cls"], s["est"], s["gt"], K_frames=s["Kf"], frame_of=s["frame_of"], delta=DELTA, taus=TAUS,
                  visib_mode="bop19", diameters=d)
    ref.close()
    for a, b, frames, local, Kb in plan_frame_batches(s["frame_of"], 11, 16, 0, n, s["Kf"]):
        r = ctx.pose_error_vsd(dev(s["depth"][frames]), dev(s["cls"][a:b]), dev(s["est"][a:b]), dev(s["gt"][a:b]), Kb, DELTA,
                               TAUS, frame_idx=dev(local), visib_mode="bop19", diameters=d[a:b])
        for k in got:
            assert np.array_equal(r[k].cpu().numpy(), got[k][a:b]), (a, k)


def test_refinement_graphs_replay_unchanged_after_bop_calls(meshes, case, sym_case):
    """graphs of the unlit, lit and RGB-D chains captured before a BOP 2019 VSD and an MSSD / MSPD call replay to the same
    bits after them"""
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
                vsd_call(c, case)
                sym_call(c, sym_case, 3000, 630)
                out = c.refine(img, clsd, inid, K, n_iter, pixel_means_rgb=synth.PIXEL_MEANS_RGB, out=out, **ch)
            side.synchronize()
            assert graphs >= 1 and lib.dim_debug_graph_count(c._h) == graphs
            for k in want:
                assert torch.equal(out[k], want[k]), (kw, list(ch), k)
        c.close()


# ------------------------------------------------------------------------------------------------ evaluate(bop=True)
def test_evaluate_with_bop(tmp_path):
    classes, _ = lm6d_fixture.build(str(tmp_path), n_per_class=2)
    ds = lm6d_io.LM6DRefine(str(tmp_path), classes, "val")
    info = {str(i + 1): {"diameter": 1000.0 * ds.diameters[c]} for i, c in enumerate(classes)}
    info["1"]["symmetries_discrete"] = [FLIP_Z.reshape(-1).tolist()]
    info["2"]["symmetries_continuous"] = [{"axis": [0, 0, 1], "offset": [0, 0, 0]}]
    js = tmp_path / "models_info.json"
    js.write_text(json.dumps(info))
    w = synth.make_weights(0)
    base = lm6d_io.evaluate(ds, w, K, n_iter=2, max_batch=3, icp_iters=2)
    off = lm6d_io.evaluate(ds, w, K, n_iter=2, max_batch=3, icp_iters=2, bop=False)
    assert np.array_equal(base[1], off[1]) and repr(base[0]) == repr(off[0]) and "bop" not in base[0]
    res, poses, gt = lm6d_io.evaluate(ds, w, K, n_iter=2, max_batch=3, icp_iters=2, bop=True, models_info_json=str(js))
    assert np.array_equal(poses, base[1]) and poses.shape[0] == 3
    assert repr({k: v for k, v in res.items() if k != "bop"}) == repr(base[0])
    meshes = [ds.mesh(c) for c in classes]
    ref = PoseRefiner(meshes, w, K=K, max_batch=3, n_iter=2)
    pairs = [(ci, p_) for ci, c in enumerate(classes) for p_ in ds.pairs(c)]
    cls = np.array([ci for ci, _ in pairs], np.int32)
    u16 = np.stack([lm6d_io.read_depth_u16(str(tmp_path / "data" / "observed" / (q[0] + "-depth.png"))) for _, q in pairs])
    diam = np.array([ds.diameters[c] for c in classes])
    syms = [bop.symmetry_transforms(bop.load_models_info_json(str(js))[i + 1]) for i in range(len(classes))]
    assert [len(s_) for s_ in syms][:2] == [2, 315]
    pts = [ds.points(c) for c in classes]
    vsd = np.stack([ref.vsd(u16, cls, q, gt, delta=DELTA, taus=TAUS, visib_mode="bop19", diameters=diam[cls])["err"]
                    for q in poses])
    e = np.stack([ref.pose_error_sym(cls, q, gt, pts, syms)["err"] for q in poses])
    ref.close()
    errs = res["bop"]["errors"]
    assert np.array_equal(errs["vsd"], vsd) and np.array_equal(errs["mssd"], e[..., 0]) and np.array_equal(errs["mspd"], e[..., 1])
    exp = pose_eval.evaluate_bop19(vsd, e[..., 0], e[..., 1], cls, len(classes), diam, 640)
    assert repr(exp["mean"]) == repr(res["bop"]["mean"]) and repr(exp["classes"]) == repr(res["bop"]["classes"])
    assert len(res["bop"]["mean"]["AR"]) == 3
    plain = lm6d_io.evaluate(ds, w, K, n_iter=2, max_batch=3, icp_iters=2, bop=True)  # no JSON: the identity only
    ref = PoseRefiner(meshes, w, K=K, max_batch=3, n_iter=2)
    e1 = np.stack([ref.pose_error_sym(cls, q, gt, pts, [np.eye(3, 4)[None]] * len(classes))["err"] for q in plain[1]])
    ref.close()
    assert np.array_equal(plain[0]["bop"]["errors"]["mssd"], e1[..., 0])
    assert np.array_equal(plain[0]["bop"]["errors"]["vsd"], vsd)
