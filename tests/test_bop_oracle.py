"""CPU: BOP 2019 pieces on the host -- the symmetry transforms and models_info.json reader (deepim_b200.bop), the MSSD /
MSPD contract and the BOP 2019 VSD (oracle/bop.py), its visibility against the reference's masks
(tests/golden/ref_vsd.npz), the average recall (pose_eval.evaluate_bop19), the results CSV and the C prototypes."""
import json
import os

import numpy as np
import pytest

from deepim_b200 import bop, pose_eval, synth
from oracle import bop as OB
from oracle import vsd as V

K = synth.K_LINEMOD.astype(np.float64)
FLIP_Z = np.array([[-1.0, 0, 0, 0], [0, -1.0, 0, 0], [0, 0, 1.0, 0], [0, 0, 0, 1.0]])


def info(disc=(), cont=()):
    return {"syms": {"symmetries_discrete": [np.asarray(T, np.float64) for T in disc], "symmetries_continuous": list(cont)}}


def test_symmetry_counts():
    assert np.array_equal(bop.symmetry_transforms(info()), np.eye(3, 4)[None])
    axis = {"axis": np.array([0.0, 0.0, 1.0]), "offset": np.zeros(3)}
    one = bop.symmetry_transforms(info(cont=[axis]))
    assert one.shape == (315, 3, 4) and np.array_equal(one[0], np.eye(3, 4))
    D = [FLIP_Z, np.diag([1.0, -1.0, -1.0, 1.0])]
    both = bop.symmetry_transforms(info(disc=D, cont=[axis]))
    assert both.shape == ((len(D) + 1) * 315, 3, 4) and np.array_equal(both[0], np.eye(3, 4))
    assert bop.symmetry_transforms(info(disc=D)).shape == (3, 3, 4)
    assert bop.symmetry_transforms(info(cont=[axis]), max_sym_disc_step=0.1).shape == (32, 3, 4)


def test_symmetries_are_rigid_and_fix_their_axis():
    axis, off = np.array([0.3, -0.5, 0.8]), np.array([0.01, -0.02, 0.005])
    T = bop.symmetry_transforms(info(disc=[FLIP_Z], cont=[{"axis": axis, "offset": off}]))
    R = T[:, :, :3]
    assert np.abs(R @ R.transpose(0, 2, 1) - np.eye(3)).max() < 1e-14
    assert np.abs(np.linalg.det(R) - 1.0).max() < 1e-14
    cont = T[:315]  # the continuous ones combined with the identity
    a = axis / np.linalg.norm(axis)
    for lam in (-0.1, 0.0, 0.07):
        p = off + lam * a
        assert np.abs(cont[:, :, :3] @ p + cont[:, :, 3] - p).max() < 1e-14
    ang = np.degrees(np.arccos(np.clip((np.trace(cont[:, :, :3], axis1=1, axis2=2) - 1) / 2, -1, 1)))
    assert ang[1] == pytest.approx(360.0 / 315, abs=1e-9) and len(np.unique(np.round(ang, 6))) == 158


def test_models_info_json_is_converted_to_metres(tmp_path):
    T = np.eye(4)
    T[:3, 3] = [10.0, -20.0, 5.0]
    path = tmp_path / "models_info.json"
    path.write_text(json.dumps({"1": {"diameter": 102.1, "min_x": -37.9},
                                "10": {"diameter": 164.6, "symmetries_discrete": [T.reshape(-1).tolist()],
                                       "symmetries_continuous": [{"axis": [0, 0, 1], "offset": [0, 0, 12.0]}]}}))
    m = bop.load_models_info_json(str(path))
    assert set(m) == {1, 10} and m[1]["diameter"] == pytest.approx(0.1021) and m[10]["diameter"] == pytest.approx(0.1646)
    assert bop.symmetry_transforms(m[1]).shape == (1, 3, 4)
    d = m[10]["syms"]["symmetries_discrete"][0]
    assert np.allclose(d[:3, 3], [0.01, -0.02, 0.005]) and np.array_equal(d[:3, :3], np.eye(3))
    assert np.allclose(m[10]["syms"]["symmetries_continuous"][0]["offset"], [0, 0, 0.012])
    assert bop.symmetry_transforms(m[10]).shape == (630, 3, 4)


@pytest.fixture(scope="module")
def pose_set():
    rng = np.random.default_rng(11)
    pts = rng.uniform(-0.05, 0.05, (500, 3))
    gt = synth.sample_pose_pairs(6, 5)[0]
    from test_icp_oracle import perturb
    est = np.stack([perturb(g, rng, t=0.01, deg=8.0) for g in gt])
    return pts, est, gt


def test_identity_only_mssd_bounds_add(pose_set):
    pts, est, gt = pose_set
    err, idx = OB.mssd_mspd(est, gt, pts, np.eye(3, 4)[None], K)
    add = [np.linalg.norm((pts @ e[:, :3].T + e[:, 3]) - (pts @ g[:, :3].T + g[:, 3]), axis=1).mean() for e, g in zip(est, gt)]
    assert (err[:, 0] >= np.array(add)).all() and (idx == 0).all() and np.isfinite(err).all()


def test_more_symmetries_never_raise_the_errors(pose_set):
    pts, est, gt = pose_set
    axis = {"axis": np.array([0.0, 1.0, 0.0]), "offset": np.zeros(3)}
    full = bop.symmetry_transforms(info(disc=[FLIP_Z], cont=[axis]), max_sym_disc_step=0.2)
    prev = None
    for S in (1, 2, 17, len(full)):
        err, idx = OB.mssd_mspd(est, gt, pts, full[:S], K)
        assert (idx < S).all()
        if prev is not None:
            assert (err <= prev).all()
        prev = err


def test_exact_symmetry_gives_zero_mssd():
    """a point set closed under a half-turn about z through an offset: est = gt . sym scores 0 at that symmetry"""
    rng = np.random.default_rng(2)
    c = np.array([0.004, -0.003, 0.0])
    half = rng.uniform(-0.04, 0.04, (300, 3))
    sym = np.eye(3, 4)
    sym[:2, :2] = -np.eye(2)
    sym[:, 3] = -sym[:, :3] @ c + c
    pts = np.concatenate([half, half @ sym[:, :3].T + sym[:, 3]])
    gt = synth.sample_pose_pairs(4, 8)[0]
    est = gt.copy()
    est[:, :, :3] = gt[:, :, :3] @ sym[:, :3]
    est[:, :, 3] = np.einsum("mij,j->mi", gt[:, :, :3], sym[:, 3]) + gt[:, :, 3]
    err, idx = OB.mssd_mspd(est, gt, pts, np.stack([np.eye(3, 4), sym]), K)
    assert (err[:, 0] <= 1e-12).all() and (idx[:, 0] == 1).all() and (err[:, 1] <= 1e-6).all()
    err1, _ = OB.mssd_mspd(est, gt, pts, np.eye(3, 4)[None], K)
    assert (err1[:, 0] > 0.01).all()


def test_points_behind_the_camera_make_mspd_infinite(pose_set):
    pts, est, gt = pose_set
    behind = est[:2].copy()
    behind[:, 2, 3] = 0.01  # the model straddles Z = 0
    err, idx = OB.mssd_mspd(behind, gt[:2], pts, bop.symmetry_transforms(info(disc=[FLIP_Z])), K)
    assert np.isinf(err[:, 1]).all() and (idx[:, 1] == 0).all() and np.isfinite(err[:, 0]).all()


def test_per_instance_cameras_equal_per_camera_calls(pose_set):
    pts, est, gt = pose_set
    K2 = K.copy()
    K2[0, 0], K2[1, 2] = 800.0, 250.0
    Ks = np.stack([K, K2] * 3)
    err, idx = OB.mssd_mspd(est, gt, pts, np.eye(3, 4)[None], Ks)
    for k, Kc in enumerate((K, K2)):
        e, i = OB.mssd_mspd(est[k::2], gt[k::2], pts, np.eye(3, 4)[None], Kc)
        assert np.array_equal(e, err[k::2]) and np.array_equal(i, idx[k::2])


@pytest.fixture(scope="module")
def ref_vsd(golden_dir):
    return np.load(os.path.join(golden_dir, "ref_vsd.npz"))


@pytest.mark.parametrize("case", [0, 1])
def test_bop19_masks_equal_the_reference_off_the_holes(ref_vsd, case):
    r = lambda k: ref_vsd["r%d_%s" % (case, k)]
    t, e, g = r("dist_test"), r("dist_est"), r("dist_gt")
    v_gt, v_est = OB.masks(t, e, g, 0.015, "bop19")
    seen = t > 0
    assert np.array_equal(v_gt[seen], r("visib_gt")[seen]) and np.array_equal(v_est[seen], r("visib_est")[seen])
    holes = (t == 0) & (g > 0)
    assert holes.sum() > 20 and v_gt[holes].all() and v_est[(t == 0) & (e > 0)].all()
    assert not v_gt[g == 0].any()


def test_bop19_vsd_with_diameters_scales_the_taus(ref_vsd):
    r = lambda k: ref_vsd["r0_%s" % k]
    t, e, g = r("dist_test"), r("dist_est"), r("dist_gt")
    d = 0.16
    rel, _ = OB.vsd_from_dist(t, e, g, 0.015, (0.05, 0.1, 0.25), "bop19", d)
    inter = np.logical_and(*OB.masks(t, e, g, 0.015, "bop19"))
    a = np.abs(g[inter] - e[inter]) / d
    n_u = int(np.count_nonzero(np.logical_or(*OB.masks(t, e, g, 0.015, "bop19"))))
    exp = [(np.count_nonzero(a >= tau) + n_u - inter.sum()) / n_u for tau in (0.05, 0.1, 0.25)]
    assert np.array_equal(rel, np.array(exp))
    with pytest.raises(ValueError):
        OB.visible(t, e, 0.015, "bop2020")


@pytest.mark.parametrize("case", [0, 1])
def test_sixd17_mode_without_diameters_is_the_vsd_oracle(ref_vsd, case):
    r = lambda k: ref_vsd["r%d_%s" % (case, k)]
    t, e, g = r("dist_test"), r("dist_est"), r("dist_gt")
    for a, b in zip(OB.masks(t, e, g, 0.015, "sixd17"), V.masks(t, e, g, 0.015)):
        assert np.array_equal(a, b)
    taus = (0.005, 0.01, 0.02, 0.05)
    got, want = OB.vsd_from_dist(t, e, g, 0.015, taus, "sixd17"), V.vsd_from_dist(t, e, g, 0.015, taus)
    assert np.array_equal(got[0], want[0]) and got[1] == want[1]


def test_bop19_vsd_scene_known_answers():
    """the full restatement: est = gt gives 0 also with a hole over half the object (BOP 2019 counts the hole as visible),
    and the SIXD 2017 mode without diameters equals oracle/vsd.py's vsd(), bad class included"""
    from oracle import oracle as O
    blob = synth.make_blob()
    G = synth.sample_pose_pairs(1, 3)[0][0]
    dep = O.render(blob, G, K, want=("depth",))["depth"]
    from test_icp_oracle import perturb
    E = perturb(G, np.random.default_rng(5), t=0.003, deg=2.0)
    holed = dep.copy()
    ys, xs = np.nonzero(dep)
    holed[ys.min():(ys.min() + ys.max()) // 2, :] = 0.0
    taus = (0.01, 0.02, 0.05)
    e, st = OB.vsd([blob], [0], G[None], G[None], holed[None], K, 0.015, taus, diameters=[0.1])
    assert st[0] == 0 and (e == 0.0).all()
    for d in (dep, holed):
        a = OB.vsd([blob], [0, 3], np.stack([E, E]), np.stack([G, G]), d[None], K, 0.015, taus, frame_idx=[0, 0],
                   visib_mode="sixd17")
        b = V.vsd([blob], [0, 3], np.stack([E, E]), np.stack([G, G]), d[None], K, 0.015, taus, frame_idx=[0, 0])
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    with pytest.raises(ValueError):
        OB.vsd([blob], [0], G[None], G[None], dep[None], K, visib_mode="bop20")


def test_evaluate_bop19_on_hand_built_errors():
    taus = pose_eval.BOP19_VSD_TAUS
    assert len(taus) == 10 and taus[0] == pytest.approx(0.05) and taus[-1] == pytest.approx(0.5)
    cls = np.array([0, 0, 1, 1])
    diam = np.array([0.1, 0.2])
    vsd = np.ones((2, 4, 10))
    vsd[0, 0] = 0.0                         # instance 0: below every threshold
    vsd[0, 1] = 0.22                        # instance 1: below the 6 thresholds 0.25 .. 0.5
    mssd = np.array([[0.0, 0.0151, 0.2, 1.0], [1.0, 1.0, 1.0, 1.0]])
    mspd = np.array([[4.0, 12.0, 60.0, np.inf], [np.inf] * 4])
    res = pose_eval.evaluate_bop19(vsd, mssd, mspd, cls, 2, diam, width=640)
    c0, c1 = res["classes"][0], res["classes"][1]
    assert c0["AR_VSD"] == pytest.approx([100 * (1 + 0.6) / 2, 0.0])
    # mssd 0.0151 against class 0's thresholds 0.005 .. 0.05 m: below 0.02 and up (7 of 10); class 1's errors (0.2, 1.0)
    # exceed all of its thresholds 0.01 .. 0.1 m
    assert c0["AR_MSSD"] == pytest.approx([100 * (1 + 0.7) / 2, 0.0]) and c1["AR_MSSD"] == [0.0, 0.0]
    assert c0["AR_MSPD"] == pytest.approx([100 * (1 + 0.8) / 2, 0.0]) and c1["AR_MSPD"] == [0.0, 0.0]
    assert c0["AR"][0] == pytest.approx((c0["AR_VSD"][0] + c0["AR_MSSD"][0] + c0["AR_MSPD"][0]) / 3)
    m = res["mean"]  # over all four instances
    assert m["AR_VSD"][0] == pytest.approx(100 * 1.6 / 4) and m["AR_MSPD"][0] == pytest.approx(100 * 1.8 / 4)
    half = pose_eval.evaluate_bop19(vsd, mssd, mspd, cls, 2, diam, width=320)  # thresholds 2.5 .. 25 px
    assert half["classes"][0]["AR_MSPD"][0] == pytest.approx(100 * (0.9 + 0.6) / 2)
    with pytest.raises(ValueError):
        pose_eval.evaluate_bop19(vsd[..., :4], mssd, mspd, cls, 2, diam)


def test_results_csv_round_trip(tmp_path):
    rng = np.random.default_rng(1)
    rows = []
    for k in range(5):
        R = synth.sample_pose_pairs(1, k)[0][0][:, :3]
        rows.append({"scene_id": k // 2, "im_id": 3 * k, "obj_id": 1 + k, "score": float(rng.uniform()), "R": R,
                     "t": rng.uniform(-0.2, 0.2, 3) + [0, 0, 0.8]})
    rows[2]["time"] = 0.0125
    path = tmp_path / "refiner_lm-test.csv"
    bop.write_results_csv(str(path), rows)
    lines = path.read_text().splitlines()
    assert lines[0] == "scene_id,im_id,obj_id,score,R,t,time" and len(lines) == 6
    assert len(lines[1].split(",")[4].split()) == 9 and lines[1].split(",")[-1] == "-1.0"
    back = bop.read_results_csv(str(path))
    for a, b in zip(rows, back):
        assert all(a[k] == b[k] for k in ("scene_id", "im_id", "obj_id", "score"))
        assert np.array_equal(np.asarray(a["R"]), b["R"]) and np.allclose(a["t"], b["t"], rtol=0, atol=1e-15)
        assert b["time"] == a.get("time", -1.0)
    assert float(lines[1].split(",")[5].split()[2]) == pytest.approx(rows[0]["t"][2] * 1000.0)
    bad = tmp_path / "bad.csv"
    bad.write_text("a,b\n")
    with pytest.raises(ValueError):
        bop.read_results_csv(str(bad))


def test_capi_declares_the_bop_entries():
    from deepim_b200 import _capi
    assert len(_capi.SIGNATURES["dim_pose_error_vsd_ex"][1]) == 20
    assert len(_capi.SIGNATURES["dim_pose_error_sym"][1]) == 12
