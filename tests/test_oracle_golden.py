"""CPU: pin the oracle against fixtures generated from the LIVE reference
(tests/golden/make_golden.py; RT_transform, calc_flow, pose_error, image.transform)."""
import os

import numpy as np
import pytest

from oracle import oracle as O
from deepim_b200 import synth


def test_se3_compose_and_delta_match_reference(golden_dir):
    g = np.load(os.path.join(golden_dir, "ref_se3.npz"))
    for coord in ("MODEL", "CAMERA", "CAMERA_NEW"):
        for k in range(len(g["pose_src"])):
            p = O.rt_transform(g["pose_src"][k], g["quat"][k], g["trans"][k], (0, 0, 0), (1, 1, 1), coord)
            np.testing.assert_allclose(p, g["pose_out_" + coord][k], rtol=0, atol=1e-14)
            p = O.rt_transform(g["pose_src"][k], g["quat"][k], g["trans"][k], g["T_means"], g["T_stds"], coord)
            np.testing.assert_allclose(p, g["pose_out_norm_" + coord][k], rtol=0, atol=1e-14)
            R, T = O.rt_delta(g["pose_src"][k], g["pose_out_norm_" + coord][k], g["T_means"], g["T_stds"], coord)
            np.testing.assert_allclose(R, g["R_delta_" + coord][k], rtol=0, atol=1e-14)
            np.testing.assert_allclose(T, g["T_delta_" + coord][k], rtol=0, atol=1e-13)


def test_rt_delta_inverts_rt_transform():
    # closed-form relation calc_RT_delta o RT_transform = id (SURVEY 4)
    rng = np.random.default_rng(0)
    obs, ini = synth.sample_pose_pairs(8, 3)
    for k in range(8):
        R, T = O.rt_delta(ini[k], obs[k], (0, 0, 0), (1, 1, 1), "camera")
        # rebuild quaternion from R (w>0 branch is enough for these small deltas)
        w = np.sqrt(max(0.0, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
        q = np.array([w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w)])
        back = O.rt_transform(ini[k], q, T, (0, 0, 0), (1, 1, 1), "camera")
        np.testing.assert_allclose(back, obs[k], atol=1e-12)


def test_quat2mat_doctest_vectors(golden_dir):
    # RT_transform.py:397-404 docstring examples, through rt_transform with identity source pose
    eye = np.hstack([np.eye(3), np.array([[0.0], [0.0], [1.0]])])
    p = O.rt_transform(eye, [0, 1.0, 0, 0], [0, 0, 0], (0, 0, 0), (1, 1, 1), "camera")
    np.testing.assert_allclose(p[:, :3], np.diag([1, -1, -1]), atol=1e-15)
    p = O.rt_transform(eye, [1.0, 0, 0, 0], [0, 0, 0], (0, 0, 0), (1, 1, 1), "camera")
    np.testing.assert_allclose(p[:, :3], np.eye(3), atol=1e-15)


def _kt_kinv(f):
    K = f["K"]
    Rs, ts, Rt, tt = f["pose_src"][:, :3], f["pose_src"][:, 3], f["pose_tgt"][:, :3], f["pose_tgt"][:, 3]
    T = np.zeros((3, 4))
    T[:, :3] = Rt @ Rs.T
    T[:, 3] = tt - T[:, :3] @ ts
    return (K @ T).astype(np.float32), np.linalg.inv(K).astype(np.float32)


def test_flow_matches_reference_calc_flow(golden_dir):
    # lib/flow_c/gpu_flow_kernel.cu restated in C vs lib/pair_matching/flow.py:calc_flow (its numpy twin)
    f = np.load(os.path.join(golden_dir, "ref_flow.npz"))
    KT, Kinv = _kt_kinv(f)
    fl, va = O.flow(f["depth_src"][None, None], f["depth_tgt"][None, None], KT[None], Kinv)
    vis = f["visible"]
    assert vis.sum() > 500
    # the two reference implementations differ only on borderline pixels (SURVEY a13): none here
    assert int((va[0, 0] != vis).sum()) == 0
    both = vis == 1
    ref = f["flow"].transpose(2, 0, 1)
    assert np.abs(fl[0][:, both] - ref[:, both]).max() < 5e-5
    assert np.all(fl[0][:, ~both] == 0)


def test_flow_matches_the_reference_cuda_kernel(golden_dir):
    """a13, second pin: the reference's UNMODIFIED lib/flow_c/gpu_flow_kernel.cu (compiled by oracle/build_ref.py into
    oracle/_ref, executed on a GPU by tests/golden/make_golden_flow_cuda.py -> ref_flow_cuda.npz) against the C restatement:
    the validity masks are identical; the flow differs by at most 2 ulp of the pixel coordinate (the reference build lets nvcc
    contract multiply-adds, the restatement is compiled without contraction so that the CUDA path can be bit-exact to IT)."""
    g = np.load(os.path.join(golden_dir, "ref_flow_cuda.npz"))
    f = np.load(os.path.join(golden_dir, "ref_flow.npz"))
    fl, va = O.flow(f["depth_src"][None, None], f["depth_tgt"][None, None], g["small_KT"], g["small_Kinv"])
    assert np.array_equal(va, g["small_valid"]) and g["small_valid"].sum() > 500
    assert np.abs(fl - g["small_flow"]).max() < 2e-5
    fl, va = O.flow(g["depth_src"], g["depth_tgt"], g["KT"], g["Kinv"])
    assert np.array_equal(va, g["valid"]) and g["valid"].sum() > 5000
    assert np.abs(fl - g["flow"]).max() < 2.5e-4 and np.abs(g["flow"]).max() > 10.0   # 2 ulp at coordinates of ~600 px
    assert np.all(fl[np.broadcast_to(va == 0, fl.shape)] == 0)


def test_add_adi_match_reference(golden_dir):
    pe = np.load(os.path.join(golden_dir, "ref_pose_error.npz"))
    assert abs(O.add_metric(pe["R_est"], pe["t_est"], pe["R_gt"], pe["t_gt"], pe["pts"]) - pe["add"]) < 1e-15
    assert abs(O.adi_metric(pe["R_est"], pe["t_est"], pe["R_gt"], pe["t_gt"], pe["pts"]) - pe["adi"]) < 1e-15


def test_image_transform_matches_reference(golden_dir):
    t = np.load(os.path.join(golden_dir, "ref_transform.npz"))
    out = synth.transform_image(t["im"])
    assert np.array_equal(out, t["out"][0])


def test_train_labels_match_reference(golden_dir):
    # calc_RT_delta(..., "QUAT") (mat2quat / eigh) and K . calc_se3 as used by batch_updater_py_multi.py:239-259
    g = np.load(os.path.join(golden_dir, "ref_se3.npz"))
    tgt32 = g["pose_out_CAMERA"].astype(np.float32)
    for k in range(len(g["pose_src"])):
        Rd, Td = O.rt_delta_f32tgt(g["pose_src"][k], tgt32[k], (0, 0, 0), (1, 1, 1), "camera")
        np.testing.assert_allclose(O.mat2quat(Rd), g["label_quat"][k], atol=1e-12)
        np.testing.assert_allclose(Td, g["label_trans"][k], atol=1e-12)
        KT = g["label_K"] @ O.calc_se3_f32(g["pose_src"][k], tgt32[k]).astype(np.float64)
        np.testing.assert_allclose(KT, g["label_KT"][k], rtol=0, atol=2e-4)  # float32 se3 storage, BLAS order


def test_rt_dist_and_arp_2d_against_reference_golden(golden_dir):
    """calc_rt_dist_m (RT_transform.py:162-173), re and arp_2d (pose_error.py:27-69, 127-132) of the live reference on 48
    pose pairs (0.5 / 4 / 30 degree perturbations, an exact 180 degree and an identity case): the inputs of the 5 cm 5 deg and
    Proj. 2D tables (LM6D_REFINE.evaluate_pose / evaluate_pose_arp_2d)."""
    g = np.load(os.path.join(golden_dir, "ref_pose_eval.npz"))
    for k in range(len(g["rot_deg"])):
        rd, td = O.rt_dist(g["poses_est"][k], g["poses_gt"][k])
        assert abs(rd - g["rot_deg"][k]) < 1e-9 and abs(rd - g["re_deg"][k]) < 1e-9
        assert abs(td - g["trans_m"][k]) < 1e-14
        assert abs(O.arp_2d(g["poses_est"][k], g["poses_gt"][k], g["pts"], g["K"]) - g["arp_2d"][k]) < 1e-10


def test_toolkit_euler_helpers_and_rendered_pose_sampling_match_the_reference(golden_dir):
    """deepim_b200/toolkit.py: static-xyz euler helpers against the live RT_transform.euler2mat / mat2euler, and the rendered-pose
    sampler against toolkit/LM6d_1_gen_rendered_pose.py's loop run with the reference's helpers and its seed-2333 stream."""
    from deepim_b200 import toolkit
    g = np.load(os.path.join(golden_dir, "ref_euler.npz"))
    for a, m, b in zip(g["angles"], g["mats"], g["back"]):
        np.testing.assert_allclose(toolkit.euler2mat(*a), m, rtol=0, atol=1e-15)
        np.testing.assert_allclose(toolkit.mat2euler(m), b, rtol=0, atol=1e-12)
    # the script's exact random stream is not reproducible (scipy's logm inside calc_rt_dist_m draws from the same global
    # numpy generator, version-dependent), so the sampler is checked on its contract: the first draw -- before any logm call --
    # equals the reference loop's, every pose satisfies the rejection rule as the REFERENCE loop's poses do, and the spread of
    # the accepted rotations matches
    ren = toolkit.gen_rendered_poses(g["poses_observed"], g["K"], n_per_observed=4, seed=2333)
    np.testing.assert_allclose(ren[0, 0], g["poses_rendered"][0, 0], rtol=0, atol=1e-14)
    big = toolkit.gen_rendered_poses(g["poses_observed"], g["K"], n_per_observed=40, seed=7)
    d_mine, d_ref = [], []
    for a in range(3):
        for P, acc in ((big[a], d_mine), (g["poses_rendered"][a], d_ref)):
            for p in P:
                rd = toolkit.rot_dist_deg(p[:, :3], g["poses_observed"][a, :, :3])
                c = g["K"] @ p[:, 3]
                assert rd <= 45.0 and 16 < c[0] / c[2] < 640 - 16 and 16 < c[1] / c[2] < 480 - 16
                acc.append(rd)
        dt = big[a, :, :, 3] - g["poses_observed"][a, :, 3]
        assert np.all(np.abs(dt.std(0) - np.array([0.01, 0.01, 0.05])) < np.array([0.004, 0.004, 0.02]))
    assert 15.0 < np.mean(d_mine) < 30.0 and 10.0 < np.mean(d_ref) < 35.0   # 15 deg per euler axis, truncated at 45 deg
