"""CPU: the float64 pose-algebra reference (tests/pose_ref.py) against the live reference's RT_transform
(tests/golden/ref_se3.npz), against its own inverse, against the oracle's eigh-based mat2quat, and Transform3D's CAMERA_NEW
reference (tests/kernel_ref.py) against finite differences."""
import os

import numpy as np
import pytest
import torch

import kernel_ref as R
import pose_ref as P
from oracle import oracle as O


@pytest.mark.parametrize("coord", P.COORDS)
def test_rt_transform_reproduces_the_reference_golden(golden_dir, coord):
    g = np.load(os.path.join(golden_dir, "ref_se3.npz"))
    pose, _ = P.rt_transform(g["pose_src"], g["quat"], g["trans"], coord=coord)
    np.testing.assert_allclose(pose, g["pose_out_" + coord], rtol=0, atol=1e-12)
    pose, _ = P.rt_transform(g["pose_src"], g["quat"], g["trans"], g["T_means"], g["T_stds"], coord)
    np.testing.assert_allclose(pose, g["pose_out_norm_" + coord], rtol=0, atol=1e-12)
    Rd, td, _ = P.calc_rt_delta(g["pose_src"], g["pose_out_norm_" + coord], g["T_means"], g["T_stds"], coord)
    np.testing.assert_allclose(Rd, g["R_delta_" + coord], rtol=0, atol=1e-12)
    np.testing.assert_allclose(td, g["T_delta_" + coord], rtol=0, atol=1e-12)


def test_train_labels_reproduce_the_reference_golden(golden_dir):
    """calc_RT_delta(..., "QUAT") against a float32 tgt (eigh in the reference, the polar factor + scipy here) and K . calc_se3
    (the reference stores se3 in float32, so KT agrees to float32 rounding of se3 only)"""
    g = np.load(os.path.join(golden_dir, "ref_se3.npz"))
    tgt32 = g["pose_out_CAMERA"].astype(np.float32)
    Rd, td, _ = P.calc_rt_delta(g["pose_src"], tgt32)
    np.testing.assert_allclose(P.mat2quat(Rd), g["label_quat"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(td, g["label_trans"], rtol=0, atol=1e-12)
    KT, S = P.kt(g["label_K"], g["pose_src"], tgt32)
    assert (np.abs(KT - g["label_KT"]) <= 8 * P.U32 * S).all()


@pytest.mark.parametrize("coord", P.COORDS)
@pytest.mark.parametrize("norm", [((0, 0, 0), (1, 1, 1)), ((0.0625, -0.125, 0.03125), (0.5, 2.0, 0.75))])
def test_calc_rt_delta_inverts_rt_transform(coord, norm):
    """over the whole rotation set, half-turns and 1e-9 rad included: delta(src, compose(src, q, t)) = (R(q), t)"""
    _, Q = P.rotation_set()
    B = len(Q)
    src = P.random_poses(B, 1)
    t = np.random.default_rng(2).normal(size=(B, 3)) * [0.05, 0.05, 0.2]
    tgt, _ = P.rt_transform(src, Q, t, *norm, coord)
    Rd, td, _ = P.calc_rt_delta(src, tgt, *norm, coord)
    np.testing.assert_allclose(Rd, P.quat2mat(Q), rtol=0, atol=1e-12)
    np.testing.assert_allclose(td, t, rtol=0, atol=1e-12)
    q = P.mat2quat(Rd)
    sign = np.where(np.abs(Q[:, 0]) <= 1e-6, np.sign((q * Q).sum(1)), 1.0)  # half-turns: either sign
    np.testing.assert_allclose(q, Q * sign[:, None], rtol=0, atol=1e-12)
    assert (q[:, 0] >= 0).all()


def test_mat2quat_agrees_with_eigh_away_from_half_turns():
    """the polar factor + scipy against the oracle's Bar-Itzhack eigh, on exact rotations and on float32-rounded ones (the
    train loop's delta is not exactly orthogonal)"""
    _, Q = P.rotation_set()
    src = P.random_poses(len(Q), 3)
    for M in (P.quat2mat(Q), P.calc_rt_delta(src, P.rt_transform(src, Q, np.zeros((len(Q), 3)))[0].astype(np.float32))[0]):
        q = P.mat2quat(M)
        for k in range(len(Q)):
            if abs(q[k, 0]) > 1e-6:
                np.testing.assert_allclose(q[k], O.mat2quat(M[k]), rtol=0, atol=1e-12)


@pytest.mark.parametrize("rot_coord", ["MODEL", "CAMERA"])
def test_transform3d_matches_the_oracle(rot_coord):
    rng = np.random.default_rng(5)
    B, N = 3, 17
    P_ = (rng.normal(size=(B, 3, N)) * 0.1).astype(np.float32)
    q = rng.normal(size=(B, 4))
    q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    t = (rng.normal(size=(B, 3)) * 0.05).astype(np.float32)
    ps = P.random_poses(B, 4).astype(np.float32)
    D = rng.normal(size=(B, 3, N)).astype(np.float32)
    Tm, Ts = (0.0625, -0.125, 0.03125), (0.5, 2.0, 0.75)
    T = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    ref, S = R.transform3d_fwd(T(P_), T(q), T(t), T(ps), Tm, Ts, rot_coord)
    assert ((ref - T(O.transform3d_forward(P_, q, t, ps, Tm, Ts, rot_coord))).abs() <= 8 * P.U32 * S).all()
    (rg, _), (tg, _) = R.transform3d_bwd(T(D), T(P_), T(q), T(t), T(ps), Tm, Ts, rot_coord)
    org, otg = O.transform3d_backward(D, P_, q, t, ps, Tm, Ts, rot_coord)
    np.testing.assert_allclose(rg.numpy(), org, rtol=1e-5, atol=1e-5 * np.abs(org).max())
    np.testing.assert_allclose(tg.numpy(), otg, rtol=1e-5, atol=1e-5 * np.abs(otg).max())


def test_transform3d_camera_new_gradient_matches_finite_differences():
    """CAMERA_NEW: the forward equals RT_transform applied to the points, and the hand-written backward (rotation through the
    normalised quaternion, translation through T_stds) equals central differences of sum(D * forward)"""
    rng = np.random.default_rng(6)
    B, N = 3, 13
    Pt = torch.from_numpy(rng.normal(size=(B, 3, N)) * 0.1)
    q = rng.normal(size=(B, 4)) * 0.2 + [1, 0, 0, 0]
    q = torch.from_numpy(q / np.linalg.norm(q, axis=1, keepdims=True))
    t = torch.from_numpy(rng.normal(size=(B, 3)) * 0.05)
    ps = torch.from_numpy(P.random_poses(B, 7))
    D = torch.from_numpy(rng.normal(size=(B, 3, N)))
    Tm, Ts = (0.0625, -0.125, 0.03125), (0.5, 2.0, 0.75)
    fwd = lambda qq, tt: R.transform3d_fwd(Pt, qq, tt, ps, Tm, Ts, "CAMERA_NEW")[0]
    pose, _ = P.rt_transform(ps.numpy(), q.numpy(), t.numpy(), Tm, Ts, "CAMERA_NEW")
    np.testing.assert_allclose(fwd(q, t).numpy(), pose[:, :, :3] @ Pt.numpy() + pose[:, :, 3:], rtol=0, atol=1e-14)
    (rg, _), (tg, _) = R.transform3d_bwd(D, Pt, q, t, ps, Tm, Ts, "CAMERA_NEW")
    h = 1e-6
    for arg, grad in ((0, rg), (1, tg)):
        x = (q, t)[arg]
        fd = torch.zeros_like(x)
        for b in range(B):
            for k in range(x.shape[1]):
                e = torch.zeros_like(x)
                e[b, k] = h
                lo, hi = [(fwd(q + s * e, t) if arg == 0 else fwd(q, t + s * e)) for s in (-1, 1)]
                fd[b, k] = ((hi - lo) * D).sum() / (2 * h)
        np.testing.assert_allclose(grad.numpy(), fd.numpy(), rtol=1e-6, atol=1e-6 * fd.abs().max().item())
