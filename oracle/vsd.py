"""CPU ORACLE (TEST INFRASTRUCTURE ONLY): the Visible Surface Discrepancy of Hodan et al. ("On Evaluation of 6D Object Pose
Estimation", ECCVW 2016), in float64 numpy; csrc/vsd.cu restates it operation by operation (compiled with -fmad=false).

Per instance, with the frame's camera K (float32), the observed depth D_test (metres, 0 = hole) and the poses P_est, P_gt:
1. D_est, D_gt: the depth renders of the mesh at float32(P_est), float32(P_gt) (the refinement loop's rasteriser,
   oracle.render).
2. Distance images as lib/utils/misc.py:20 depth_im_to_dist_im computes them with a float32 K under numpy 2:
       X = ((j - cx) * d) * float32(1 / fx),  Y = ((i - cy) * d) * float32(1 / fy),  dist = sqrt((X*X + Y*Y) + d*d)
   in float64 (the reciprocal is a float32 division; np.linalg.norm sums the three squares left to right).
   tests/golden/ref_vsd.npz pins this against the live function bit for bit.
3. Visibility as lib/utils/visibility.py computes it:
       vis(a) = (dist_test > 0) & (dist_a > 0) & (float32(dist_a) - float32(dist_test) <= float32(delta))
       V_gt = vis(gt),  V_est = vis(est) | (V_gt & (dist_est > 0))
4. The "step" cost of the paper: inter = V_gt & V_est, union = V_gt | V_est, for each tau
       c_tau = #{inter pixels with |dist_gt - dist_est| >= tau}   (float64)
       e_tau = (c_tau + |union| - |inter|) / |union|,  e_tau = 1 when the union is empty.
Every sum is an integer count, so e does not depend on any reduction order.
"""
from __future__ import annotations

import numpy as np

from . import oracle as O

STATUS_EMPTY, STATUS_BAD_CLASS, STATUS_BAD_FRAME = 1, 2, 8


def dist_image(depth, K):
    """depth [H,W] (float32 metres) -> distance image [H,W] float64 (step 2)"""
    K = np.asarray(K, np.float32).reshape(3, 3)
    d = np.asarray(depth, np.float32).astype(np.float64)
    H, W = d.shape
    j = np.arange(W, dtype=np.float64)[None, :]
    i = np.arange(H, dtype=np.float64)[:, None]
    rfx = float(np.float32(1.0) / K[0, 0])
    rfy = float(np.float32(1.0) / K[1, 1])
    X = ((j - float(K[0, 2])) * d) * rfx
    Y = ((i - float(K[1, 2])) * d) * rfy
    return np.sqrt((X * X + Y * Y) + d * d)


def visible(dist_test, dist_model, delta):
    """step 3's vis(): float32 difference against float32(delta)"""
    diff = np.asarray(dist_model).astype(np.float32) - np.asarray(dist_test).astype(np.float32)
    return (dist_test > 0) & (dist_model > 0) & (diff <= np.float32(delta))


def masks(dist_test, dist_est, dist_gt, delta):
    """(V_gt, V_est)"""
    v_gt = visible(dist_test, dist_gt, delta)
    v_est = visible(dist_test, dist_est, delta) | (v_gt & (dist_est > 0))
    return v_gt, v_est


def vsd_from_dist(dist_test, dist_est, dist_gt, delta, taus):
    """step 4 -> (e [n_tau] float64, empty union)"""
    v_gt, v_est = masks(dist_test, dist_est, dist_gt, delta)
    inter = v_gt & v_est
    n_union, n_inter = int(np.count_nonzero(v_gt | v_est)), int(np.count_nonzero(inter))
    if n_union == 0:
        return np.ones(len(taus)), True
    diff = np.abs(dist_gt[inter] - dist_est[inter])
    c = np.array([np.count_nonzero(diff >= float(t)) for t in taus], np.float64)
    return (c + float(n_union - n_inter)) / float(n_union), False


def vsd(meshes, cls_idx, poses_est, poses_gt, depth_frames, K, delta=0.015, taus=(0.02,), frame_idx=None, znear=0.25,
        zfar=6.0):
    """dim_pose_error_vsd restated: meshes indexed by class, poses [B,3,4], depth_frames [F,H,W] float32 metres, K [3,3] or
    [F,3,3], frame_idx [B] or None (instance b observes frame b).  Returns err [B,n_tau] float64, status [B] int32 (bit 0
    empty union, bit 1 bad class, bit 3 frame index outside [0, F): frame 0 instead)."""
    depth_frames = np.asarray(depth_frames, np.float32)
    F, H, W = depth_frames.shape
    B = len(cls_idx)
    Ks = np.asarray(K, np.float32)
    Ks = np.broadcast_to(Ks.reshape(3, 3), (F, 3, 3)) if Ks.ndim == 2 else Ks
    err, status = np.zeros((B, len(taus))), np.zeros(B, np.int32)
    for b in range(B):
        f = b if frame_idx is None else int(frame_idx[b])
        st = 0
        if not 0 <= f < F:
            f, st = 0, STATUS_BAD_FRAME
        c = int(cls_idx[b])
        dt = dist_image(depth_frames[f], Ks[f])
        if 0 <= c < len(meshes) and meshes[c] is not None:
            ren = [O.render(meshes[c], P, Ks[f], znear, zfar, H, W, want=("depth",))["depth"] for P in (poses_est[b], poses_gt[b])]
            de, dg = dist_image(ren[0], Ks[f]), dist_image(ren[1], Ks[f])
        else:
            st |= STATUS_BAD_CLASS
            de = dg = np.zeros((H, W))
        err[b], empty = vsd_from_dist(dt, de, dg, delta, taus)
        status[b] = st | (STATUS_EMPTY if empty else 0)
    return err, status
