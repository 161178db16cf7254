"""CPU ORACLE (TEST INFRASTRUCTURE ONLY): BOP 2019's symmetry-aware point errors MSSD and MSPD (Hodan et al., "BOP
Challenge 2019"), in float64 numpy; csrc/bop.cu restates it operation by operation (compiled with -fmad=false).

Per instance m (poses [3,4], camera K_m [3,3]) and symmetry s (syms[s] [3,4]):
1. The GT-symmetric pose, elementwise in this order:
       R_gs[i,j] = (R_gt[i,0] R_s[0,j] + R_gt[i,1] R_s[1,j]) + R_gt[i,2] R_s[2,j]
       t_gs[i]   = ((R_gt[i,0] t_s[0] + R_gt[i,1] t_s[1]) + R_gt[i,2] t_s[2]) + t_gt[i]
2. Points as pose_error_kernel (ADD) transforms them: q[r] = ((P[r,0] x + P[r,1] y) + P[r,2] z) + P[r,3].
3. MSSD(s) = max_p sqrt((dx*dx + dy*dy) + dz*dz) of T_est p - T_gs p.
4. Projections as pose_error2d_kernel (Proj. 2D): c[r] = (K[r,0] q0 + K[r,1] q1) + K[r,2] q2, (u, v) = (c0 / c2, c1 / c2);
   MSPD(s) = max_p sqrt(du*du + dv*dv), du = u_est - u_gs.  A point with Z = q2 <= 0 under either pose makes MSPD(s) = +inf
   (a deliberate deviation: BOP would project the mirrored point).
5. MSSD = min_s MSSD(s), MSPD = min_s MSPD(s); the index is the lowest s reaching the minimum.
max, min and sqrt are exact in any order, so the device's reductions cannot change a bit.

BOP 2019's Visible Surface Discrepancy (dim_pose_error_vsd_ex) is oracle/vsd.py's contract with two switches, restated here
from that module's distance images and SIXD 2017 visibility:
- visib_mode "bop19" replaces vsd.py's step-3 vis() by
      vis(a) = (dist_a > 0) & ((float32(dist_a) - float32(dist_test) <= float32(delta)) | (dist_test == 0))
  so sensor holes count as visible (V_est = vis(est) | (V_gt & (dist_est > 0)) is unchanged);
- diameters [B] (metres) make the taus fractions of each instance's diameter: c_tau counts
  |dist_gt - dist_est| / diameter >= tau (a float64 division).
With "sixd17" and no diameters, vsd() here equals oracle/vsd.py's vsd().
"""
from __future__ import annotations

import numpy as np

from . import oracle as O
from . import vsd as V

_S_BLOCK = 64  # symmetries per numpy block (memory only; the result does not depend on it)


def sym_poses(pose_gt, syms):
    """step 1: [S,3,4] GT-symmetric poses of one GT pose [3,4] and syms [S,3,4]"""
    g = np.asarray(pose_gt, np.float64)
    q = np.asarray(syms, np.float64)
    out = np.empty(q.shape)
    for i in range(3):
        for j in range(3):
            out[:, i, j] = (g[i, 0] * q[:, 0, j] + g[i, 1] * q[:, 1, j]) + g[i, 2] * q[:, 2, j]
        out[:, i, 3] = ((g[i, 0] * q[:, 0, 3] + g[i, 1] * q[:, 1, 3]) + g[i, 2] * q[:, 2, 3]) + g[i, 3]
    return out


def transform(P, pts):
    """step 2: P [...,3,4], pts [N,3] -> [...,3,N]"""
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    P = np.asarray(P, np.float64)[..., None]
    return np.stack([((P[..., r, 0, :] * x + P[..., r, 1, :] * y) + P[..., r, 2, :] * z) + P[..., r, 3, :] for r in range(3)],
                    axis=-2)


def project(K, q):
    """step 4: K [3,3], q [...,3,N] -> (u, v) [...,N]"""
    c = [(K[r, 0] * q[..., 0, :] + K[r, 1] * q[..., 1, :]) + K[r, 2] * q[..., 2, :] for r in range(3)]
    with np.errstate(divide="ignore", invalid="ignore"):
        return c[0] / c[2], c[1] / c[2]


def mssd_mspd(poses_est, poses_gt, points, syms, K):
    """dim_pose_error_sym restated: poses [M,3,4], points [N,3], syms [S,3,4], K [3,3] or [M,3,3] (float64).
    Returns err [M,2] float64 (MSSD metres, MSPD pixels) and idx [M,2] int32 (the minimising symmetries)."""
    poses_est, poses_gt = np.asarray(poses_est, np.float64), np.asarray(poses_gt, np.float64)
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    syms = np.asarray(syms, np.float64).reshape(-1, 3, 4)
    M = len(poses_est)
    Ks = np.asarray(K, np.float64)
    Ks = np.broadcast_to(Ks.reshape(3, 3), (M, 3, 3)) if Ks.size == 9 else Ks.reshape(M, 3, 3)
    err, idx = np.zeros((M, 2)), np.zeros((M, 2), np.int32)
    for m in range(M):
        e = transform(poses_est[m], pts)                     # [3,N]
        ue, ve = project(Ks[m], e)
        d_s, p_s = [], []
        for s0 in range(0, len(syms), _S_BLOCK):
            g = transform(sym_poses(poses_gt[m], syms[s0:s0 + _S_BLOCK]), pts)  # [s,3,N]
            d = e[None] - g
            d_s.append(np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).max(axis=1))
            ug, vg = project(Ks[m], g)
            du, dv = ue[None] - ug, ve[None] - vg
            p = np.sqrt(du * du + dv * dv)
            behind = (e[2] <= 0)[None] | (g[:, 2] <= 0)
            p_s.append(np.where(behind.any(axis=1), np.inf, np.where(behind, 0.0, p).max(axis=1)))
        for k, v in enumerate((np.concatenate(d_s), np.concatenate(p_s))):
            idx[m, k] = int(np.argmin(v))  # the first minimum
            err[m, k] = v[idx[m, k]]
    return err, idx


VISIB_MODES = ("sixd17", "bop19")


def visible(dist_test, dist_model, delta, visib_mode="bop19"):
    """vis() of the visibility mode: "sixd17" is oracle/vsd.py's; "bop19" counts sensor holes as visible"""
    if visib_mode == "sixd17":
        return V.visible(dist_test, dist_model, delta)
    if visib_mode != "bop19":
        raise ValueError("visib_mode must be one of %s" % (VISIB_MODES,))
    diff = np.asarray(dist_model).astype(np.float32) - np.asarray(dist_test).astype(np.float32)
    return (dist_model > 0) & ((diff <= np.float32(delta)) | (dist_test == 0))


def masks(dist_test, dist_est, dist_gt, delta, visib_mode="bop19"):
    """(V_gt, V_est)"""
    v_gt = visible(dist_test, dist_gt, delta, visib_mode)
    v_est = visible(dist_test, dist_est, delta, visib_mode) | (v_gt & (dist_est > 0))
    return v_gt, v_est


def vsd_from_dist(dist_test, dist_est, dist_gt, delta, taus, visib_mode="bop19", diameter=None):
    """oracle/vsd.py's step 4 under the visibility mode, with taus relative to `diameter` when given
    -> (e [n_tau] float64, empty union)"""
    v_gt, v_est = masks(dist_test, dist_est, dist_gt, delta, visib_mode)
    inter = v_gt & v_est
    n_union, n_inter = int(np.count_nonzero(v_gt | v_est)), int(np.count_nonzero(inter))
    if n_union == 0:
        return np.ones(len(taus)), True
    diff = np.abs(dist_gt[inter] - dist_est[inter])
    if diameter is not None:
        diff = diff / float(diameter)
    c = np.array([np.count_nonzero(diff >= float(t)) for t in taus], np.float64)
    return (c + float(n_union - n_inter)) / float(n_union), False


def vsd(meshes, cls_idx, poses_est, poses_gt, depth_frames, K, delta=0.015, taus=(0.02,), frame_idx=None, znear=0.25,
        zfar=6.0, visib_mode="bop19", diameters=None):
    """dim_pose_error_vsd_ex restated: oracle/vsd.py's vsd() (same arguments, renders, distance images and status bits) under
    visib_mode, with diameters [B] (metres; taus relative to them) or None (taus in metres)."""
    if visib_mode not in VISIB_MODES:
        raise ValueError("visib_mode must be one of %s" % (VISIB_MODES,))
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
            f, st = 0, V.STATUS_BAD_FRAME
        c = int(cls_idx[b])
        dt = V.dist_image(depth_frames[f], Ks[f])
        if 0 <= c < len(meshes) and meshes[c] is not None:
            ren = [O.render(meshes[c], P, Ks[f], znear, zfar, H, W, want=("depth",))["depth"] for P in (poses_est[b], poses_gt[b])]
            de, dg = V.dist_image(ren[0], Ks[f]), V.dist_image(ren[1], Ks[f])
        else:
            st |= V.STATUS_BAD_CLASS
            de = dg = np.zeros((H, W))
        err[b], empty = vsd_from_dist(dt, de, dg, delta, taus, visib_mode, None if diameters is None else diameters[b])
        status[b] = st | (V.STATUS_EMPTY if empty else 0)
    return err, status
