"""Float64 reference of the pose algebra (lib/pair_matching/RT_transform.py), independent of the device and of any
eigen-solver: the refinement compose (dim_se3_compose, the fused loop's compose) and the train-time update's refined pose,
labels and KT (dim_train_update).  Transform3D's reference lives in tests/kernel_ref.py.

Conventions, restated from RT_transform.py:
  - quaternions are (w, x, y, z); a delta quaternion is normalised before use (RT_transform, l.135);
  - R_transform: MODEL R = R_src R_delta, CAMERA / CAMERA_NEW R = R_delta R_src; R_inv_transform is its inverse;
  - T_transform: d = t T_stds + T_means, z = z_src / exp(d_z); MODEL / CAMERA x = z (d_x + x_src / z_src),
    CAMERA_NEW x = z_src d_x + x_src (y likewise); T_inv_transform is its inverse, d_z = log(z_src / z_tgt);
  - the train loop's tgt is a float32 array, so T_tgt[0] / T_tgt[2] of MODEL / CAMERA is a float32 division (l.118-119):
    calc_rt_delta does it in float32 when pose_tgt is float32;
  - mat2quat (l.432-509) is the eigenvector of the largest eigenvalue of Bar-Itzhack's symmetric 4x4, which is the
    quaternion of the rotation nearest to M (the orthogonal polar factor, Davenport's q-method).  Here: the polar factor by
    SVD, then scipy's Rotation.from_matrix, w >= 0.

Each function returns (value, S) where S is the same expression evaluated on magnitudes, the scale of a rounding bound
(as tests/kernel_ref.py does)."""
import numpy as np
from scipy.spatial.transform import Rotation

U32 = 2.0 ** -24   # float32 unit roundoff
ULP64 = 2.0 ** -52  # float64 spacing at 1
COORDS = ("MODEL", "CAMERA", "CAMERA_NEW")


def _coord(c):
    c = c.upper()
    if c not in COORDS:
        raise ValueError("unknown rot_coord %r" % c)
    return c


def quat2mat(q):
    """[..., 4] (w, x, y, z), any non-zero norm -> [..., 3, 3]"""
    q = np.asarray(q, np.float64)
    return Rotation.from_quat(q.reshape(-1, 4)[:, [1, 2, 3, 0]]).as_matrix().reshape(q.shape[:-1] + (3, 3))


def mat2quat(M):
    """[..., 3, 3] near-rotation -> [..., 4] (w, x, y, z) of its polar factor, w >= 0.  Where w is 0 (half-turns) the sign
    is scipy's."""
    M = np.asarray(M, np.float64)
    U, _, Vt = np.linalg.svd(M.reshape(-1, 3, 3))
    D = np.ones((len(U), 3))
    D[:, 2] = np.sign(np.linalg.det(U @ Vt))
    R = (U * D[:, None, :]) @ Vt
    q = Rotation.from_matrix(R).as_quat()[:, [3, 0, 1, 2]]
    q[q[:, 0] < 0] *= -1
    return q.reshape(M.shape[:-2] + (4,))


def rotation_set(seed=0, n_random=64):
    """(names, quaternions float64 [n, 4]) of the deltas the pose tests run: identity; 1e-9, 1e-6, 1e-3 rad about random
    axes; n_random rotations uniform on SO(3); exactly pi about x, y, z and a generic axis (w = 0); pi - 1e-6 and pi - 1e-3
    about a generic axis"""
    rng = np.random.default_rng(seed)

    def axis():
        a = rng.normal(size=3)
        return a / np.linalg.norm(a)

    def about(theta, a):
        return np.concatenate([[np.cos(theta / 2)], np.sin(theta / 2) * a])

    names, qs = ["identity"], [np.array([1.0, 0, 0, 0])]
    for th in (1e-9, 1e-6, 1e-3):
        names.append("%g rad" % th)
        qs.append(about(th, axis()))
    for q in Rotation.random(n_random, random_state=seed).as_quat()[:, [3, 0, 1, 2]]:
        names.append("uniform")
        qs.append(q)
    generic = axis()
    for nm, a in (("x", np.eye(3)[0]), ("y", np.eye(3)[1]), ("z", np.eye(3)[2]), ("generic axis", generic)):
        names.append("pi about " + nm)
        qs.append(np.concatenate([[0.0], a]))
    for d in (1e-6, 1e-3):
        names.append("pi - %g rad" % d)
        qs.append(about(np.pi - d, generic))
    qs = np.stack(qs)
    qs[qs[:, 0] < 0] *= -1
    return names, qs


def random_poses(B, seed, z=(0.3, 2.0)):
    """float64 [B, 3, 4]: uniform rotations, x, y within +-0.3 z, z uniform in `z`"""
    rng = np.random.default_rng(seed)
    P = np.zeros((B, 3, 4))
    P[:, :, :3] = Rotation.random(B, random_state=seed).as_matrix()
    P[:, 2, 3] = rng.uniform(*z, size=B)
    P[:, :2, 3] = rng.uniform(-0.3, 0.3, size=(B, 2)) * P[:, 2:3, 3]
    return P


def rt_transform(pose_src, q, t, Tm=(0, 0, 0), Ts=(1, 1, 1), coord="CAMERA"):
    """RT_transform (l.127-151) of [B, 3, 4] source poses by deltas q [B, 4], t [B, 3] -> (pose [B, 3, 4], S)"""
    coord = _coord(coord)
    ps = np.asarray(pose_src, np.float64)
    Rd = quat2mat(q)
    Rs, s = ps[:, :, :3], ps[:, :, 3]
    # quat2mat's rounding errors are absolute (entries of a rotation are <= 1), so the scale of R_src R_delta is R_src's
    # magnitudes summed over the contracted index, as if |R_delta| were all ones
    ones = np.ones((3, 3))
    if coord == "MODEL":
        R, SR = Rs @ Rd, np.abs(Rs) @ ones
    else:
        R, SR = Rd @ Rs, ones @ np.abs(Rs)
    t = np.asarray(t, np.float64)
    Tm, Ts = np.asarray(Tm, np.float64), np.asarray(Ts, np.float64)
    d = t * Ts + Tm
    Sd = np.abs(t * Ts) + np.abs(Tm)
    z2 = s[:, 2] / np.exp(d[:, 2])
    Sz = np.abs(z2) * (1 + Sd[:, 2])
    T, ST = np.zeros((len(ps), 3)), np.zeros((len(ps), 3))
    T[:, 2], ST[:, 2] = z2, Sz
    for k in range(2):
        if coord == "CAMERA_NEW":
            T[:, k] = s[:, 2] * d[:, k] + s[:, k]
            ST[:, k] = np.abs(s[:, 2]) * Sd[:, k] + np.abs(s[:, k])
        else:
            r = s[:, k] / s[:, 2]
            T[:, k] = z2 * (d[:, k] + r)
            ST[:, k] = Sz * (Sd[:, k] + np.abs(r))
    return np.concatenate([R, T[:, :, None]], 2), np.concatenate([SR, ST[:, :, None]], 2)


def calc_rt_delta(pose_src, pose_tgt, Tm=(0, 0, 0), Ts=(1, 1, 1), coord="CAMERA"):
    """calc_RT_delta (l.16-44, rot_type MATRIX) -> (R_delta [B, 3, 3], t_delta [B, 3], S of t_delta).  pose_tgt float32:
    T_tgt[0] / T_tgt[2] and T_tgt[1] / T_tgt[2] are float32 divisions (MODEL / CAMERA), as in the train loop."""
    coord = _coord(coord)
    ps = np.asarray(pose_src, np.float64)
    tg32 = np.asarray(pose_tgt)
    pt = tg32.astype(np.float64)
    Rs, Rt = ps[:, :, :3], pt[:, :, :3]
    Rd = np.swapaxes(Rs, 1, 2) @ Rt if coord == "MODEL" else Rt @ np.swapaxes(Rs, 1, 2)
    s, g = ps[:, :, 3], pt[:, :, 3]
    d, Sd = np.zeros((len(ps), 3)), np.zeros((len(ps), 3))
    for k in range(2):
        if coord == "CAMERA_NEW":
            d[:, k] = (g[:, k] - s[:, k]) / s[:, 2]
            Sd[:, k] = (np.abs(g[:, k]) + np.abs(s[:, k])) / np.abs(s[:, 2])
        else:
            r = (tg32[:, k, 3] / tg32[:, 2, 3]).astype(np.float64)  # float32 / float32 when tgt is float32
            d[:, k] = r - s[:, k] / s[:, 2]
            Sd[:, k] = np.abs(r) + np.abs(s[:, k] / s[:, 2])
    d[:, 2] = np.log(s[:, 2] / g[:, 2])
    Sd[:, 2] = np.abs(d[:, 2])
    Tm, Ts = np.asarray(Tm, np.float64), np.asarray(Ts, np.float64)
    return Rd, (d - Tm) / Ts, (Sd + np.abs(Tm)) / np.abs(Ts)


def kt(K, refined, tgt):
    """K . calc_se3(refined, tgt) = K [R_t R_r^T | t_t - R_t R_r^T t_r] in float64 -> (KT [B, 3, 4], S)"""
    K = np.asarray(K, np.float64)
    r, g = np.asarray(refined, np.float64), np.asarray(tgt, np.float64)
    Rr, tr, Rt, tt = r[:, :, :3], r[:, :, 3:], g[:, :, :3], g[:, :, 3:]
    RrT = np.swapaxes(Rr, 1, 2)
    se3 = np.concatenate([Rt @ RrT, tt - Rt @ (RrT @ tr)], 2)
    S = np.concatenate([np.abs(Rt) @ np.abs(RrT), np.abs(tt) + np.abs(Rt) @ (np.abs(RrT) @ np.abs(tr))], 2)
    return K @ se3, np.abs(K) @ S


def light_position(offset, refined):
    """the ModelNet branch's light for a float64 pose: offset + (t_x, -t_y, -t_z), float64 [B, 3]"""
    r = np.asarray(refined, np.float64)
    o = np.asarray(offset, np.float64)
    return np.stack([o[0] + r[:, 0, 3], o[1] - r[:, 1, 3], o[2] - r[:, 2, 3]], 1)
