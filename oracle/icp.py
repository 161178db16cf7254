"""CPU ORACLE (TEST INFRASTRUCTURE ONLY): projective point-to-plane ICP against observed depth, in float64.

The reference has no ICP of its own (its evaluation only reads `-pose_icp.txt` poses computed elsewhere), so this module
*defines* what dim_icp computes; csrc/icp.cu restates it operation by operation (compiled with -fmad=false).

Per instance: the model surface is the depth render at float32(P0) (the rasteriser of the refinement loop, oracle.render).
Model pixel (i, j) has depth d > 0, so do its four neighbours, and no neighbour differs from d by more than max_dist.  It
back-projects to X = ((j - cx) d / fx, (i - cy) d / fy, d) (the inverse of raster_vertex_kernel's sx = fx x / z + cx, pixel
(i, j) sampling image point (j, i)); its normal is normalize((X[i,j+1] - X[i,j-1]) x (X[i+1,j] - X[i-1,j])), flipped so
that n . X < 0.  Iteration k (state: the float64 pose P_k):
    R_D = R_k R0^T, t_D = t_k - R_D t0;  Y = R_D X + t_D, m = R_D n
    q = (rint(fy Y.y / Y.z + cy), rint(fx Y.x / Y.z + cx)), inside the frame, Y.z > 0; d_o = depth[q] finite and > 0
    Z = backproject(q, d_o); inlier iff |Y.z - d_o| < max_dist; r = m . (Y - Z), J = (Y x m, m)
    A = sum J J^T, g = sum J r, c = #inliers, e = sum r^2
    c < min_points or a Cholesky pivot <= 1e-12 max(diag A): pose unchanged; else xi = -A^-1 g = (w, v),
    P_{k+1} = (Rodrigues(w) R_k, Rodrigues(w) t_k + v)
J is the derivative of r with the normal m and the target Z frozen at the linearisation point (point-to-plane
Gauss-Newton): r(xi) = m . (exp([w]x) Y + v - Z).

Every per-pixel value up to the accumulation is computed elementwise in the same float64 order as the device, so an
association fed the device's P_k reproduces the device's inlier count exactly; the sums differ from the device's
fixed-order reduction only by rounding.
"""
from __future__ import annotations

import math

import numpy as np

from . import oracle as O

STATUS_EMPTY, STATUS_BAD_CLASS, STATUS_BAD_FRAME, STATUS_NO_SOLVE = 1, 2, 8, 16
UPPER = [(a, b) for a in range(6) for b in range(a, 6)]  # the 21 entries of A in the order the device accumulates them


def _intr(K):
    K = np.asarray(K, np.float32).reshape(3, 3)
    return float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])


def model_surface(depth, K, max_dist):
    """Model pixels of a rendered depth [H,W] float32 -> (X [N,3], n [N,3]) float64, row-major pixel order."""
    fx, fy, cx, cy = _intr(K)
    md = float(np.float32(max_dist))
    d = np.asarray(depth, np.float32).astype(np.float64)
    H, W = d.shape
    c = d[1:-1, 1:-1]
    nb = [d[1:-1, 2:], d[1:-1, :-2], d[2:, 1:-1], d[:-2, 1:-1]]  # right, left, down, up
    ok = c > 0
    for e in nb:
        ok &= (e > 0) & ~(np.abs(e - c) > md)
    ii, jj = np.nonzero(ok)
    ii, jj = ii + 1, jj + 1

    def bp(i, j):
        z = d[i, j]
        return ((j - cx) * z) / fx, ((i - cy) * z) / fy, z

    X = bp(ii, jj)
    r, l, dn, up = bp(ii, jj + 1), bp(ii, jj - 1), bp(ii + 1, jj), bp(ii - 1, jj)
    a = [r[k] - l[k] for k in range(3)]
    b = [dn[k] - up[k] for k in range(3)]
    c0 = a[1] * b[2] - a[2] * b[1]
    c1 = a[2] * b[0] - a[0] * b[2]
    c2 = a[0] * b[1] - a[1] * b[0]
    ln = np.sqrt((c0 * c0 + c1 * c1) + c2 * c2)
    keep = ln != 0
    with np.errstate(invalid="ignore", divide="ignore"):
        n = [c0 / ln, c1 / ln, c2 / ln]
    flip = ((n[0] * X[0] + n[1] * X[1]) + n[2] * X[2]) > 0
    n = [np.where(flip, -v, v) for v in n]
    return np.stack(X, 1)[keep], np.stack(n, 1)[keep]


def increment(P0, Pk):
    """(R_D, t_D) as nested Python floats: R_D = R_k R0^T, t_D = t_k - R_D t0, each sum left to right."""
    P0, Pk = np.asarray(P0, np.float64).tolist(), np.asarray(Pk, np.float64).tolist()
    R = [[(Pk[a][0] * P0[b][0] + Pk[a][1] * P0[b][1]) + Pk[a][2] * P0[b][2] for b in range(3)] for a in range(3)]
    t = [Pk[a][3] - ((R[a][0] * P0[0][3] + R[a][1] * P0[1][3]) + R[a][2] * P0[2][3]) for a in range(3)]
    return R, t


def associate(X, n, P0, Pk, depth, K, max_dist, points=False):
    """The inliers of one iteration: (J [c,6], r [c]) float64; points=True appends their Y, m and Z [c,3]."""
    fx, fy, cx, cy = _intr(K)
    md = float(np.float32(max_dist))
    R, t = increment(P0, Pk)
    H, W = depth.shape
    x0, x1, x2 = X[:, 0], X[:, 1], X[:, 2]
    n0, n1, n2 = n[:, 0], n[:, 1], n[:, 2]
    Y = [((R[a][0] * x0 + R[a][1] * x1) + R[a][2] * x2) + t[a] for a in range(3)]
    m = [(R[a][0] * n0 + R[a][1] * n1) + R[a][2] * n2 for a in range(3)]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        u = (fx * Y[0]) / Y[2] + cx
        v = (fy * Y[1]) / Y[2] + cy
        qj, qi = np.rint(u), np.rint(v)
        ok = (Y[2] > 0) & (qj >= 0) & (qj <= W - 1) & (qi >= 0) & (qi <= H - 1)
    qi_, qj_ = np.where(ok, qi, 0).astype(np.int64), np.where(ok, qj, 0).astype(np.int64)
    do = np.asarray(depth, np.float32)[qi_, qj_]
    ok &= np.isfinite(do) & (do > 0)
    do = do.astype(np.float64)
    Z = [((qj - cx) * do) / fx, ((qi - cy) * do) / fy, do]
    ok &= np.abs(Y[2] - do) < md
    Y = [y[ok] for y in Y]
    m = [y[ok] for y in m]
    Z = [z[ok] for z in Z]
    r = (m[0] * (Y[0] - Z[0]) + m[1] * (Y[1] - Z[1])) + m[2] * (Y[2] - Z[2])
    J = np.stack([Y[1] * m[2] - Y[2] * m[1], Y[2] * m[0] - Y[0] * m[2], Y[0] * m[1] - Y[1] * m[0], m[0], m[1], m[2]], 1)
    return (J, r, np.stack(Y, 1), np.stack(m, 1), np.stack(Z, 1)) if points else (J, r)


def rodrigues(w):
    """exp([w]x) as nested floats; I + [w]x below |w| = 1e-12"""
    th = math.sqrt((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2])
    if th < 1e-12:
        return [[1.0, -w[2], w[1]], [w[2], 1.0, -w[0]], [-w[1], w[0], 1.0]]
    k = [w[0] / th, w[1] / th, w[2] / th]
    s, c = math.sin(th), math.cos(th)
    C = 1.0 - c
    return [[c + C * k[0] * k[0], C * k[0] * k[1] - s * k[2], C * k[0] * k[2] + s * k[1]],
            [C * k[1] * k[0] + s * k[2], c + C * k[1] * k[1], C * k[1] * k[2] - s * k[0]],
            [C * k[2] * k[0] - s * k[1], C * k[2] * k[1] + s * k[0], c + C * k[2] * k[2]]]


def solve(A, g, c, Pk, min_points):
    """-> (P_{k+1}, solved).  Cholesky with the pivot test of the contract; unsolved keeps P_k."""
    Pk = np.asarray(Pk, np.float64)
    if c < min_points:
        return Pk.copy(), False
    A = np.asarray(A, np.float64).tolist()
    g = np.asarray(g, np.float64).tolist()
    tol = 1e-12 * max(A[i][i] for i in range(6))
    L = [[0.0] * 6 for _ in range(6)]
    for j in range(6):
        s = A[j][j]
        for k in range(j):
            s -= L[j][k] * L[j][k]
        if s <= tol:
            return Pk.copy(), False
        L[j][j] = math.sqrt(s)
        for i in range(j + 1, 6):
            s = A[j][i]
            for k in range(j):
                s -= L[i][k] * L[j][k]
            L[i][j] = s / L[j][j]
    y = [0.0] * 6
    for i in range(6):
        s = -g[i]
        for k in range(i):
            s -= L[i][k] * y[k]
        y[i] = s / L[i][i]
    x = [0.0] * 6
    for i in range(5, -1, -1):
        s = y[i]
        for k in range(i + 1, 6):
            s -= L[k][i] * x[k]
        x[i] = s / L[i][i]
    dR = rodrigues(x[:3])
    P = Pk.tolist()
    out = np.zeros((3, 4))
    for a in range(3):
        for b in range(3):
            out[a, b] = (dR[a][0] * P[0][b] + dR[a][1] * P[1][b]) + dR[a][2] * P[2][b]
        out[a, 3] = ((dR[a][0] * P[0][3] + dR[a][1] * P[1][3]) + dR[a][2] * P[2][3]) + x[3 + a]
    return out, True


def step(render_depth, P0, Pk, depth, K, max_dist=0.02, min_points=64, surface=None):
    """One iteration fed P_k (teacher forcing): (P_{k+1}, c, e, A [6,6], g [6]).  render_depth: the depth render at
    float32(P0); surface: model_surface(render_depth, K, max_dist) when already computed."""
    X, n = surface if surface is not None else model_surface(render_depth, K, max_dist)
    J, r = associate(X, n, P0, Pk, depth, K, max_dist)
    A, g, c, e = J.T @ J, J.T @ r, len(r), float(r @ r)
    P1, _ = solve(A, g, c, Pk, min_points)
    return P1, c, e, A, g


def icp(meshes, cls_idx, pose_in, depth_frames, K, n_iter=10, max_dist=0.02, min_points=64, frame_idx=None, znear=0.25,
        zfar=6.0):
    """dim_icp restated: meshes indexed by class, pose_in [B,3,4], depth_frames [F,H,W] float32 metres, K [3,3] or
    [F,3,3], frame_idx [B] or None (instance b observes frame b).  Returns poses [n_iter,B,3,4], inliers, rms, status."""
    pose_in = np.asarray(pose_in, np.float64)
    depth_frames = np.asarray(depth_frames, np.float32)
    F, H, W = depth_frames.shape
    B = len(pose_in)
    Ks = np.asarray(K, np.float32)
    Ks = np.broadcast_to(Ks.reshape(3, 3), (F, 3, 3)) if Ks.ndim == 2 else Ks
    res = {"poses": np.zeros((n_iter, B, 3, 4)), "inliers": np.zeros((n_iter, B), np.int32),
           "rms": np.zeros((n_iter, B), np.float32), "status": np.zeros((n_iter, B), np.int32)}
    for b in range(B):
        f = b if frame_idx is None else int(frame_idx[b])
        base = 0
        if not 0 <= f < F:
            f, base = 0, STATUS_BAD_FRAME
        c_ = int(cls_idx[b])
        if 0 <= c_ < len(meshes) and meshes[c_] is not None:
            ren = O.render(meshes[c_], pose_in[b], Ks[f], znear, zfar, H, W, want=("depth",))["depth"]
            surf = model_surface(ren, Ks[f], max_dist)
        else:
            base |= STATUS_BAD_CLASS
            surf = (np.zeros((0, 3)), np.zeros((0, 3)))
        P = pose_in[b].copy()
        for k in range(n_iter):
            st = base
            if len(surf[0]) == 0:
                st |= STATUS_EMPTY
                c, e, P1 = 0, 0.0, P
            else:
                J, r = associate(surf[0], surf[1], pose_in[b], P, depth_frames[f], Ks[f], max_dist)
                c, e = len(r), float(r @ r)
                P1, ok = solve(J.T @ J, J.T @ r, c, P, min_points)
                if not ok:
                    st |= STATUS_NO_SOLVE
            res["poses"][k, b], res["inliers"][k, b], res["status"][k, b] = P1, c, st
            res["rms"][k, b] = math.sqrt(e / c) if c else 0.0
            P = P1
    return res
