"""CPU: the ICP contract (oracle/icp.py) on its own -- fixed point, linearisation, convergence -- and the C prototype of
dim_icp in the ctypes table.  The convergence bound asserted here is the one tests/test_gpu_icp.py holds the device to."""
import math

import numpy as np
import pytest

from deepim_b200 import synth
from oracle import icp as I
from oracle import oracle as O

K = synth.K_LINEMOD
# worst ADD(after 10 iterations) / ADD(before) the oracle reaches below over the C2 and C3 blobs from 1 cm / 3 deg
# perturbations against mm-quantised depth (0.014); the cube is left out: most of its views show one or two planes, which
# leave point-to-plane ICP free to slide
ADD_RATIO_BOUND = 0.02


def perturb(P, rng, t=0.01, deg=3.0):
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    th = np.deg2rad(deg)
    Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    d = rng.normal(size=3)
    Q = P.copy()
    Q[:, :3] = (np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx) @ P[:, :3]
    Q[:, 3] = P[:, 3] + d * (t / np.linalg.norm(d))
    return Q


def add(P, G, pts):
    return np.linalg.norm(pts @ P[:, :3].T + P[:, 3] - (pts @ G[:, :3].T + G[:, 3]), axis=1).mean()


def mm(depth):
    """the u16 file's millimetres, read back as the loader does"""
    return np.rint(depth.astype(np.float64) * 1000.0).astype(np.uint16).astype(np.float32) / np.float32(1000.0)


@pytest.fixture(scope="module")
def blob():
    return synth.make_blob()


def test_fixed_point(blob):
    """observed depth = the render at P: ICP from P keeps P, with residuals at float64 rounding level"""
    P = synth.sample_pose_pairs(1, 4)[0][0]
    dep = O.render(blob, P, K, want=("depth",))["depth"]
    res = I.icp([blob], [0], P[None], dep[None], K, n_iter=3)
    assert (res["status"] == 0).all() and (res["inliers"] > 1000).all()
    assert np.abs(res["poses"] - P).max() < 1e-12
    assert (res["rms"].astype(np.float64) ** 2 < 1e-20).all()
    _, c, e, _, _ = I.step(dep, P, P, dep, K)
    assert c == res["inliers"][0, 0] and e < 1e-20


def test_jacobian_matches_finite_differences(blob):
    """J = (Y x m, m) is d r / d xi for r(xi) = m . (exp([w]x) Y + v - Z), the normal and the target held at the
    linearisation point"""
    G = synth.sample_pose_pairs(1, 5)[0][0]
    P0 = perturb(G, np.random.default_rng(1))
    ren = O.render(blob, P0, K, want=("depth",))["depth"]
    obs = O.render(blob, G, K, want=("depth",))["depth"]
    X, n = I.model_surface(ren, K, 0.02)
    Pk = perturb(P0, np.random.default_rng(2), t=0.002, deg=0.5)
    J, r, Ys, ms, Z = I.associate(X, n, P0, Pk, obs, K, 0.02, points=True)
    assert len(r) > 1000
    assert np.abs(np.einsum("ij,ij->i", ms, Ys - Z) - r).max() < 1e-15
    h = 1e-6
    for a in range(6):
        xi = np.zeros(6)
        xi[a] = h
        fd = []
        for s in (1.0, -1.0):
            w, v = s * xi[:3], s * xi[3:]
            Rw = np.array(I.rodrigues(list(w)))
            fd.append(np.einsum("ij,ij->i", ms, Ys @ Rw.T + v - Z))
        num = (fd[0] - fd[1]) / (2 * h)
        assert np.abs(num - J[:, a]).max() <= 1e-6 * np.abs(J[:, a]).max(), a


def test_solve_refuses_few_points_and_singular_systems():
    P = np.hstack([np.eye(3), np.array([[0.0], [0.0], [1.0]])])
    A, g = np.eye(6), np.ones(6)
    assert I.solve(A, g, 5, P, 6)[1] is False
    A[5, 5] = 1e-13
    P1, ok = I.solve(A, g, 100, P, 6)
    assert ok is False and np.array_equal(P1, P)
    P1, ok = I.solve(np.eye(6), np.zeros(6), 100, P, 6)
    assert ok and np.abs(P1 - P).max() == 0.0


@pytest.mark.parametrize("mesh_id", ["C2", "C3-04", "C3-12"])
def test_convergence_from_1cm_3deg(mesh_id):
    """1 cm / 3 deg perturbations against the depth rendered at the true pose and rounded to mm: ADD shrinks by at least 5x,
    and to the recorded bound"""
    mesh = synth.make_blob() if mesh_id == "C2" else synth.make_linemod_like_set()[int(mesh_id[3:])]
    pts = mesh.verts.astype(np.float64)
    rng = np.random.default_rng(7)
    obs, _ = synth.sample_pose_pairs(4, 11)
    for G in obs:
        dep = mm(O.render(mesh, G, K, want=("depth",))["depth"])
        P0 = perturb(G, rng)
        res = I.icp([mesh], [0], P0[None], dep[None], K, n_iter=10)
        ratio = add(res["poses"][-1, 0], G, pts) / add(P0, G, pts)
        assert ratio <= 0.2 and ratio <= ADD_RATIO_BOUND, ratio
        assert (res["status"] == 0).all()


def test_status_bits():
    """out of view -> bit 0 (pose kept), bad class -> bits 0 + 1, bad frame -> bit 3, starved -> bit 4"""
    blob = synth.make_blob()
    G = synth.sample_pose_pairs(1, 6)[0][0]
    dep = mm(O.render(blob, G, K, want=("depth",))["depth"])
    away = G.copy()
    away[:, 3] = [5.0, 0.0, 0.8]
    poses = np.stack([G, away, G, G])
    res = I.icp([blob], [0, 0, 3, 0], poses, dep[None], K, n_iter=2, frame_idx=[0, 0, 0, 7], min_points=6)
    assert list(res["status"][0]) == [0, 1, 3, 8]
    assert np.array_equal(res["poses"][-1, 1], away)
    res = I.icp([blob], [0], G[None], dep[None], K, n_iter=1, min_points=10 ** 7)
    assert res["status"][0, 0] == 16 and np.array_equal(res["poses"][0, 0], G)
    assert res["inliers"][0, 0] > 0 and math.isfinite(res["rms"][0, 0])


def test_capi_declares_dim_icp():
    """the new entry is in the ctypes table; the header-coverage tests check its prototype"""
    from deepim_b200 import _capi
    assert "dim_icp" in _capi.SIGNATURES and "dim_depth_from_u16" in _capi.SIGNATURES
    assert len(_capi.SIGNATURES["dim_icp"][1]) == 19
