"""CPU: the VSD contract (oracle/vsd.py) -- its distance images and visibility masks against the reference's own functions
(tests/golden/ref_vsd.npz, made by make_golden_vsd.py), known answers of the error, and the C prototype of
dim_pose_error_vsd in the ctypes table."""
import os

import numpy as np
import pytest

from deepim_b200 import synth
from oracle import oracle as O
from oracle import vsd as V

K = synth.K_LINEMOD
TAUS = (0.005, 0.01, 0.02, 0.05)
# worst e (every tau above) the oracle gives for the cube turned 90 deg about each face axis, over 8 sampled poses: 1.25e-4
# (a few silhouette pixels the rasteriser's fill rule assigns differently)
CUBE_TURN_BOUND = 1e-3


@pytest.fixture(scope="module")
def ref(golden_dir):
    return np.load(os.path.join(golden_dir, "ref_vsd.npz"))


@pytest.mark.parametrize("case", [0, 1])
def test_distance_images_and_masks_equal_the_reference(ref, case):
    r = lambda k: ref["r%d_%s" % (case, k)]
    for n in ("test", "gt", "est"):
        assert np.array_equal(V.dist_image(r("depth_" + n), r("K")), r("dist_" + n)), n
    v_gt, v_est = V.masks(r("dist_test"), r("dist_est"), r("dist_gt"), 0.015)
    assert np.array_equal(v_gt, r("visib_gt")) and np.array_equal(v_est, r("visib_est"))
    assert r("visib_gt").sum() > 500 and (r("visib_gt") != r("visib_est")).any()


@pytest.mark.parametrize("case", [0, 1])
def test_masks_on_the_delta_boundary_equal_the_reference(ref, case):
    """float32(dist_model) - float32(dist_test) == float32(delta) is visible, also for delta = 0.1 where float32(0.1) > 0.1
    makes the same difference invisible in float64; at about 1 m the nearest difference below is visible, above is not"""
    b = lambda k: ref["b%d_%s" % (case, k)]
    delta = float(b("delta"))
    v_gt, v_est = V.masks(b("dist_test"), b("dist_est"), b("dist_gt"), delta)
    assert np.array_equal(v_gt, b("visib_gt")) and np.array_equal(v_est, b("visib_est"))
    t, m = b("dist_test"), b("dist_est")
    on = (t > 0) & (m > 0)
    diff = m.astype(np.float32) - t.astype(np.float32)
    assert on.sum(1).min() > 30 and (diff[0][on[0]] == np.float32(delta)).all()
    vis = V.visible(t, m, delta)
    assert vis[0][on[0]].all() and vis[1][on[1]].all() and not vis[2].any()
    if delta == 0.1:
        assert not (diff[0][on[0]].astype(np.float64) <= delta).any()


@pytest.fixture(scope="module")
def blob_scene():
    blob = synth.make_blob()
    G = synth.sample_pose_pairs(1, 3)[0][0]
    return blob, G, O.render(blob, G, K, want=("depth",))["depth"]


def test_est_equal_gt_on_exact_depth_is_zero(blob_scene):
    blob, G, dep = blob_scene
    e, st = V.vsd([blob], [0], G[None], G[None], dep[None], K, 0.015, TAUS)
    assert st[0] == 0 and (e == 0.0).all()


def test_disjoint_renders_and_empty_union_are_one(blob_scene):
    blob, G, dep = blob_scene
    away = G.copy()
    away[0, 3] += 0.3  # beside the object, still in view
    e, st = V.vsd([blob], [0], away[None], G[None], dep[None], K, 0.015, TAUS)
    assert st[0] == 0 and (e == 1.0).all()
    e, st = V.vsd([blob], [0], G[None], G[None], np.zeros_like(dep)[None], K, 0.015, TAUS)  # nothing observed
    assert st[0] == V.STATUS_EMPTY and (e == 1.0).all()


def test_error_does_not_increase_with_tau(blob_scene):
    blob, G, dep = blob_scene
    rng = np.random.default_rng(4)
    from test_icp_oracle import perturb
    taus = np.linspace(0.001, 0.1, 16)
    for _ in range(3):
        e, _ = V.vsd([blob], [0], perturb(G, rng)[None], G[None], dep[None], K, 0.015, taus)
        assert (np.diff(e[0]) <= 0).all() and e[0, 0] > e[0, -1]


def test_occluder_removes_its_pixels_from_both_masks(blob_scene):
    blob, G, dep = blob_scene
    from test_icp_oracle import perturb
    E = perturb(G, np.random.default_rng(5), t=0.003, deg=1.0)
    ys, xs = np.nonzero(dep)
    occ = np.zeros(dep.shape, bool)
    occ[ys.min():(ys.min() + ys.max()) // 2, xs.min():(xs.min() + xs.max()) // 2] = True
    occluded = dep.copy()
    occluded[occ] = np.float32(float(G[2, 3]) - 0.06)
    d_e = V.dist_image(O.render(blob, E, K, want=("depth",))["depth"], K)
    d_g = V.dist_image(dep, K)
    free = V.masks(V.dist_image(dep, K), d_e, d_g, 0.015)
    hidden = V.masks(V.dist_image(occluded, K), d_e, d_g, 0.015)
    for f, h in zip(free, hidden):
        assert (f & occ).sum() > 100 and not (h & occ).any()
        assert np.array_equal(f & ~occ, h & ~occ)


def test_cube_turned_90_degrees_about_a_face_axis():
    cube = synth.make_cube()
    worst = 0.0
    for s in range(8):
        G = synth.sample_pose_pairs(1, 30 + s)[0][0]
        dep = O.render(cube, G, K, want=("depth",))["depth"]
        for a, b in ((1, 2), (0, 2), (0, 1)):
            R = np.eye(3)
            R[a, a] = R[b, b] = 0.0
            R[a, b], R[b, a] = -1.0, 1.0
            E = G.copy()
            E[:, :3] = G[:, :3] @ R
            e, st = V.vsd([cube], [0], E[None], G[None], dep[None], K, 0.015, TAUS)
            assert st[0] == 0
            worst = max(worst, e.max())
    assert worst < CUBE_TURN_BOUND, worst


def test_status_bits(blob_scene):
    """bad class -> bits 0 + 1 (e = 1), frame index outside [0, F) -> frame 0 and bit 3"""
    blob, G, dep = blob_scene
    poses = np.stack([G, G, G])
    e, st = V.vsd([blob], [0, 4, 0], poses, poses, dep[None], K, 0.015, TAUS, frame_idx=[0, 0, 5])
    assert list(st) == [0, 3, 8] and (e[0] == 0).all() and (e[1] == 1).all() and (e[2] == 0).all()


def test_capi_declares_dim_pose_error_vsd():
    from deepim_b200 import _capi
    assert len(_capi.SIGNATURES["dim_pose_error_vsd"][1]) == 18
