"""Generate tests/golden/ref_vsd.npz from the LIVE reference (runs only where /root/reference exists).

    python tests/golden/make_golden_vsd.py

Calls the reference's lib/utils/misc.py depth_im_to_dist_im and lib/utils/visibility.py estimate_visib_mask_gt / _est the
way a caller does (K a float32 array, delta a Python float) and stores their inputs and outputs.  Nothing from the
reference is copied.

Cases (render case r<k>_*): the observed depth is an oracle render of the C2 blob or the cube, mm-quantised, with
rectangular holes and an occluder (a plane 6 cm in front of the object over part of it); D_gt and D_est are oracle renders
at the true pose and at a pose 1 cm / 3 deg away.  Case 0 uses the float32-cast LINEMOD K, case 1 a second camera.
Boundary cases (b<k>_*): distance images built so that float32(dist_model) - float32(dist_test) is exactly float32(delta)
(row 0), and at about 1 m the nearest differences at or below it (row 1) and above it (row 2), for delta = 0.015 and
delta = 0.1 (float32(0.1) > 0.1: a difference of float32(0.1) is visible in float32, not in float64).
"""
import os
import sys

import numpy as np

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "mx-deepim_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

CAM2 = np.array([[1066.778, 0.0, 312.9869], [0.0, 1067.487, 241.3109], [0.0, 0.0, 1.0]], np.float32)


def import_reference():
    if not os.path.isdir(REF):
        raise SystemExit("reference not present; fixtures are committed, nothing to do")
    sys.path.insert(0, REF)
    from lib.utils import misc, visibility
    return misc.depth_im_to_dist_im, visibility.estimate_visib_mask_gt, visibility.estimate_visib_mask_est


def sensor(mesh, G, K, rng):
    """mm-quantised depth at G with three holes and an occluder 6 cm in front of the object"""
    from oracle import oracle as O
    from test_icp_oracle import mm
    d = mm(O.render(mesh, G, K, want=("depth",))["depth"])
    ys, xs = np.nonzero(d)
    y0, y1, x0, x1 = ys.min(), ys.max(), xs.min(), xs.max()
    for _ in range(3):
        k = rng.integers(len(ys))
        d[max(ys[k] - 3, 0):ys[k] + 3, max(xs[k] - 4, 0):xs[k] + 4] = 0.0
    occ = np.zeros_like(d, bool)
    occ[y0 - 4:(y0 + y1) // 2, x0 - 4:(x0 + x1) // 2] = True
    d[occ] = np.float32(float(G[2, 3]) - 0.06)
    return d


def main():
    dist_im, visib_gt, visib_est = import_reference()
    from oracle import oracle as O
    from deepim_b200 import synth
    from test_icp_oracle import perturb
    out = {}
    rng = np.random.default_rng(11)
    meshes = [synth.make_blob(), synth.make_cube()]
    for k, (mesh, K) in enumerate(zip(meshes, (synth.K_LINEMOD.astype(np.float32), CAM2))):
        G = synth.sample_pose_pairs(1, 20 + k)[0][0]
        G[2, 3] += (0.4, 1.2)[k]  # farther away: a smaller fixture
        E = perturb(G, rng)
        d_test = sensor(mesh, G, K, rng)
        d_gt = O.render(mesh, G, K, want=("depth",))["depth"]
        d_est = O.render(mesh, E, K, want=("depth",))["depth"]
        t, g, e = dist_im(d_test, K), dist_im(d_gt, K), dist_im(d_est, K)
        vg = visib_gt(t, g, 0.015)
        ve = visib_est(t, e, vg, 0.015)
        out.update({"r%d_K" % k: K, "r%d_depth_test" % k: d_test, "r%d_depth_gt" % k: d_gt, "r%d_depth_est" % k: d_est,
                    "r%d_pose_gt" % k: G, "r%d_pose_est" % k: E, "r%d_dist_test" % k: t, "r%d_dist_gt" % k: g,
                    "r%d_dist_est" % k: e, "r%d_visib_gt" % k: vg, "r%d_visib_est" % k: ve})
    for k, delta in enumerate((0.015, 0.1)):
        dl = np.float32(delta)
        # row 0: float32(delta) = N 2^-e with 2^23 <= N < 2^24; distances n 2^-e with n + N < 2^24 make the float32 sum and
        # difference exact (a few centimetres at most).  Rows 1, 2: distances around 1 m, where no difference equals
        # float32(delta): the largest one <= float32(delta) and the smallest one above it.
        mant, ex = np.frexp(dl)
        N = int(mant * 2 ** 24)
        scale = np.float32(2.0 ** (int(ex) - 24))
        t0 = rng.integers(1, 2 ** 24 - N, 64).astype(np.float32) * scale
        m0 = t0 + dl
        assert ((m0 - t0) == dl).all()
        t1 = rng.uniform(0.5, 1.5, (2, 64)).astype(np.float32)
        r = t1 + dl
        above = (r - t1) > dl
        lo = np.where(above, np.nextafter(r, np.float32(0)), r)
        hi = np.where(above, r, np.nextafter(r, np.float32(9)))
        assert ((lo[0] - t1[0]) <= dl).all() and ((hi[1] - t1[1]) > dl).all()
        t32, m32 = np.stack([t0, t1[0], t1[1]]), np.stack([m0, lo[0], hi[1]])
        t, m = t32.astype(np.float64), m32.astype(np.float64)
        t[:, :4] = 0.0  # holes
        m[:, 4:8] = 0.0  # no model
        gt = m[::-1].copy()
        vg = visib_gt(t, gt, delta)
        ve = visib_est(t, m, vg, delta)
        out.update({"b%d_delta" % k: np.float64(delta), "b%d_dist_test" % k: t, "b%d_dist_gt" % k: gt,
                    "b%d_dist_est" % k: m, "b%d_visib_gt" % k: vg, "b%d_visib_est" % k: ve})
    path = os.path.join(HERE, "ref_vsd.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
