"""GPU: the pose algebra of geom.cu against the float64 reference of tests/pose_ref.py, over the whole rotation group
(identity, 1e-9 ... 1e-3 rad, uniform rotations, exact and near half-turns), every rot_coord, a trivial and a non-trivial
(T_means, T_stds), and batches that cross each kernel's block:
  se3_compose_kernel (dim_se3_compose, 64-thread blocks)      B = 1, 63, 64, 65, 130
  train_pose_kernel (dim_train_update, 32-thread blocks)      B = 1, 31, 32, 33, 65: refined pose, rotation label (the
                                                              Jacobi solver), translation label, KT, the lit light
  transform3d_fwd / bwd_kernel, CAMERA_NEW and the others     N = 3000 and 257 (one past the backward's 256-thread block)
and fit_batch under a non-default configuration: its re-render composes under the context's trans_means / trans_stds /
rot_coord.

Bounds (derived, not fitted; U = 2^-24, ulp64 = 2^-52, S = the magnitude each pose_ref function returns):
  compose (float64 both sides)     |dev - ref| <= 4 ulp64 S
  refined pose (float32 store)     |dev - ref| <= 1 float32 ulp of float32(ref) + 4 ulp64 S (a double-rounding tie)
  rotation label                   | |q| - 1 | <= 4 U;  |quat2mat(q) - R_delta|max <= 8 U + 1e-15;
                                   |q - q_ref| <= 4 U |q_ref| + 16 ulp64 (q_ref from scipy; +-q_ref where |w_ref| <= 1e-6);
                                   w >= 0.  The absolute term is the float64 solvers' noise on a component that is zero, a
                                   half-turn's w: observed 2.2e-15 = 10 ulp64 (pi about x, MODEL) on an H100 80GB HBM3
  translation label                |dev - ref| <= 2 U S + 2e-15 / |T_stds|
  KT                               |dev - ref| <= 8 U S
  Transform3D                      tests/kernel_ref.py's bound, rho = 0, kappa as test_gpu_train_heads.py's transform3d"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

import kernel_ref as R  # noqa: E402
import pose_ref as P  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402

K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
NAMES, QSET = P.rotation_set()
NORMS = {"trivial": ((0.0, 0.0, 0.0), (1.0, 1.0, 1.0)), "scaled": ((0.0625, -0.125, 0.03125), (0.5, 2.0, 0.75))}
KAPPA_T3D = 8.8  # test_gpu_train_heads.py's "transform3d" family: 4 x its observed 2.199 on an H100 80GB HBM3 at 400 W


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def ctx():
    """geometry only: a 64 x 80 frame, no network, one cube with normals (for the lit re-render)"""
    c = Context(0, max_batch=130, height=64, width=80, max_classes=1, max_verts=2000, max_faces=4000)
    cube = synth.make_cube()
    c.upload_mesh(0, cube)
    c.upload_normals(0, synth.vertex_normals(cube))
    yield c
    c.close()


def rotations(B, start):
    """B deltas of the rotation set, cycling from index start, and their names"""
    idx = (start + np.arange(B)) % len(QSET)
    return QSET[idx], [NAMES[i] for i in idx]


def assert_within(what, err, allow, names=None):
    bad = err > allow
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err / np.maximum(allow, 1e-300), 0)), err.shape)
        raise AssertionError("%s: %d entries out of bound; worst at %s%s: err %.3g allow %.3g"
                             % (what, int(bad.sum()), i, " (%s)" % names[i[0]] if names else "", err[i], allow[i]))


def check_f32_rounding(what, dev32, ref64, S, names):
    """dev32 is float32(ref64) to one float32 ulp (ties of the float64 value)"""
    r32 = ref64.astype(np.float32)
    assert_within(what, np.abs(dev32.astype(np.float64) - r32), np.spacing(np.abs(r32)).astype(np.float64)
                  + 4 * P.ULP64 * S, names)


# ---------------------------------------------------------------------------------------------------- compose
@pytest.mark.parametrize("norm", sorted(NORMS))
@pytest.mark.parametrize("coord", P.COORDS)
def test_se3_compose_against_float64(ctx, coord, norm):
    Tm, Ts = NORMS[norm]
    rng = np.random.default_rng(11)
    start = 0
    for B in (1, 63, 64, 65, 130):
        q, names = rotations(B, start)
        start += B
        src = P.random_poses(B, 100 + B)
        t = (rng.normal(size=(B, 3)) * [0.05, 0.05, 0.2]).astype(np.float32)
        se3 = np.concatenate([q.astype(np.float32), t], 1)
        out = ctx.se3_compose(dev(src), dev(se3), Tm, Ts, coord).cpu().numpy()
        ref, S = P.rt_transform(src, se3[:, :4], t, Tm, Ts, coord)
        assert_within("B=%d compose" % B, np.abs(out - ref), 4 * P.ULP64 * S, names)
        for scale in (1e-3, 1e3):  # the quaternion is normalised before use
            s = se3.copy()
            s[:, :4] = (se3[:, :4] * scale).astype(np.float32)
            o = ctx.se3_compose(dev(src), dev(s), Tm, Ts, coord).cpu().numpy()
            ref_s, S_s = P.rt_transform(src, s[:, :4], t, Tm, Ts, coord)
            assert_within("B=%d compose, rot x %g" % (B, scale), np.abs(o - ref_s), 4 * P.ULP64 * S_s, names)
        s = se3.copy()
        s[:, :4] *= -1  # -q is the same rotation, and normalising and squaring it is exact
        assert np.array_equal(ctx.se3_compose(dev(src), dev(s), Tm, Ts, coord).cpu().numpy(), out), "B=%d -q" % B


# ----------------------------------------------------------------------------------------------- train update
def update_case(B, start, coord, norm, seed):
    """src, rot_est, trans_est, tgt (float32) such that the label's rotation delta is the rotation set's element; rot_est is
    the identity on even instances and a random small rotation on odd ones"""
    Tm, Ts = NORMS[norm]
    rng = np.random.default_rng(seed)
    q, names = rotations(B, start)
    src32 = P.random_poses(B, seed).astype(np.float32)
    rot = np.tile(np.float32([1, 0, 0, 0]), (B, 1))
    rot[1::2] = (np.array([1.0, 0, 0, 0]) + rng.normal(size=(B // 2, 4)) * 0.1).astype(np.float32)
    tr = (rng.normal(size=(B, 3)) * 0.05).astype(np.float32)
    refined, S = P.rt_transform(src32.astype(np.float64), rot, tr, Tm, Ts, coord)
    td = rng.normal(size=(B, 3)) * [0.05, 0.05, 0.2]
    tgt32 = P.rt_transform(refined, q, td, Tm, Ts, coord)[0].astype(np.float32)
    return src32, rot, tr, tgt32, refined, S, names


def run_update(ctx, case, coord, norm, lighting=None):
    src32, rot, tr, tgt32 = case[:4]
    B = len(src32)
    Tm, Ts = NORMS[norm]
    out = ctx.train_update(dev(np.zeros(B, np.int32)), dev(src32), dev(rot), dev(tr), dev(tgt32), None, K,
                           pixel_means_rgb=MEANS, T_means=Tm, T_stds=Ts, rot_coord=coord, want_flow=False, lighting=lighting)
    kt, light = ctx.debug_train_update(B)
    return {k: v.cpu().numpy() for k, v in out.items() if v is not None}, kt, light


def check_update(out, kt_dev, case, coord, norm, B):
    tgt32, refined, S, names = case[3:]
    Tm, Ts = NORMS[norm]
    check_f32_rounding("B=%d refined pose" % B, out["src_pose"], refined, S, names)
    Rd, tl, St = P.calc_rt_delta(refined, tgt32, Tm, Ts, coord)
    q = out["rot"].astype(np.float64)
    assert_within("B=%d |q| - 1" % B, np.abs(np.linalg.norm(q, axis=1) - 1), np.full(B, 4 * P.U32), names)
    assert_within("B=%d quat2mat(q) - R_delta" % B, np.abs(P.quat2mat(q) - Rd), np.full(Rd.shape, 8 * P.U32 + 1e-15), names)
    qr = P.mat2quat(Rd)
    half = (np.abs(qr[:, 0]) <= 1e-6) & ((q * qr).sum(1) < 0)
    qr[half] *= -1
    assert_within("B=%d rotation label vs scipy" % B, np.abs(q - qr), 4 * P.U32 * np.abs(qr) + 16 * P.ULP64, names)
    assert (q[:, 0] >= 0).all(), "B=%d: a rotation label with w < 0: %s" % (B, [names[n] for n in np.nonzero(q[:, 0] < 0)[0]])
    assert_within("B=%d translation label" % B, np.abs(out["trans"] - tl), 2 * P.U32 * St + 2e-15 / np.abs(Ts), names)
    ref_kt, Sk = P.kt(K, refined, tgt32)
    assert_within("B=%d KT" % B, np.abs(kt_dev - ref_kt), 8 * P.U32 * Sk, names)


@pytest.mark.parametrize("norm", sorted(NORMS))
@pytest.mark.parametrize("coord", P.COORDS)
def test_train_update_against_float64(ctx, coord, norm):
    start = 0
    for B in (1, 31, 32, 33, 65):
        case = update_case(B, start, coord, norm, 200 + B)
        start += B
        out, kt, _ = run_update(ctx, case, coord, norm)
        check_update(out, kt, case, coord, norm, B)
    assert start >= len(QSET)  # every delta of the set was a label


@pytest.mark.parametrize("coord", P.COORDS)
def test_train_update_batch_split_is_bit_identical(ctx, coord):
    """one call of 65 instances and the same instances as 32 + 33: identical outputs, KT included"""
    case = update_case(65, 7, coord, "scaled", 300)
    whole, kt, _ = run_update(ctx, case, coord, "scaled")
    parts = [run_update(ctx, tuple(a[lo:hi] for a in case[:4]), coord, "scaled") for lo, hi in ((0, 32), (32, 65))]
    for k in whole:
        assert np.array_equal(whole[k], np.concatenate([p[0][k] for p in parts])), k
    assert np.array_equal(kt, np.concatenate([p[1] for p in parts]))


@pytest.mark.parametrize("coord", P.COORDS)
def test_train_update_light_follows_the_float64_refined_pose(ctx, coord):
    B, offset = 33, (0.0, 0.5, 0.5)
    case = update_case(B, 3, coord, "scaled", 400)
    inten = dev(np.ones((B, 3), np.float32))
    out, kt, light = run_update(ctx, case, coord, "scaled", {"intensity": inten, "offset": offset, "brightness_ratio": 0.7})
    check_update(out, kt, case, coord, "scaled", B)
    ref = P.light_position(offset, case[4])
    S = np.abs(np.asarray(offset)) + np.abs(case[4][:, :, 3]) + case[5][:, :, 3]
    check_f32_rounding("light position", light, ref, S, case[6])


# ------------------------------------------------------------------------------------------------ Transform3D
@pytest.mark.parametrize("N", [3000, 257])
@pytest.mark.parametrize("coord", P.COORDS)
def test_transform3d_against_float64(ctx, coord, N):
    rng = np.random.default_rng(N)
    B = 3
    T = lambda a: torch.from_numpy(np.asarray(a, np.float64)).cuda()
    for norm in sorted(NORMS):
        Tm, Ts = NORMS[norm]
        pts = (rng.normal(size=(B, 3, N)) * 0.05).astype(np.float32)
        q = QSET[rng.choice(len(QSET), B)]
        q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
        t = (rng.normal(size=(B, 3)) * 0.05).astype(np.float32)
        ps = P.random_poses(B, N).astype(np.float32)
        og = rng.normal(size=(B, 3, N)).astype(np.float32)
        out = ctx.transform3d(dev(pts), dev(q), dev(t), dev(ps), Tm, Ts, coord)
        ref, S = R.transform3d_fwd(T(pts), T(q), T(t), T(ps), Tm, Ts, coord)
        R.check("t3d_pose", "forward %s %s N=%d" % (coord, norm, N), out, ref, S, 0.0, KAPPA_T3D)
        rg, tg = ctx.transform3d_backward(dev(og), dev(pts), dev(q), dev(t), dev(ps), Tm, Ts, coord)
        (rref, Sr), (tref, St) = R.transform3d_bwd(T(og), T(pts), T(q), T(t), T(ps), Tm, Ts, coord)
        R.check("t3d_pose", "rotation gradient %s %s N=%d" % (coord, norm, N), rg, rref, Sr, 0.0, KAPPA_T3D)
        R.check("t3d_pose", "translation gradient %s %s N=%d" % (coord, norm, N), tg, tref, St, 0.0, KAPPA_T3D)
    print("Transform3D %s N=%d: observed kappa %.3f" % (coord, N, R.OBSERVED["t3d_pose"]))


# ------------------------------------------------------------------------------------------------- fit_batch
def test_fit_batch_re_renders_under_the_context_config():
    """Trainer(config = MODEL, non-zero trans_means, non-unit trans_stds): inner iteration 2 trains on src_pose =
    float32(RT_transform(src, rot_est_norm, trans_est)) under that configuration -- the one the step's Transform3D used --
    and on the render of exactly that pose"""
    from deepim_b200.trainer import Trainer, fit_batch, make_device_batch
    B = 2
    meshes = [synth.make_cube(), synth.make_blob()]
    tctx = Context(0, max_batch=B, max_classes=2, max_verts=6000, max_faces=11000)
    try:
        for i, m in enumerate(meshes):
            tctx.upload_mesh(i, m)
        Tm, Ts = NORMS["scaled"]
        tr = Trainer(tctx, synth.make_train_weights(0), config={"rot_coord": "MODEL", "trans_means": Tm, "trans_stds": Ts})
        batch, cls, tgt, depth_gt = make_device_batch(tctx, meshes, B, 11, K, MEANS)
        steps, updates, fronts = [], [], []
        step, update, front = tr.step, tctx.train_update, tr.zoom_front
        tr.step = lambda z, **kw: steps.append(step(z, **kw)) or steps[-1]
        tctx.train_update = lambda *a, **kw: updates.append(update(*a, **kw)) or updates[-1]
        tr.zoom_front = lambda b, KK: fronts.append(b["src_pose"].clone()) or front(b, KK)
        fit_batch(tr, batch, cls, tgt, depth_gt, K, n_inner=2)
        torch.cuda.synchronize()
        assert len(steps) == 2 and len(updates) == 1 and len(fronts) == 2
        src = batch["src_pose"].cpu().numpy().astype(np.float64)
        rot, trans = steps[0]["rot_est_norm"].cpu().numpy(), steps[0]["trans_est"].cpu().numpy()
        ref, S = P.rt_transform(src, rot, trans, Tm, Ts, "MODEL")
        second = fronts[1].cpu().numpy()
        check_f32_rounding("inner iteration 2 src_pose", second, ref, S, None)
        assert np.array_equal(second, updates[0]["src_pose"].cpu().numpy())
        r = tctx.render(cls, fronts[1], K, pixel_means_rgb=batch["pixel_means_rgb"], trunc_u8=False)
        assert r["mask"].sum() > 100
        for k in ("image", "depth", "mask"):
            assert torch.equal(r[k], updates[0][k + "_rendered"]), k
    finally:
        tctx.close()


def teardown_module():
    if "t3d_pose" in R.OBSERVED:
        print("\nTransform3D: largest kappa needed over every case %.3f (bound %g)" % (R.OBSERVED["t3d_pose"], KAPPA_T3D))
