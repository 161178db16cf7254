"""GPU: vertex-coloured meshes (dim_mesh_upload_colours).  dim_render (both truncation paths), dim_render_lit and
dim_render_dataset on the rasteriser's test scenes with vertex colours, bit for bit against the CPU checker
(tests/colour_oracle.c) and against the float64 ray caster; batches mixing textured and coloured classes; re-uploads that
switch a class's colour source; the refinement loop (every network, lighting, precision, frame map and per-frame cameras,
graphs, the host entry) and the train-time update on a coloured C2 blob against the oracle; PoseRefiner from binary PLY
files; and every refusal of the upload leaving the previous mesh in place."""

import numpy as np
import pytest
import torch

from deepim_b200 import _capi as capi
from deepim_b200 import lighting, lm6d_io, synth
from deepim_b200.context import Context
from oracle import oracle as O

import colour_oracle as CO
import colour_scenes as CS
import raster_ref as RR
import raster_scenes as RS

if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

pytestmark = pytest.mark.gpu
SCENES = RS.geometry_scenes() + RS.mesh_scenes() + [RS.batch16_scene()]
MEANS = synth.PIXEL_MEANS_RGB
MEANS32 = MEANS.astype(np.float32)
FACTOR = 1000.0
LIT_RATIO = np.float32(0.7)
K = synth.K_LINEMOD
N_ITER = 4
KEYS = ("poses", "se3", "zoom_factor", "bbox")


def dev(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else np.asarray(a, dtype))).cuda()


# ------------------------------------------------------------------------------------------------------- renders
@pytest.fixture(scope="module")
def contexts():
    cs = {}
    yield cs
    for c in cs.values():
        c.close()


def context(contexts, s):
    if s.view not in contexts:
        contexts[s.view] = Context(0, max_batch=16, height=s.H, width=s.W, max_classes=16, max_verts=60000,
                                   max_faces=120000)
    ctx = contexts[s.view]
    for k, m in enumerate(s.meshes):
        ctx.upload_mesh(k, m)
    return ctx


def render_all(ctx, s, b0, b1):
    cls, poses = dev(s.cls[b0:b1]), dev(np.stack([i[1] for i in s.inst[b0:b1]]))
    lpos = dev(np.stack([i[2] for i in s.inst[b0:b1]]))
    inten = dev(np.stack([i[3] for i in s.inst[b0:b1]]))
    ratio = dev(np.array([i[4] for i in s.inst[b0:b1]], np.float32))
    geo = dict(znear=s.zn, zfar=s.zf)
    out = {}
    for trunc in (True, False):
        out[trunc] = ctx.render(cls, poses, s.K, pixel_means_rgb=MEANS, trunc_u8=trunc,
                                want=("image", "depth", "mask", "bgr"), **geo)
    out["lit"] = ctx.render_lit(cls, poses, s.K, lpos, inten, LIT_RATIO, pixel_means_rgb=MEANS,
                                want=("image", "depth", "mask", "bgr"), **geo)
    out["ds"] = ctx.render_dataset(cls, poses, s.K, depth_factor=FACTOR, light_position=lpos, light_intensity=inten,
                                   brightness_ratio=ratio, want=("lit_bgr", "bgr", "depth", "label"), **geo)
    torch.cuda.synchronize()
    return {k: {n: t.cpu().numpy() for n, t in v.items() if t is not None} for k, v in out.items()}


def check_scene(ctx, s):
    rep = RR.Report(repr(s))
    geo = dict(zn=s.zn, zf=s.zf, H=s.H, W=s.W)
    for c0 in range(0, len(s.inst), 16):
        got = render_all(ctx, s, c0, min(c0 + 16, len(s.inst)))
        for k in range(len(got["lit"]["bgr"])):
            c, pose, lpos, inten, ratio = s.inst[c0 + k]
            m = s.meshes[c]
            ref = RR.Render(m, pose, s.K, s.H, s.W, s.zn, s.zf, m.normals)
            for t in (True, False):
                g = got[t]
                RR.check_render(rep, ref, g["depth"][k, 0], g["mask"][k, 0])
                CS.check_colours(rep, ref, g["bgr"][k], t)
                o = CO.render(m, pose, s.K, means_rgb=MEANS, trunc_u8=t, **geo)
                for n in ("bgr", "image"):
                    assert np.array_equal(g[n][k], o[n]), (repr(s), c0 + k, t, n)
                assert np.array_equal(g["depth"][k, 0], o["depth"]) and np.array_equal(g["mask"][k, 0], o["mask"])
                assert np.array_equal(g["bbox"][k], o["bbox"])
            g = got["lit"]
            RR.check_render(rep, ref, g["depth"][k, 0], g["mask"][k, 0])
            CS.check_lit_colours(rep, ref, g["bgr"][k], lpos, inten, LIT_RATIO, "modelnet")
            o = CO.render_lit(m, m.normals, pose, s.K, lpos, inten, LIT_RATIO, means_rgb=MEANS, **geo)
            for n in ("bgr", "image", "bbox"):
                assert np.array_equal(g[n][k], o[n]), (repr(s), c0 + k, "lit", n)
            g = got["ds"]
            CS.check_lit_colours(rep, ref, g["lit_bgr"][k], lpos, inten, ratio, "py_light")
            CS.check_colours(rep, ref, g["bgr"][k], True)
            RR.check_u16(rep, ref, g["depth"][k], g["label"][k], FACTOR)
            assert np.array_equal(g["bgr"][k], got[True]["bgr"][k].astype(np.uint8))  # (uint8)(c * 255) both ways
            o = CO.render_dataset(m, pose, s.K, lpos, inten, ratio, depth_factor=FACTOR, **geo)
            for n in ("lit_bgr", "bgr", "depth", "label"):
                assert np.array_equal(g[n][k], o[n]), (repr(s), c0 + k, "dataset", n)
    return rep


@pytest.mark.parametrize("s", SCENES, ids=repr)
def test_coloured_renders_against_float64_and_oracle(contexts, s):
    s = CS.coloured_scene(s)
    rep = check_scene(context(contexts, s), s)
    print(rep)
    assert rep.ok, str(rep)


@pytest.fixture(scope="module")
def kinds():
    """classes 0, 1: the textured cube and C2 blob; 2, 3: the same geometry with vertex colours"""
    ms = RS.meshes()
    tex = [ms["cube"], ms["c2"]]
    return tex + [CS.coloured(m, k) for k, m in enumerate(tex)]


def renders(ctx, cls, poses):
    args = (dev(np.asarray(cls, np.int32)), dev(poses), K)
    lp = np.stack([O.light_position(p) for p in poses])
    inten = np.tile(np.float32([1.1, 0.9, 1.0]), (len(cls), 1))
    out = {t: ctx.render(*args, pixel_means_rgb=MEANS, trunc_u8=t, want=("image", "depth", "mask", "bgr")) for t in (0, 1)}
    out["lit"] = ctx.render_lit(*args, dev(lp), dev(inten), 0.7, pixel_means_rgb=MEANS, want=("image", "bgr"))
    out["ds"] = ctx.render_dataset(*args, light_position=dev(lp), light_intensity=dev(inten),
                                   brightness_ratio=dev(np.full(len(cls), 0.6, np.float32)), want=("lit_bgr", "bgr", "depth"))
    torch.cuda.synchronize()
    return {(k, n): t.cpu().numpy() for k, v in out.items() for n, t in v.items() if t is not None}


def test_mixed_batch_equals_single_kind_batches(kinds):
    poses = synth.sample_pose_pairs(8, 21)[0].astype(np.float32)
    cls = np.array([0, 2, 1, 3, 2, 0, 3, 1])
    ctx = Context(0, max_batch=8, max_classes=4, max_verts=6000, max_faces=11000)
    fresh = Context(0, max_batch=8, max_classes=4, max_verts=6000, max_faces=11000)
    try:
        for k, m in enumerate(kinds):
            ctx.upload_mesh(k, m)
        for k, m in enumerate(kinds[:2]):
            fresh.upload_mesh(k, m)
        mixed = renders(ctx, cls, poses)
        tex, col = cls < 2, cls >= 2
        a = renders(ctx, cls[tex], poses[tex])
        b = renders(ctx, cls[col], poses[col])
        c = renders(fresh, cls[tex], poses[tex])
        for key, v in mixed.items():
            assert np.array_equal(v[tex], a[key]), key
            assert np.array_equal(v[col], b[key]), key
            assert np.array_equal(v[tex], c[key]), key
        assert (mixed[(1, "mask")].reshape(8, -1).sum(1) > 100).all()
    finally:
        ctx.close()
        fresh.close()


def test_reupload_switches_the_colour_source(kinds):
    pose = synth.sample_pose_pairs(1, 4)[0][0].astype(np.float32)
    ctx = Context(0, max_batch=1, max_classes=1, max_verts=6000, max_faces=11000)
    try:
        for m, ref in ((kinds[1], O.render), (kinds[3], CO.render), (kinds[1], O.render), (kinds[3], CO.render)):
            ctx.upload_mesh(0, m)
            got = ctx.render(dev(np.zeros(1, np.int32)), dev(pose[None]), K, pixel_means_rgb=MEANS, want=("image", "bgr"))
            want = ref(m, pose, K, means_rgb=MEANS)
            assert np.array_equal(got["bgr"][0].cpu().numpy(), want["bgr"])
            assert np.array_equal(got["image"][0].cpu().numpy(), want["image"])
            assert np.array_equal(got["bbox"][0].cpu().numpy(), want["bbox"])
    finally:
        ctx.close()


def test_refused_uploads_leave_the_previous_mesh(kinds):
    m = kinds[3]
    pose = synth.sample_pose_pairs(1, 6)[0][0].astype(np.float32)
    ctx = Context(0, max_batch=1, max_classes=2, max_verts=len(m.verts), max_faces=len(m.faces))
    try:
        ctx.upload_mesh(0, m)
        before = ctx.render(dev(np.zeros(1, np.int32)), dev(pose[None]), K, want=("bgr", "depth"))
        before = {k: v.cpu().numpy() for k, v in before.items() if v is not None}
        v, f, c = m.verts, m.faces, m.colours

        def call(cls, verts, cols, faces):
            verts, cols, faces = [np.ascontiguousarray(a) for a in (verts, cols, faces)]
            return capi.lib.dim_mesh_upload_colours(ctx._h, cls, verts.ctypes.data, cols.ctypes.data, len(verts),
                                                     faces.ctypes.data, len(faces))

        bad_c = {}
        for name, val in (("nan", np.nan), ("inf", np.inf), ("above", 1.0001), ("below", -1e-6)):
            cc = c.copy()
            cc[17, 1] = val
            bad_c[name] = cc
        big = np.concatenate([v, v[:1]])
        cases = [("class", (2, v, c, f)), ("class", (-1, v, c, f)), ("verts", (0, big, np.concatenate([c, c[:1]]), f)),
                 ("faces", (0, v, c, np.concatenate([f, f]))), ("index", (0, v, c, np.where(f == 5, len(v), f))),
                 ("index", (0, v, c, np.where(f == 5, -1, f)))] + [("colour " + k, (0, v, cc, f)) for k, cc in bad_c.items()]
        for what, args in cases:
            assert call(*args) != 0, what
            err = capi.lib.dim_last_error().decode()
            if what.startswith("colour"):
                assert "vertex 17" in err, err
            after = ctx.render(dev(np.zeros(1, np.int32)), dev(pose[None]), K, want=("bgr", "depth"))
            for k in ("bgr", "depth", "bbox"):
                assert np.array_equal(after[k].cpu().numpy(), before[k]), (what, k)
        assert call(0, v, c, f) == 0
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------- refinement and training
@pytest.fixture(scope="module")
def blob():
    m = synth.make_blob()
    m.normals = synth.vertex_normals(m)
    c = CS.coloured(m, 7)
    return c


def make_case(blob, B=4, seed=51, K_of=None):
    obs, ini = synth.sample_pose_pairs(B, seed)
    u8 = []
    for b in range(B):
        r = CO.render(blob, obs[b], K if K_of is None else K_of[b], means_rgb=MEANS)
        u8.append(synth.composite_observed(r["bgr"], r["mask"], b))
    u8 = np.stack(u8)
    img = np.stack([synth.transform_image(u8[b]) for b in range(B)])
    depth = np.stack([CO.render(blob, obs[b], K, want=("depth",))["depth"] for b in range(B)])[:, None].astype(np.float32)
    return dict(B=B, obs=obs, ini=ini, cls=np.zeros(B, np.int32), u8=u8, img=img, depth=depth)


def make_ctx(blob, weights, B=4, **kw):
    c = Context(0, max_batch=B, max_classes=1, max_verts=6000, max_faces=11000, **kw)
    c.upload_mesh(0, blob)
    c.load_weights(weights)
    return c


def check_teacher_forced(res, ref, prec=capi.PREC_FP16):
    rtol, ttol = (1e-4, 1e-3) if prec != capi.PREC_BF16 else (5e-3, 1e-2)
    assert np.array_equal(res["bbox"].cpu().numpy(), ref["bbox"])
    assert np.array_equal(res["zoom_factor"].cpu().numpy(), ref["zoom_factor"])
    se3 = res["se3"].cpu().numpy()
    assert np.abs(se3[..., :4] - ref["se3"][..., :4]).max() < rtol
    assert np.abs(se3[..., 4:] - ref["se3"][..., 4:]).max() < ttol


def override(case, ref):
    return dev(np.concatenate([case["ini"][None], ref["poses"][:N_ITER - 1]], 0))


VARIANTS = ["unlit", "lit", "rgbd", "image_only"]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("prec", [capi.PREC_FP16, capi.PREC_BF16, capi.PREC_BF16X3], ids=["fp16", "bf16", "bf16x3"])
def test_refine_teacher_forced_against_oracle(blob, variant, prec):
    if variant == "image_only":
        w, kw = synth.make_train_weights(0, input_mask=False), {"input_mask": False}
    elif variant == "rgbd":
        w, kw = synth.make_weights(0, input_depth=True), {"input_depth": True}
    else:
        w, kw = synth.make_weights(0), {}
    c = make_case(blob)
    inten = lighting.sample_intensity(np.random.default_rng(11), (N_ITER, c["B"]))
    lit = {"intensity": inten, "offset": lighting.OFFSET, "brightness_ratio": 0.7} if variant == "lit" else None
    depth = c["depth"] if variant == "rgbd" else None
    with CO.dispatching():
        ref = O.refine(w, [blob], c["cls"], c["img"], c["ini"], K, N_ITER, MEANS32, lighting=lit, depth_observed=depth,
                       input_mask=variant != "image_only")
    ctx = make_ctx(blob, w, **kw)
    try:
        dlit = None if lit is None else dict(lit, intensity=dev(inten))
        ddepth = None if depth is None else dev(depth)
        res = ctx.refine(dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER, pixel_means_rgb=MEANS, precision=prec,
                         pose_override=override(c, ref), lighting=dlit, depth_observed=ddepth)
        check_teacher_forced(res, ref, prec)
        assert not ctx.refine_status(c["B"], N_ITER).numpy().any()
    finally:
        ctx.close()


def test_refine_frames_with_per_frame_cameras_against_oracle(blob):
    """two frames seen by two cameras, instances mapped to them crosswise: each camera's sub-batch against the oracle"""
    cams = [K, np.array([[600.0, 0, 330.5], [0, 590.0, 250.2], [0, 0, 1]], np.float32)]
    idx = np.array([0, 1, 1, 0], np.int32)
    c = make_case(blob, K_of=[cams[i] for i in idx])
    frames = c["img"][[0, 1]]
    inst_img = frames[idx]  # instance b observes frame idx[b]
    w = synth.make_weights(0)
    refs = {}
    with CO.dispatching():
        for k in (0, 1):
            s = idx == k
            refs[k] = O.refine(w, [blob], c["cls"][s], inst_img[s], c["ini"][s], cams[k], N_ITER, MEANS32)
    ref = {n: np.zeros((N_ITER, c["B"]) + refs[0][n].shape[2:], refs[0][n].dtype) for n in KEYS}
    for k in (0, 1):
        for n in KEYS:
            ref[n][:, idx == k] = refs[k][n]
    ctx = make_ctx(blob, w)
    try:
        res = ctx.refine_frames(dev(frames), dev(idx), dev(c["cls"]), dev(c["ini"]), dev(np.stack([cams[i] for i in (0, 1)])),
                                N_ITER, pixel_means_rgb=MEANS, pose_override=override(c, ref))
        check_teacher_forced(res, ref)
    finally:
        ctx.close()


def test_graph_replay_and_host_entry_equal_the_eager_device_run(blob):
    from deepim_b200._capi import check, lib
    w = synth.make_weights(0)
    c = make_case(blob)
    ctx = make_ctx(blob, w)
    try:
        args = (dev(c["img"]), dev(c["cls"]), dev(c["ini"]), K, N_ITER)
        check(lib.dim_debug_set_option(ctx._h, b"graph", 0))
        eager = {k: v.clone() for k, v in ctx.refine(*args, pixel_means_rgb=MEANS).items()}
        torch.cuda.synchronize()
        check(lib.dim_debug_set_option(ctx._h, b"graph", 1))
        out = None
        for _ in range(3):  # warm-up, capture + launch, replay
            out = ctx.refine(*args, pixel_means_rgb=MEANS, out=out)
            torch.cuda.synchronize()
            for k in KEYS:
                assert torch.equal(out[k], eager[k]), k
        poses, se3 = ctx.refine_host(c["u8"], c["cls"], c["ini"], K, N_ITER, pixel_means_rgb=MEANS)
        d = ctx.refine(*args, pixel_means_rgb=MEANS)
        assert np.array_equal(poses, d["poses"].cpu().numpy())
        assert np.array_equal(se3, d["se3"].cpu().numpy())
    finally:
        ctx.close()


def test_train_update_on_a_coloured_mesh_against_oracle(blob):
    w = synth.make_weights(0)
    c = make_case(blob)
    B = c["B"]
    rng = np.random.default_rng(5)
    rot = rng.normal(0, 0.02, (B, 4)).astype(np.float32)
    rot[:, 0] = 1.0
    rot /= np.linalg.norm(rot, axis=1, keepdims=True)
    trans = rng.normal(0, 0.01, (B, 3)).astype(np.float32)
    src = c["ini"].astype(np.float32)
    tgt = c["obs"].astype(np.float32)
    with CO.dispatching():
        ref = O.train_update([blob], c["cls"], src, rot, trans, tgt, c["depth"], K, MEANS)
    ctx = make_ctx(blob, w)
    try:
        got = ctx.train_update(dev(c["cls"]), dev(src), dev(rot), dev(trans), dev(tgt), dev(c["depth"]), K,
                               pixel_means_rgb=MEANS)
        torch.cuda.synchronize()
        for k in ("image_rendered", "depth_rendered", "mask_rendered"):
            assert np.array_equal(got[k].cpu().numpy(), ref[k]), k
        assert (ref["mask_rendered"].reshape(B, -1).sum(1) > 100).all()
    finally:
        ctx.close()


def test_pose_refiner_from_binary_ply_files(tmp_path, blob):
    from deepim_b200.refiner import PoseRefiner
    cube = synth.make_cube()
    paths = []
    for k, m in enumerate((blob, cube)):
        col = np.clip(np.rint((m.colours if m.colours is not None else np.full((len(m.verts), 3), 0.3)) * 255), 0, 255)
        head = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face %d\n"
                "property list uchar int vertex_indices\nend_header\n" % (len(m.verts), len(m.faces))).encode()
        vdt = np.dtype([("p", "<f4", 3), ("c", "u1", 3)])
        vs = np.zeros(len(m.verts), vdt)
        vs["p"], vs["c"] = m.verts, col
        fdt = np.dtype([("n", "u1"), ("i", "<i4", 3)])
        fs = np.zeros(len(m.faces), fdt)
        fs["n"], fs["i"] = 3, m.faces
        p = tmp_path / ("obj_%06d.ply" % (k + 1))
        p.write_bytes(head + vs.tobytes() + fs.tobytes())
        paths.append(str(p))
    meshes = [lm6d_io.load_ply(p) for p in paths]
    assert all(m.colours is not None and m.tex is None for m in meshes)
    w = synth.make_weights(0)
    obs, ini = synth.sample_pose_pairs(2, 9)
    cls = np.array([0, 1], np.int32)
    u8 = []
    for b in range(2):
        r = CO.render(meshes[cls[b]], obs[b], K)
        u8.append(synth.composite_observed(r["bgr"], r["mask"], b))
    u8 = np.stack(u8)
    img = np.stack([synth.transform_image(u) for u in u8])
    r = PoseRefiner(meshes, w, K=K, max_batch=2, n_iter=N_ITER)
    try:
        poses = np.asarray(r.refine(u8, cls, ini))
    finally:
        r.close()
    with CO.dispatching():
        ref = O.refine(w, meshes, cls, img, ini, K, N_ITER, MEANS32)
    assert poses.shape == ref["poses"].shape
    assert np.abs(poses - ref["poses"]).max() < 1e-3
