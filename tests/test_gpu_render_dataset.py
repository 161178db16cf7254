"""GPU: dim_render_dataset (the data-preparation render of toolkit/LM6d_ds_1 ... ds_4 and LM6d_0) bit for bit against the
CPU oracle, against dim_render / dim_render_lit where the formulas meet, its refusals, the Render_Py_Light stand-in, and
toolkit.gen_syn_set end to end."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from deepim_b200 import _capi as capi
from deepim_b200 import augment, lm6d_io, synth, toolkit
from deepim_b200.context import Context
from deepim_b200.render_py_light import Render_Py_Light
from oracle import oracle as O

import py_light_oracle as PL

pytestmark = pytest.mark.gpu
K = toolkit.K_LM.astype(np.float32)
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_syn.npz"))


def dev(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else np.asarray(a, dtype))).cuda()


@pytest.fixture(scope="module")
def meshes():
    ms = [synth.make_cube(), synth.make_blob(nlat=24, nlon=48, tex_size=128)]
    for m in ms:
        m.normals = synth.vertex_normals(m)
    return ms


@pytest.fixture(scope="module")
def ctx(meshes):
    c = Context(0, max_batch=16, max_classes=2, max_verts=20000, max_faces=40000)
    for i, m in enumerate(meshes):
        c.upload_mesh(i, m)
    yield c
    c.close()


def scene(B=16, seed=3):
    """two classes, every ratio and light colour (zero channels included), objects cut by each border, one out of view,
    one straddling the near plane"""
    rs = np.random.RandomState(seed)
    cls = (np.arange(B) % 2).astype(np.int32)
    poses = np.zeros((B, 3, 4), np.float64)
    shifts = [(0, 0, 0.7), (-0.43, 0, 0.7), (0.43, 0, 0.7), (0, -0.3, 0.7), (0, 0.3, 0.7), (3.0, 0, 0.7), (0, 0, 0.27)]
    for b in range(B):
        poses[b, :, :3] = synth.random_rotation(rs)
        poses[b, :, 3] = shifts[b] if b < len(shifts) else (rs.normal(0, 0.05), rs.normal(0, 0.05), 0.6 + rs.rand() * 0.4)
    ratio = np.array([toolkit.BRIGHTNESS_RATIOS[b % 5] for b in range(B)], np.float32)
    inten = (toolkit.LIGHT_COLOURS[np.arange(B) % 7] * rs.uniform(0.9, 1.1, (B, 3))).astype(np.float32)
    lpos = np.stack([O.light_position(poses[b], np.array(toolkit.LIGHT_OFFSETS[b % 6]) * 0.5) for b in range(B)])
    return cls, poses.astype(np.float32), lpos.astype(np.float32), inten, ratio


def run(ctx, cls, poses, lpos, inten, ratio):
    return {k: v.cpu().numpy() for k, v in ctx.render_dataset(
        dev(cls), dev(poses), K, light_position=dev(lpos), light_intensity=dev(inten), brightness_ratio=dev(ratio),
        want=("lit_bgr", "bgr", "depth", "label")).items()}


@pytest.mark.parametrize("B", [16, 1])
def test_render_dataset_bit_exact_against_the_oracle(ctx, meshes, B):
    sc = scene()
    sc = tuple(a[:B] for a in sc) if B == 1 else sc
    got = run(ctx, *sc)
    cls, poses, lpos, inten, ratio = sc
    for b in range(B):
        ref = PL.render_dataset(meshes[cls[b]], poses[b], K, lpos[b], inten[b], ratio[b])
        for k in ("lit_bgr", "bgr", "depth", "label"):
            assert np.array_equal(got[k][b], ref[k]), (b, k, int((got[k][b] != ref[k]).sum()))
    if B == 16:
        assert not got["label"][5].any() and not got["lit_bgr"][5].any() and not got["depth"][5].any()  # out of view
        for b in range(1, 5):  # cut by a border: covered pixels on the image edge
            edge = np.concatenate([got["label"][b][:, 0], got["label"][b][:, -1], got["label"][b][0], got["label"][b][-1]])
            assert edge.any(), b
        assert got["label"][6].any() and (got["depth"][6][got["label"][6] > 0] >= 250).all()  # clipped at znear
        assert {tuple(c) for c in toolkit.LIGHT_COLOURS[np.arange(16) % 7]} == {tuple(c) for c in toolkit.LIGHT_COLOURS}


def test_unlit_half_equals_dim_render(ctx):
    cls, poses, *_ = scene()
    got = ctx.render_dataset(dev(cls), dev(poses), K, want=("bgr", "depth", "label"))
    ref = ctx.render(dev(cls), dev(poses), K, trunc_u8=False, want=("bgr", "depth"))
    depth = ref["depth"].cpu().numpy()[:, 0]
    assert np.array_equal(got["bgr"].cpu().numpy(), ref["bgr"].cpu().numpy().astype(np.uint8))
    assert np.array_equal(got["depth"].cpu().numpy(), (depth * np.float32(1000.0)).astype(np.uint16))
    assert np.array_equal(got["label"].cpu().numpy(), (depth != 0).astype(np.uint8))


def test_lit_half_at_white_light_equals_dim_render_lit(ctx):
    cls, poses, lpos, _, _ = scene()
    white = np.ones((16, 3), np.float32)
    for r in toolkit.BRIGHTNESS_RATIOS:
        got = run(ctx, cls, poses, lpos, white, np.full(16, r, np.float32))["lit_bgr"]
        ref = ctx.render_lit(dev(cls), dev(poses), K, dev(lpos), dev(white), r, want=("bgr",))["bgr"].cpu().numpy()
        assert np.array_equal(got, ref.astype(np.uint8)), r


def _raw(c, cls, poses, lp, li, ratio, lit, bgr):
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    rc = capi.lib.dim_render_dataset(c._h, p(cls), p(poses), len(poses), capi.farr(K.reshape(9), 9), 0.25, 6.0, 1000.0,
                                     p(lp), p(li), p(ratio), p(lit), p(bgr), None, None, None)
    torch.cuda.synchronize()
    return rc, capi.lib.dim_last_error().decode()


def test_refusals_leave_the_outputs_untouched(ctx):
    cls, poses, lpos, inten, ratio = (dev(a) for a in scene())
    lit = torch.full((16, 480, 640, 3), 0xAB, dtype=torch.uint8, device="cuda")
    bgr = lit.clone()
    rc, msg = _raw(ctx, cls, poses, None, inten, ratio, lit, bgr)
    assert rc != 0 and "light_position" in msg
    rc, msg = _raw(ctx, cls, poses, lpos, inten, None, lit, bgr)
    assert rc != 0 and "brightness_ratio" in msg
    rc, msg = _raw(ctx, cls, poses, lpos, inten, ratio, None, bgr)
    assert rc != 0 and "lit_bgr" in msg
    bare = Context(0, max_batch=16, max_classes=1)
    try:
        bare.upload_mesh(0, synth.make_cube())  # no normals
        rc, msg = _raw(bare, torch.zeros_like(cls), poses, lpos, inten, ratio, lit, bgr)
        assert rc != 0 and "normals" in msg
        with pytest.raises(ValueError):
            bare.render_dataset(torch.zeros_like(cls), poses, K, light_position=lpos, want=("bgr",))
    finally:
        bare.close()
    assert (lit == 0xAB).all() and (bgr == 0xAB).all()


def test_render_py_light_stand_in_equals_the_entry(ctx, meshes):
    cls, poses, lpos, inten, ratio = scene()
    rm = Render_Py_Light(meshes[1], K, brightness_ratios=toolkit.BRIGHTNESS_RATIOS, ctx=ctx, mesh_slot=1)
    got = run(ctx, np.ones(16, np.int32), poses, lpos, inten, ratio)
    for b in range(16):
        q = toolkit.mat2quat(poses[b, :, :3].astype(np.float64))
        R32 = toolkit.quat2mat(q).astype(np.float32)
        row = run(ctx, np.ones(1, np.int32), np.hstack([R32, poses[b, :, 3:]])[None], lpos[b:b + 1], inten[b:b + 1],
                  ratio[b:b + 1])
        bgr, depth = rm.render(q, poses[b, :, 3], lpos[b], inten[b], brightness_k=b % 5)
        assert bgr.dtype == np.uint8 and depth.dtype == np.float32
        assert np.array_equal(bgr, row["lit_bgr"][0]), b
        assert np.array_equal((depth * np.float32(1000.0)).astype(np.uint16), row["depth"][0]), b
    assert got["lit_bgr"].any()


def test_gen_syn_set_end_to_end(ctx, meshes, tmp_path):
    classes = ["ape", "can"]
    lm, syn_root = str(tmp_path / "LM6d_refine"), str(tmp_path / "LM6d_refine_syn")
    rs = np.random.RandomState(9)
    os.makedirs(os.path.join(lm, "image_set", "observed"))
    for ci, c in enumerate(classes):  # real training frames: the poses ds_0 takes its statistics from
        os.makedirs(os.path.join(lm, "data", "gt_observed", c))
        idx = ["%02d/%06d" % (ci + 1, i + 1) for i in range(10)]
        with open(os.path.join(lm, "image_set", "observed", "%s_train.txt" % c), "w") as f:
            f.write("".join(x + "\n" for x in idx))
        for x in idx:
            pose = np.hstack([synth.random_rotation(rs), [[rs.normal(0, 0.03)], [rs.normal(0, 0.03)], [0.8 + rs.normal(0, 0.05)]]])
            toolkit._write_pose_txt(os.path.join(lm, "data", "gt_observed", c, x.split("/")[1] + "-pose.txt"), ci + 1, pose)
    syn = toolkit.gen_syn_set(lm, syn_root, ctx, classes, num_images=24, workers=4)
    draws = toolkit.syn_light_draws(syn)
    d = os.path.join(syn_root, "data")
    for c in classes:
        sel = [0, 5, 23]
        pose = [toolkit.se3_q2m(syn[c][i]) for i in sel]
        p32 = np.stack([np.hstack([toolkit.quat2mat(toolkit.mat2quat(p[:3, :3])), p[:, 3:]]) for p in pose]).astype(np.float32)
        r = run(ctx, np.full(3, classes.index(c), np.int32), p32, draws[c]["position"][sel].astype(np.float32),
                draws[c]["intensity"][sel].astype(np.float32),
                np.array([toolkit.BRIGHTNESS_RATIOS[k] for k in draws[c]["ratio_k"][sel]], np.float32))
        gt = ctx.render_dataset(dev(np.full(3, classes.index(c), np.int32)), dev(np.stack(pose), np.float32), K,
                                want=("bgr",))["bgr"].cpu().numpy()
        for j, i in enumerate(sel):
            base = "%s/%06d" % (c, i + 1)
            assert np.array_equal(lm6d_io.read_color(os.path.join(d, "observed", base + "-color.png")), r["lit_bgr"][j])
            assert np.array_equal(lm6d_io.read_depth_u16(os.path.join(d, "observed", base + "-depth.png")), r["depth"][j])
            assert np.array_equal(lm6d_io.read_label(os.path.join(d, "observed", base + "-label.png")), r["label"][j])
            assert np.array_equal(lm6d_io.read_color(os.path.join(d, "gt_observed", base + "-color.png")), gt[j])
            assert r["label"][j].any()
    # every path the live LM6D_REFINE_SYN.load_render_annotation resolves for these classes' first images
    conv = str(tmp_path)
    for path in GOLD["annotation_paths"].tolist():
        if path.split("/")[3] in classes:
            assert os.path.exists(os.path.join(conv, path)), path
    # the data_syn augmentation takes the observed colour and label as the training config reads them
    obs = np.stack([lm6d_io.read_color(os.path.join(d, "observed", "ape/%06d-color.png" % i)) for i in (1, 2)])
    lab = np.stack([lm6d_io.read_label(os.path.join(d, "observed", "ape/%06d-label.png" % i)) for i in (1, 2)])
    augment.BackgroundBank(ctx, [np.full((300, 400, 3), 77, np.uint8)])
    img, comp = ctx.replace_background(dev(obs, np.float32), dev(lab[:, None], np.float32), np.array([0, -1], np.int32),
                                       synth.PIXEL_MEANS_RGB, want_composite=True)
    comp = comp.cpu().numpy()
    assert img.shape == (2, 3, 480, 640)
    assert np.array_equal(comp[0][lab[0] > 0], obs[0][lab[0] > 0]) and (comp[0][lab[0] == 0] != 0).any()
    assert np.array_equal(comp[1], obs[1])
