"""GPU: `dim_render` (image / depth / mask / bgr / bbox, trunc_u8 on and off), `dim_render_lit` and `dim_render_dataset`
against the float64 ray caster (tests/raster_ref.py) and bit for bit against the CPU oracle, on the scenes of
tests/raster_scenes.py: every context size and camera, odd sizes, far vertices, slivers, the 48 / 49-pixel coverage
paths, partial blocks and warps, B = max_batch.  Plus the exact self-consistency of each render's outputs."""
import numpy as np
import pytest
import torch

from deepim_b200 import synth
from deepim_b200.context import Context
from oracle import oracle as O

import py_light_oracle as PL
import raster_ref as RR
import raster_scenes as RS

if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

pytestmark = pytest.mark.gpu
SCENES = RS.geometry_scenes() + RS.mesh_scenes() + [RS.batch16_scene()]
MEANS = synth.PIXEL_MEANS_RGB
FACTOR = 1000.0
LIT_RATIO = np.float32(0.7)


def dev(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else np.asarray(a, dtype))).cuda()


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
    """every render of instances b0 .. b1 - 1 of scene s, as numpy"""
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


def self_consistent(r, trunc):
    """mask == (depth > 0.2), bbox == min / max of the mask, image == float32 of (bgr - mean) by the path's rule"""
    for b in range(len(r["depth"])):
        d, mk = r["depth"][b, 0], r["mask"][b, 0]
        assert np.array_equal(mk, (d > 0.2).astype(np.float32))
        ys, xs = np.nonzero(mk)
        want = [xs.min(), xs.max(), ys.min(), ys.max()] if len(xs) else [-1, -1, -1, -1]
        assert list(r["bbox"][b]) == want
        rgb = r["bgr"][b][..., ::-1].transpose(2, 0, 1)
        if trunc:
            img = (rgb.astype(np.float64) - MEANS[:, None, None]).astype(np.float32)
        else:
            img = rgb - MEANS.astype(np.float32)[:, None, None]
        assert np.array_equal(r["image"][b], img)


def check_scene(ctx, s, b0=0, b1=None):
    b1 = len(s.inst) if b1 is None else b1
    rep = RR.Report(repr(s))
    for c0 in range(b0, b1, 16):
        got = render_all(ctx, s, c0, min(c0 + 16, b1))
        for t in (True, False):
            self_consistent(got[t], t)
        self_consistent(got["lit"], True)
        for k in range(min(16, b1 - c0)):
            c, pose, lpos, inten, ratio = s.inst[c0 + k]
            m = s.meshes[c]
            geo = dict(zn=s.zn, zf=s.zf, H=s.H, W=s.W)
            ref = RR.Render(m, pose, s.K, s.H, s.W, s.zn, s.zf, m.normals)
            for t in (True, False):
                g = got[t]
                RR.check_render(rep, ref, g["depth"][k, 0], g["mask"][k, 0], g["bgr"][k], t)
                o = O.render(m, pose, s.K, means_rgb=MEANS, trunc_u8=t, **geo)
                for n in ("bgr", "image"):
                    assert np.array_equal(g[n][k], o[n]), (repr(s), c0 + k, t, n)
                assert np.array_equal(g["depth"][k, 0], o["depth"]) and np.array_equal(g["mask"][k, 0], o["mask"])
                assert np.array_equal(g["bbox"][k], o["bbox"])
            g = got["lit"]
            RR.check_render(rep, ref, g["depth"][k, 0], g["mask"][k, 0])
            RR.check_lit(rep, ref, g["bgr"][k], lpos, inten, LIT_RATIO, "modelnet")
            o = O.render_lit(m, m.normals, pose, s.K, lpos, inten, LIT_RATIO, means_rgb=MEANS, **geo)
            for n in ("bgr", "image", "bbox"):
                assert np.array_equal(g[n][k], o[n]), (repr(s), c0 + k, "lit", n)
            g = got["ds"]
            RR.check_lit(rep, ref, g["lit_bgr"][k], lpos, inten, ratio, "py_light")
            RR.check_render(rep, ref, g["label"][k], bgr=g["bgr"][k], trunc_u8=True, label=True)
            RR.check_u16(rep, ref, g["depth"][k], g["label"][k], FACTOR)
            o = PL.render_dataset(m, pose, s.K, lpos, inten, ratio, depth_factor=FACTOR, **geo)
            for n in ("lit_bgr", "bgr", "depth", "label"):
                assert np.array_equal(g[n][k], o[n]), (repr(s), c0 + k, "dataset", n)
    return rep


@pytest.mark.parametrize("s", SCENES, ids=repr)
def test_device_against_float64_and_oracle(contexts, s):
    rep = check_scene(context(contexts, s), s)
    print(rep)
    assert rep.ok, str(rep)


def test_device_ownership_grid(contexts):
    s, tri2 = RS.ownership_grid()
    ctx = context(contexts, s)
    got = render_all(ctx, s, 0, 1)
    owner = RS.grid_owner(tri2, s.H, s.W)
    for g in (got[True]["bgr"][0], got[False]["bgr"][0], got["ds"]["bgr"][0]):
        g = np.rint(g).astype(np.int64)
        face = np.where(got[True]["depth"][0, 0] > 0, g[..., 2] + 256 * g[..., 1], -1)
        assert np.array_equal(face, owner), int((face != owner).sum())


def test_large_then_small_object_in_one_context(contexts):
    """a frame-filling render, then a small one into the same context: nothing of the first may show in the second"""
    ms = RS.meshes()
    s = RS.Scene("large then small", "lm")
    for b in range(16):
        s.add(ms["c5"], RS.pose(synth.random_rotation(np.random.RandomState(b)), (0.0, 0.0, 0.35)), seed=b)
    ctx = context(contexts, s)
    big = render_all(ctx, s, 0, 16)
    assert (big[True]["mask"].reshape(16, -1).sum(1) > 5000).all()
    s2 = RS.Scene("small after large", "lm")
    for b, p in enumerate(RS.object_poses(16, "lm", 7)):
        p[2, 3] = 1.9
        s2.add(ms[("cube", "c2", "c5")[b % 3]], p, seed=b)
    rep = check_scene(context(contexts, s2), s2)
    print(rep)
    assert rep.ok, str(rep)
