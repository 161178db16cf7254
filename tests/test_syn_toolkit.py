"""LM6d_refine_syn data preparation on the host: the random sequences, file names, pose files and lists of
deepim_b200.toolkit against tests/golden/ref_syn.npz (the live toolkit/LM6d_0 and LM6d_ds_0 ... ds_4 scripts, render calls
recorded; tests/golden/make_golden_syn.py), with a fake renderer; and the Render_Py_Light shading of the CPU checker
tests/py_light_oracle.c (the oracle's rasteriser, unchanged, plus the new shading)."""
import io
import os

import numpy as np
import pytest
import torch

from deepim_b200 import synth, toolkit
from oracle import oracle as O

import py_light_oracle as PL

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_syn.npz"))
IDX2CLASS = dict(zip(GOLD["idx2class_ids"].tolist(), GOLD["idx2class_names"].tolist()))
TEXT = dict(zip(GOLD["text_names"].tolist(), GOLD["text_values"].tolist()))
KEEP = int(GOLD["syn_keep"])


def _gt_observed_poses():
    """LM6d_0's gt_observed pose files, read as ds_0 reads them"""
    out = {}
    for c in IDX2CLASS.values():
        names = sorted(n for n in TEXT if n.startswith("LM6d_refine/data/gt_observed/%s/" % c))
        out[c] = np.stack([np.loadtxt(io.StringIO(TEXT[n]), skiprows=1) for n in names])
    return out


@pytest.fixture(scope="module")
def syn_poses():
    return toolkit.gen_syn_observed_poses(_gt_observed_poses(), toolkit.K_LM, int(GOLD["num_images"]))


def _cut(syn):
    return {c: v[:KEEP] for c, v in syn.items()}


def test_syn_observed_poses_equal_the_script_bit_for_bit(syn_poses):
    assert sorted(syn_poses) == sorted(IDX2CLASS.values())
    for c, v in syn_poses.items():
        ref = GOLD["syn_pose/" + c]
        assert v.dtype == np.float64 and np.array_equal(v.astype(np.float32).astype(np.float64), v)
        assert np.array_equal(v[:len(ref)], ref), c
    assert toolkit.syn_poses_sha256(syn_poses) == str(GOLD["syn_sha256"])


def test_light_draws_equal_every_recorded_render_call(syn_poses):
    draws = toolkit.syn_light_draws(_cut(syn_poses))
    cat = lambda k: np.concatenate([draws[c][k] for c in sorted(draws)])
    assert np.array_equal(cat("position"), GOLD["call/LM6d_ds_1/light_position"])
    assert np.array_equal(cat("intensity"), GOLD["call/LM6d_ds_1/light_intensity"])
    assert np.array_equal(cat("ratio_k"), GOLD["call/LM6d_ds_1/brightness_k"])
    assert set(GOLD["call/LM6d_ds_1/brightness_k"].tolist()) == set(range(5))


def test_rendered_poses_are_the_scripts(syn_poses):
    """ds_1 renders quat2mat(mat2quat(R)) of se3_q2m(q), ds_2 R itself; LM6d_0 quat2mat(mat2quat(R)) of the meta pose"""
    q = np.concatenate([v for _, v in sorted(_cut(syn_poses).items())])
    pose = np.stack([toolkit.se3_q2m(x) for x in q])
    assert np.array_equal(pose[:, :3, :3], GOLD["call/LM6d_ds_2/R"])
    assert np.array_equal(pose[:, :, 3], GOLD["call/LM6d_ds_1/t"])
    assert np.array_equal(np.stack([toolkit.quat2mat(toolkit.mat2quat(p[:3, :3])) for p in pose]), GOLD["call/LM6d_ds_1/R"])
    # for every recorded pose the two float32 casts agree, so write_syn_observed_set renders ds_1 and ds_2 in one pass
    assert np.array_equal(GOLD["call/LM6d_ds_1/R"].astype(np.float32), GOLD["call/LM6d_ds_2/R"].astype(np.float32))
    lm0 = np.concatenate([GOLD["input_pose/" + c] for c in IDX2CLASS.values()])
    assert np.array_equal(np.stack([toolkit.quat2mat(toolkit.mat2quat(p[:3, :3])) for p in lm0]), GOLD["call/LM6d_0/R"])


def test_brightness_constants_parse_to_the_device_values():
    """the shader's constants are "{}".format(1 - r) and r parsed as float32; the device computes 1.0f - float32(r)"""
    for r in toolkit.BRIGHTNESS_RATIOS:
        assert np.float32("{}".format(1 - r)) == np.float32(1) - np.float32(r)
        assert np.float32("{}".format(r)) == np.float32(r)


def test_label_png_equals_the_scripts_float64_label(tmp_path):
    import cv2
    lab = (np.random.RandomState(0).rand(48, 64) > 0.5)
    f64 = np.zeros(lab.shape)
    f64[lab] = 1
    cv2.imwrite(str(tmp_path / "a.png"), f64)
    cv2.imwrite(str(tmp_path / "b.png"), lab.astype(np.uint8))
    assert (tmp_path / "a.png").read_bytes() == (tmp_path / "b.png").read_bytes()


class FakeCtx:
    """render / render_dataset with the Context signatures, black images on the CPU"""
    device = torch.device("cpu")
    H, W = 480, 640

    def render_dataset(self, cls_idx, pose, K, znear, zfar, depth_factor, light_position=None, light_intensity=None,
                       brightness_ratio=None, want=()):
        B = len(pose)
        shapes = {"lit_bgr": ((B, 480, 640, 3), torch.uint8), "bgr": ((B, 480, 640, 3), torch.uint8),
                  "depth": ((B, 480, 640), torch.uint16), "label": ((B, 480, 640), torch.uint8)}
        return {k: torch.zeros(shapes[k][0], dtype=shapes[k][1]) for k in want}

    def render(self, cls_idx, pose, K, znear, zfar, trunc_u8=False, want=()):
        B = len(pose)
        return {"bgr": torch.zeros(B, 480, 640, 3), "depth": torch.zeros(B, 1, 480, 640)}


def _files(root, top):
    out = []
    for d, _, fs in os.walk(root):
        out += [os.path.join(top, os.path.relpath(os.path.join(d, f), root)) for f in fs]
    return sorted(out)


def test_syn_writers_write_the_scripts_files(syn_poses, tmp_path):
    syn = _cut(syn_poses)
    root = str(tmp_path / "LM6d_refine_syn")
    slots = {c: 0 for c in syn}
    toolkit.write_syn_observed_set(root, FakeCtx(), syn, toolkit.syn_light_draws(syn), slots, workers=3)
    classes = sorted(syn)
    for ci, c in enumerate(classes):  # ds_4's names and sorted pair lists; its poses (ds_3) are not reproducible
        index = ["{}/{:06d}".format(c, i + 1) for i in range(KEEP)]
        toolkit.write_rendered_set(root, FakeCtx(), c, ci, 0, index, np.zeros((KEEP, 1, 3, 4)), toolkit.K_LM,
                                   syn_names=True)
    got = _files(root, "LM6d_refine_syn")
    want = sorted(f for f in GOLD["files"].tolist() if f.startswith("LM6d_refine_syn/") and "/poses/" not in f)
    assert got == want
    assert set(GOLD["annotation_paths"].tolist()) <= set(got)
    for name, text in TEXT.items():
        if name.startswith("LM6d_refine_syn/") and "/rendered/" not in name and "/poses/" not in name:
            assert open(os.path.join(str(tmp_path), name)).read() == text, name


def test_gt_observed_writer_writes_the_scripts_files(tmp_path):
    import scipy.io as sio
    root = str(tmp_path / "LM6d_refine")
    os.makedirs(os.path.join(root, "image_set", "observed"))
    for cls_idx, c in IDX2CLASS.items():  # the fabricated input of make_golden_syn.py
        names = sorted(n for n in TEXT if n.startswith("LM6d_refine/data/gt_observed/%s/" % c))
        index = ["%02d/%s" % (cls_idx, n.split("/")[-1].split("-")[0]) for n in names]
        os.makedirs(os.path.join(root, "data", "observed", "%02d" % cls_idx))
        with open(os.path.join(root, "image_set", "observed", "%s_all.txt" % c), "w") as f:
            f.write("".join(x + "\n" for x in index))
        for k, (idx, pose) in enumerate(zip(index, GOLD["input_pose/" + c])):
            if k % 2:
                meta = {"cls_indexes": np.array([[99], [cls_idx]], np.float64), "poses": np.stack([np.eye(3, 4), pose], 2)}
            else:
                meta = {"cls_indexes": np.array([[cls_idx], [0]], np.float64), "poses": pose}
            sio.savemat(os.path.join(root, "data", "observed", idx + "-meta.mat"), meta)
    toolkit.write_gt_observed_set(root, FakeCtx(), {c: 0 for c in IDX2CLASS.values()}, IDX2CLASS, workers=2)
    got = _files(os.path.join(root, "data", "gt_observed"), "LM6d_refine/data/gt_observed")
    assert got == sorted(f for f in GOLD["files"].tolist() if f.startswith("LM6d_refine/data/gt_observed/"))
    for name in got:
        if name.endswith("-pose.txt"):
            assert open(os.path.join(str(tmp_path), name)).read() == TEXT[name], name


# ------------------------------------------------------------------------------------------------ oracle
@pytest.fixture(scope="module")
def cube():
    m = synth.make_cube()
    m.normals = synth.vertex_normals(m)
    return m


def test_oracle_py_light_at_white_light_equals_the_modelnet_formula(cube):
    pose = np.array([[0.8, -0.6, 0.0, 0.01], [0.36, 0.48, -0.8, -0.02], [0.48, 0.64, 0.6, 0.6]], np.float32)
    lp = O.light_position(pose, (1.0, 0.0, 1.0))
    for r in toolkit.BRIGHTNESS_RATIOS:
        a = PL.render_dataset(cube, pose, synth.K_LINEMOD, lp, np.ones(3, np.float32), r)
        b = O.render_lit(cube, cube.normals, pose, synth.K_LINEMOD, lp, np.ones(3, np.float32), r, want=("bgr", "depth"))
        assert np.array_equal(a["lit_bgr"], b["bgr"].astype(np.uint8))
        assert np.array_equal(a["depth"], (b["depth"] * np.float32(1000.0)).astype(np.uint16))
        assert np.array_equal(a["label"], (b["depth"] != 0).astype(np.uint8))
        assert a["label"].sum() > 1000


def test_oracle_py_light_known_answer_on_a_quad_facing_the_light():
    """a camera-facing quad lit from the camera's direction: brightness = 1, so colour = texel * (a0 + a1 * I_c)"""
    tex = np.array([[[200, 120, 40]]], np.uint8)
    quad = synth.Mesh(np.array([[-0.1, -0.1, 0], [0.1, -0.1, 0], [0.1, 0.1, 0], [-0.1, 0.1, 0]], np.float32),
                      np.full((4, 2), 0.5, np.float32), np.array([[0, 1, 2], [0, 2, 3]], np.int32), tex)
    quad.normals = np.tile(np.array([0, 0, -1], np.float32), (4, 1))  # towards the camera (OpenCV frame)
    pose = np.hstack([np.eye(3), [[0], [0], [0.5]]]).astype(np.float32)
    light = np.array([0, 0, 1e4], np.float32)  # GL frame: far along the viewing axis behind the camera
    for r, inten in [(0.2, (0.0, 0.0, 1.05)), (0.4, (1.1, 0.95, 0.0)), (0.3, (1.0, 1.0, 1.0))]:
        inten = np.array(inten, np.float32)
        out = PL.render_dataset(quad, pose, synth.K_LINEMOD, light, inten, r)
        a1 = np.float32(r)
        a0 = np.float32(1) - a1
        c = (tex[0, 0].astype(np.float32) / np.float32(255)) * (a0 + (a1 * np.float32(1)) * inten)
        want = np.rint(np.clip(c, 0, 1) * np.float32(255)).astype(np.uint8)[::-1]
        assert np.array_equal(out["lit_bgr"][240, 320], want), (r, out["lit_bgr"][240, 320], want)
        assert np.array_equal(out["bgr"][240, 320], tex[0, 0, ::-1])
        assert out["depth"][240, 320] == 500 and out["label"][240, 320] == 1
