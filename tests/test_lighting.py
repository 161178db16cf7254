"""CPU: the ModelNet branch's lighting -- the dim_lighting ABI struct, the light helpers against the reference's own
statements, and the oracle's lit loop against its unlit one where the lighting is neutral."""
import ctypes
import os

import numpy as np
import pytest

from deepim_b200 import lighting, synth
from oracle import oracle as O


def test_lighting_struct_layout_matches_the_header(root, tmp_path):
    """dim_lighting crosses the C ABI by pointer: the ctypes mirror must have the C compiler's layout of the header's struct."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("gcc not on PATH")
    from deepim_b200 import _capi
    src = tmp_path / "layout.c"
    fields = [f for f, _ in _capi.Lighting._fields_]
    assert fields == ["intensity", "offset", "brightness_ratio"]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "deepim_b200.h"\nint main(void) {\n  printf("%zu", sizeof(dim_lighting));\n'
                   + "".join('  printf(" %%zu", offsetof(dim_lighting, %s));\n' % f for f in fields) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)])
    nums = [int(x) for x in subprocess.check_output([str(exe)]).decode().split()]
    assert nums[0] == ctypes.sizeof(_capi.Lighting)
    assert nums[1:] == [getattr(_capi.Lighting, f).offset for f in fields]


def _reference_light(pose):
    """The reference's statements (deepim/core/tester.py:146-160), verbatim, for light index 2."""
    light_position = [0, 1, 1]
    light_position = np.array(light_position) * 0.5
    light_position[0] += pose[0, 3]
    light_position[1] -= pose[1, 3]
    light_position[2] -= pose[2, 3]
    return np.float32(light_position)  # the glumpy uniform is float32


def test_light_position_hand_worked():
    pose = np.zeros((3, 4))
    pose[:, :3] = np.eye(3)
    pose[:, 3] = (0.25, -0.125, 0.75)
    assert np.array_equal(lighting.modelnet_light_position(pose), np.array([0.25, 0.625, -0.25], np.float32))
    pose[:, 3] = (-0.03, 0.02, 0.8)
    got = lighting.modelnet_light_position(pose)
    assert got.dtype == np.float32
    assert np.array_equal(got, np.array([np.float32(-0.03), np.float32(0.5 - 0.02), np.float32(0.5 - 0.8)], np.float32))
    # a batch of poses [n,3,4] gives [n,3]; a custom offset is honoured
    poses = np.stack([pose, pose])
    assert np.array_equal(lighting.modelnet_light_position(poses, (1.0, 0.0, 0.0)),
                          np.tile(np.array([np.float32(1.0 - 0.03), np.float32(-0.02), np.float32(-0.8)]), (2, 1)))


def test_light_position_rounds_once_from_float64():
    """The light is float32(offset -/+ t) evaluated on the float64 pose, not float32(offset) -/+ float32(t): on poses where the
    two differ in the last bit the helper follows the reference (and so does the lit CPU checker)."""
    rng = np.random.default_rng(3)
    differs = 0
    for _ in range(2000):
        pose = np.zeros((3, 4))
        pose[:, :3] = synth.random_rotation(rng)
        pose[:, 3] = (rng.uniform(-0.1, 0.1), rng.uniform(-0.1, 0.1), rng.uniform(0.4, 1.2))
        ref = _reference_light(pose)
        assert np.array_equal(lighting.modelnet_light_position(pose), ref)
        assert np.array_equal(O.light_position(pose), ref)
        p32 = pose.astype(np.float32)
        f32_first = np.array([np.float32(0) + p32[0, 3], np.float32(0.5) - p32[1, 3], np.float32(0.5) - p32[2, 3]], np.float32)
        differs += int(not np.array_equal(f32_first, ref))
    assert differs > 0  # the sample does exercise the double-rounding difference


def test_sample_intensity_is_seeded_uniform_float32():
    a = lighting.sample_intensity(np.random.default_rng(5), (4, 3))
    b = lighting.sample_intensity(np.random.default_rng(5), (4, 3))
    assert a.shape == (4, 3, 3) and a.dtype == np.float32
    assert np.array_equal(a, b)
    assert (a >= np.float32(0.9)).all() and (a <= np.float32(1.1)).all()
    # float64 draws cast to float32, as np.random.uniform followed by the float32 uniform
    assert np.array_equal(a, np.random.default_rng(5).uniform(0.9, 1.1, size=(4, 3, 3)).astype(np.float32))
    src = lighting.LightSource.of({"seed": 5})
    assert np.array_equal(src.draw((4, 3)), a)
    assert not np.array_equal(src.draw((4, 3)), a)  # fresh draws afterwards
    assert src.offset == (0.0, 0.5, 0.5) and src.brightness_ratio == 0.7
    with pytest.raises(ValueError):
        lighting.LightSource.of({"seed": 1, "ratio": 0.5})


def test_oracle_lit_loop_with_neutral_light_equals_its_unlit_loop():
    """brightness_ratio 0 and unit intensity: every lit colour is round(texel) = the unlit (uint8-truncated) colour, so the
    lit CPU loop reproduces the oracle's unlit one exactly."""
    mesh = synth.make_cube()
    mesh.normals = synth.vertex_normals(mesh)
    K, means = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB.astype(np.float32)
    weights = synth.make_weights(0)
    obs, ini = synth.sample_pose_pairs(1, 17)
    r = O.render(mesh, obs[0], K)
    img = synth.transform_image(synth.composite_observed(r["bgr"], r["mask"], 0))[None]
    cls = np.zeros(1, np.int32)
    unlit = O.refine(weights, [mesh], cls, img, ini, K, 2, means)
    lit = O.refine(weights, [mesh], cls, img, ini, K, 2, means,
                   lighting={"intensity": np.ones((2, 1, 3), np.float32), "offset": (0.0, 0.5, 0.5), "brightness_ratio": 0.0})
    for k in ("poses", "se3", "zoom_factor", "bbox"):
        assert np.array_equal(lit[k], unlit[k]), k
    # and a real light changes the colours but not the geometry of the render
    pose = ini[0]
    li = np.array([1.05, 0.95, 1.0], np.float32)
    a = O.render(mesh, pose, K, means_rgb=means)
    b = O.render_lit(mesh, mesh.normals, pose, K, O.light_position(pose), li, 0.7, means_rgb=means)
    assert np.array_equal(a["mask"], b["mask"]) and np.array_equal(a["depth"], b["depth"])
    assert not np.array_equal(a["image"], b["image"])
