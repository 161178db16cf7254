"""CPU: the RGB-D network's host-side pieces -- the loader's depth conversion, the oracle's RGB-D loop against its RGB
loop, the 10-channel checkpoint and weight helpers, and the HGMMA / TMA code of its conv1 kernel."""
import os
import re

import numpy as np
import pytest

from oracle import oracle as O
from deepim_b200 import mx_params, synth


def test_depth_conversion_matches_the_reference_expression():
    """image.py:203,218: float32(u16) / DEPTH_FACTOR with a Python float is float32 division by the float32 factor."""
    u16 = np.arange(0, 65536, dtype=np.uint16).reshape(256, 256)
    for factor in (1000.0, 10000.0, 999.9, 1.0 / 3.0):
        got = O.depth_from_u16(u16, factor)
        ref = u16.astype(np.float32) / np.float32(factor)
        assert got.dtype == np.float32
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), factor
    # and not float64 division rounded afterwards (the two differ for some inputs)
    f64 = (u16.astype(np.float64) / 999.9).astype(np.float32)
    assert not np.array_equal(O.depth_from_u16(u16, 999.9), f64)


def test_conv1_input_channel_order():
    """deepIM_flownet.py:35-43: images /255, depths /255, then the masks."""
    B, H, W = 1, 4, 5
    rng = np.random.default_rng(0)
    zio, zir = rng.uniform(-120, 150, (B, 3, H, W)).astype(np.float32), rng.uniform(-120, 150, (B, 3, H, W)).astype(np.float32)
    zdo, zdr = rng.uniform(0, 2, (B, 1, H, W)).astype(np.float32), rng.uniform(0, 2, (B, 1, H, W)).astype(np.float32)
    zmo, zmr = (rng.uniform(size=(B, 1, H, W)) > 0.5).astype(np.float32), (rng.uniform(size=(B, 1, H, W)) > 0.5).astype(np.float32)
    x = O.conv1_input(zio, zir, zdo, zdr, zmo, zmr)
    assert x.shape == (B, 10, H, W) and x.dtype == np.float32
    assert np.array_equal(x[:, 6:7], zdo / np.float32(255)) and np.array_equal(x[:, 7:8], zdr / np.float32(255))
    assert np.array_equal(x[:, 8:9], zmo) and np.array_equal(x[:, 9:], zmr)


def test_checker_with_zero_depth_columns_reproduces_the_rgb_loop():
    """With flow_conv1's depth columns zero the RGB-D checker computes the RGB loop: bboxes and zoom factors bit-exact,
    se3 and poses to fp32 summation-order level (the 10-channel convolution sums in a different order)."""
    m = synth.make_cube()
    weights = synth.make_weights(0)
    obs, ini = synth.sample_pose_pairs(1, 5)
    r = O.render(m, obs[0], synth.K_LINEMOD, means_rgb=synth.PIXEL_MEANS_RGB)
    img = synth.transform_image(synth.composite_observed(r["bgr"], r["mask"], 0))[None]
    depth = (r["depth"] + np.float32(0.5) * (r["depth"] == 0)).astype(np.float32)[None, None]
    cls = np.zeros(1, np.int32)
    ref = O.refine(weights, [m], cls, img, ini, synth.K_LINEMOD, 2, synth.PIXEL_MEANS_RGB.astype(np.float32))
    got = O.refine(synth.with_depth_channels(weights), [m], cls, img, ini, synth.K_LINEMOD, 2,
                   synth.PIXEL_MEANS_RGB.astype(np.float32), depth_observed=depth)
    assert np.array_equal(got["bbox"], ref["bbox"])
    assert np.array_equal(got["zoom_factor"], ref["zoom_factor"])
    assert np.abs(got["se3"] - ref["se3"]).max() < 1e-6
    assert np.abs(got["poses"] - ref["poses"]).max() < 1e-6
    # a real depth column changes the output
    w = synth.make_weights(0, input_depth=True)
    moved = O.refine(w, [m], cls, img, ini, synth.K_LINEMOD, 1, synth.PIXEL_MEANS_RGB.astype(np.float32), depth_observed=depth)
    assert np.abs(moved["se3"][0] - ref["se3"][0]).max() > 1e-6


def test_depth_weights_and_ten_channel_checkpoint_round_trip(tmp_path):
    w8 = synth.make_weights(3)
    w10 = synth.make_weights(3, input_depth=True)
    assert w10["flow_conv1_weight"].shape == (64, 10, 7, 7)
    # the RGB channels are the 8-channel set's, the depth channels sit at 6 and 7
    assert np.array_equal(w10["flow_conv1_weight"][:, [0, 1, 2, 3, 4, 5, 8, 9]], w8["flow_conv1_weight"])
    assert np.abs(w10["flow_conv1_weight"][:, 6:8]).max() > 0
    for k in w8:
        if k != "flow_conv1_weight":
            assert np.array_equal(w8[k], w10[k]), k
    z = synth.with_depth_channels(w8)
    assert not z["flow_conv1_weight"][:, 6:8].any()
    n8 = sum(v.size for v in w8.values())
    assert sum(v.size for v in w10.values()) - n8 == 64 * 2 * 49 == 6272
    # MXNet .params round trip; the mode follows from flow_conv1_weight
    mx_params.save_checkpoint(str(tmp_path / "rgbd"), 3, w10)
    arg, aux = mx_params.load_checkpoint(str(tmp_path / "rgbd"), 3)
    assert not aux and sorted(arg) == sorted(w10)
    for k in w10:
        assert arg[k].dtype == np.float32 and np.array_equal(arg[k], w10[k]), k
    assert mx_params.input_depth_of(arg) is True
    assert mx_params.input_depth_of(w8) is False
    with pytest.raises(ValueError):
        mx_params.input_depth_of({"flow_conv1_weight": np.zeros((64, 6, 7, 7), np.float32)})


def test_rgbd_conv1_kernel_is_wgmma_and_tma(root):
    """conv1 of the RGB-D network is a Hopper-native kernel: HGMMA on TMA-staged operands, in all three precisions."""
    import shutil
    import subprocess
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    so = os.path.join(root, "mx-deepim_b200", "libdeepim_b200.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    per_kernel, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            per_kernel[cur] = {"HGMMA": 0, "UTMALDG": 0}
        elif cur:
            for k in per_kernel[cur]:
                if re.search(r"\b%s\b" % k, line):
                    per_kernel[cur][k] += 1
    ks = {k: v for k, v in per_kernel.items() if "conv1_rgbd_kernel" in k and v["HGMMA"]}
    assert len(ks) == 3, sorted(per_kernel)
    for k, v in ks.items():
        assert v["HGMMA"] >= 49 and v["UTMALDG"] >= 1, (k, v)


def test_library_reports_the_rgbd_parameter_table():
    """dim_train_param_info(input_depth=1): the RGB table with flow_conv1_weight (64, 10, 7, 7), 6 272 floats more."""
    from deepim_b200.trainer import param_table, flatten_params, unflatten_params
    rgb, rgbd = param_table(False), param_table(True)
    assert [k for k, _ in rgb] == [k for k, _ in rgbd]
    assert sum(n for _, n in rgbd) - sum(n for _, n in rgb) == 6272
    for (k, n8), (_, n10) in zip(rgb, rgbd):
        assert n10 == (64 * 10 * 49 if k == "flow_conv1_weight" else n8), k
    w = synth.make_train_weights(1, input_depth=True)
    flat = flatten_params(w)
    assert flat.size == sum(n for _, n in rgbd)
    back = unflatten_params(flat, w)
    for k in w:
        assert np.array_equal(back[k], w[k]), k

