"""CPU: the image-only network's host-side pieces (config.network.INPUT_MASK: False) -- the oracle's ZoomImage against the
reference operator's fixture, its 6-channel tower, the parameter table, the 6-channel checkpoint and weight helpers."""
import hashlib
import os
import sys

import numpy as np
import pytest

from oracle import oracle as O
from deepim_b200 import mx_params, synth

HERE = os.path.dirname(os.path.abspath(__file__))


def test_checker_zoom_image_reproduces_the_reference_operator():
    """The oracle's ZoomImage step against ref_mx_zoom_small.npz (the reference's unmodified ZoomImage operator): the zoom
    factor and both zoomed images bit for bit."""
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import mx_cases as C
    g = np.load(os.path.join(HERE, "golden", "ref_mx_zoom_small.npz"))
    c = C.zoom_case(int(g["seed"]), int(g["B"]), int(g["H"]), int(g["W"]))
    zio, zir, zf, _ = O.zoom_image(c["img_o"], c["img_r"], c["pose"], c["K"], C.PIXEL_MEANS_RGB)
    assert np.array_equal(zf, g["zimg_factor"])
    assert hashlib.sha256(zio.tobytes()).digest() == g["zimg_o_sha"].tobytes()
    assert hashlib.sha256(zir.tobytes()).digest() == g["zimg_r_sha"].tobytes()


def test_conv1_input_is_the_two_images():
    """deepIM_flownet.py:53-62 without INPUT_MASK: observed/255 then rendered/255, nothing else."""
    rng = np.random.default_rng(0)
    zio, zir = rng.uniform(-120, 150, (2, 3, 4, 5)).astype(np.float32), rng.uniform(-120, 150, (2, 3, 4, 5)).astype(np.float32)
    x = O.conv1_input(zio, zir)
    assert x.shape == (2, 6, 4, 5) and x.dtype == np.float32
    assert np.array_equal(x[:, :3], zio / np.float32(255)) and np.array_equal(x[:, 3:], zir / np.float32(255))


def test_six_channel_tower_is_the_eight_channel_one_with_zero_mask_columns():
    """The oracle's tower with W6 and no masks equals it with W6 plus zero mask columns, whatever the masks hold."""
    w6 = synth.make_train_weights(2, input_mask=False)
    w8 = dict(w6, flow_conv1_weight=np.concatenate([w6["flow_conv1_weight"], np.zeros((64, 2, 7, 7), np.float32)], axis=1))
    rng = np.random.default_rng(1)
    zio, zir = rng.uniform(-120, 150, (1, 3, 480, 640)).astype(np.float32), rng.uniform(-120, 150, (1, 3, 480, 640)).astype(np.float32)
    m = (rng.uniform(size=(1, 1, 480, 640)) > 0.5).astype(np.float32)
    r6, t6 = O.net_forward(w6, zio, zir)
    r8, t8 = O.net_forward(w8, zio, zir, m, 1 - m)
    assert np.abs(r6 - r8).max() < 1e-5 and np.abs(t6 - t8).max() < 1e-5


def test_weights_and_six_channel_checkpoint_round_trip(tmp_path):
    w8 = synth.make_train_weights(3)
    w6 = synth.make_train_weights(3, input_mask=False)
    assert w6["flow_conv1_weight"].shape == (64, 6, 7, 7)
    assert np.array_equal(w6["flow_conv1_weight"], w8["flow_conv1_weight"][:, :6])
    for k in w8:
        if k != "flow_conv1_weight":
            assert np.array_equal(w8[k], w6[k]), k
    with pytest.raises(ValueError):
        synth.make_train_weights(3, input_depth=True, input_mask=False)
    mx_params.save_checkpoint(str(tmp_path / "nomask"), 5, w6)
    arg, aux = mx_params.load_checkpoint(str(tmp_path / "nomask"), 5)
    assert not aux and sorted(arg) == sorted(w6)
    for k in w6:
        assert arg[k].dtype == np.float32 and np.array_equal(arg[k], w6[k]), k
    assert mx_params.network_of(arg) == {"input_depth": False, "input_mask": False}
    assert mx_params.network_of(w8) == {"input_depth": False, "input_mask": True}
    assert mx_params.network_of(synth.make_weights(3, input_depth=True)) == {"input_depth": True, "input_mask": True}
    with pytest.raises(ValueError, match="image-only"):
        mx_params.network_of({"flow_conv1_weight": np.zeros((64, 7, 7, 7), np.float32)})


def test_library_reports_the_nomask_parameter_table():
    """dim_train_param_info(input_mask=0): the RGB table with flow_conv1_weight (64, 6, 7, 7), 6 272 floats fewer: 57 742 892."""
    from deepim_b200.trainer import flatten_params, param_table, tensor_sizes, unflatten_params
    rgb, nm = param_table(), param_table(input_mask=False)
    assert [k for k, _ in rgb] == [k for k, _ in nm]
    assert sum(n for _, n in nm) == 57742892 == sum(n for _, n in rgb) - 6272
    for (k, n8), (_, n6) in zip(rgb, nm):
        assert n6 == (64 * 6 * 49 if k == "flow_conv1_weight" else n8), k
    assert sum(n for _, n in tensor_sizes(input_mask=False)) == 57742892
    w = synth.make_train_weights(1, input_mask=False)
    flat = flatten_params(w)
    assert flat.size == 57742892
    back = unflatten_params(flat, w)
    for k in w:
        assert np.array_equal(back[k], w[k]), k

