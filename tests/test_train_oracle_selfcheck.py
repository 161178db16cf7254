"""CPU: self-consistency of the training oracle (oracle/train_oracle.py).  The oracle is PARITY UNPINNED for MXNet's
arithmetic, but its gradient wiring (autograd + the reference's hand-written Transform3D backward + the pass-through
ZoomTrans backward + MakeLoss / LogisticRegressionOutput scaling) can be checked against finite differences of its own
objective, and its shapes / parameter count against the reference's graph (SURVEY 8 row a10)."""
import numpy as np

from oracle import oracle as O, train_oracle as T
from deepim_b200 import synth

K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB


def _batch():
    mesh = synth.make_cube()
    obs, ini = synth.sample_pose_pairs(1, 5)
    tgt32, src32 = obs.astype(np.float32), ini.astype(np.float32)
    r = O.render(mesh, obs[0], K, trunc_u8=False)
    depth_gt, mask_gt = r["depth"][None, None], r["mask"][None, None]
    upd = O.train_update([mesh], np.zeros(1, np.int32), src32, np.array([[1, 0, 0, 0]], np.float32), np.zeros((1, 3), np.float32),
                         tgt32, depth_gt, K, MEANS)
    img = synth.transform_image(synth.composite_observed(r["bgr"], r["mask"], 0))[None]
    pts = np.zeros((1, 3, 3000), np.float32)
    pw = np.zeros((1, 3, 3000), np.float32)
    v = mesh.verts[:3000]
    pts[0, :, :len(v)], pw[0, :, :len(v)] = v.T, 1
    pobs = (tgt32[0, :, :3] @ pts[0] + tgt32[0, :, 3:4])[None].astype(np.float32)
    box = O.box_mask(O.mask_bbox(mask_gt[0, 0], 0.0), 480, 640)[None, None]
    return dict(image_observed=img, image_rendered=upd["image_rendered"], mask_observed=box, mask_gt_observed=mask_gt,
                mask_rendered=upd["mask_rendered"], src_pose=upd["src_pose"], rot=upd["rot"], trans=upd["trans"], flow=upd["flow"],
                flow_weights=upd["flow_weights"], point_cloud_model=pts, point_cloud_weights=pw, point_cloud_observed=pobs)


def test_training_oracle_gradients_match_finite_differences():
    w = synth.make_train_weights(0)
    batch = _batch()
    zin, lab = T.zoom_inputs(batch, K, MEANS)
    out, g = T.graph(w, zin, lab, requires_grad=True)
    # shapes of the decoder (deepIM_flownet.py:121-165) and the parameter count of the train graph (57.75 M)
    assert out["concat2"].shape == (1, 1026, 15, 20) and out["concat3"].shape == (1, 770, 30, 40)
    assert out["flow_est_crop"].shape == (1, 2, 480, 640) and out["mask_prob"].shape == (1, 1, 480, 640)
    assert sum(v.size for v in w.values()) == 57749164
    assert np.abs(g["upsampling_weight"]).max() == 0 and np.abs(g["mask_upsampling_weight"]).max() == 0   # lr_mult 0
    assert abs(np.linalg.norm(out["rot_est_norm"][0]) - 1.0) < 1e-6

    def objective(name, idx, delta):
        w2 = dict(w)
        a = w[name].copy()
        a.reshape(-1)[idx] += delta
        w2[name] = a
        return T.graph(w2, zin, lab, requires_grad=False)[0]["objective"]

    # trans head -> invZoomTrans (gradient passes unscaled, b_zoom_grad=False) -> Transform3D backward; rot head -> L2Normalization
    # -> Transform3D's quaternion backward; mask head -> LogisticRegressionOutput scaling (grad_scale / (480*640))
    wx = float(lab["zoom_factor"][0, 0])
    for name, idx, h, scale in (("trans_bias", 2, 2e-3, 1.0), ("trans_bias", 0, 2e-3, wx), ("rot_bias", 1, 2e-3, 1.0),
                                ("mask_conv3_bias", 0, 5e-2, 1.0)):
        fd = (objective(name, idx, h) - objective(name, idx, -h)) / (2 * h)
        # quirk kept from the reference: invZoomTrans is built with b_zoom_grad=False, so its backward does NOT multiply the
        # x / y gradient by the zoom factor (zoom_trans.py:60-68): the "gradient" the optimiser sees is the true one / wx
        an = float(g[name].reshape(-1)[idx]) * scale
        assert abs(fd - an) <= 0.04 * max(abs(an), abs(fd)) + 2e-4, (name, idx, fd, an)


def test_bf16_storage_explains_the_device_gradient_deviation():
    """Calibration of the GPU tolerances (tests/test_gpu_train.py: cosine >= 0.995, error <= 0.15 max|g| on 99 % of the entries): running the ORACLE
    with the device's storage format emulated (bf16 operand weights, activations and activation gradients; fp32 accumulation)
    on the same batch deviates from the fp32 oracle like the device did (tests/golden/train_check_device.json: the gradient
    cosines of tools/gpu_train_check.py on an H100) --
    i.e. the device's deviation is the cost of the storage format, not of the kernels."""
    import json
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "tools"))
    import gpu_train_check as G
    meshes = [synth.make_cube(), synth.make_blob()]
    w = synth.make_train_weights(0)
    batch = G.make_batch(meshes, 2, 11)                      # the batch of the recorded device run
    zin, lab = T.zoom_inputs(batch, K, MEANS)
    _, g32 = T.graph(w, zin, lab, requires_grad=True)
    _, g16 = T.graph(w, zin, lab, requires_grad=True, emulate_bf16=True)
    dev = json.load(open(os.path.join(root, "tests", "golden", "train_check_device.json")))["grads"]
    worst_gap = 0.0
    for k, d in dev.items():
        if k in T.FROZEN:
            continue
        e = G.cmp(g16[k], g32[k])
        assert e["cos"] > 0.995, (k, e)                      # the emulation itself stays inside the GPU test's tolerance
        worst_gap = max(worst_gap, e["cos"] - d["cos"])
        assert d["cos"] > e["cos"] - 2.5e-3, (k, d["cos"], e["cos"])   # the device is as close to fp32 as the emulation (+- noise)
    assert worst_gap < 2.5e-3
