"""GPU: the training step of the image-only network (a dim_ctx_set_input_mask(ctx, 0) context) against the train oracle with
the 6-channel input (train_oracle.forward_backward(input_mask=False)), against the 8-channel step with zero mask columns, its
parameter table, and fit_batch in bf16 and bf16x3.  With PRED_MASK the training graph still zooms with ZoomMask and learns
the mask; only the network input loses the mask channels."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from oracle import train_oracle as T  # noqa: E402
from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.trainer import Trainer, fit_batch, make_device_batch, param_table  # noqa: E402
import gpu_train_check as G  # noqa: E402

K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
B, SEED = 2, 11


def make_ctx(meshes, input_mask):
    c = Context(0, max_batch=B, max_classes=2, max_verts=6000, max_faces=11000, input_mask=input_mask)
    for i, m in enumerate(meshes):
        c.upload_mesh(i, m)
    return c


@pytest.fixture(scope="module")
def setup():
    meshes = [synth.make_cube(), synth.make_blob()]
    w = synth.make_train_weights(0, input_mask=False)
    batch = G.make_batch(meshes, B, SEED)
    ctx = make_ctx(meshes, False)
    tr = Trainer(ctx, w)
    yield meshes, w, batch, ctx, tr
    ctx.close()


def device_batch(batch):
    b = {k: dev(v) for k, v in batch.items()}
    b["pixel_means_rgb"] = MEANS.astype(np.float32)
    return b


def test_nomask_param_table(setup):
    meshes, w, batch, ctx, tr = setup
    assert int(capi.lib.dim_train_param_count(ctx._h)) == tr.n == sum(n for _, n in param_table(input_mask=False)) == 57742892
    p = tr.get_params()
    for k in w:
        assert np.array_equal(p[k], w[k]), k


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_nomask_training_step_matches_the_checker(setup, precision):
    """Losses within 2e-3 of the fp32 checker in both precisions; gradient cosines >= 0.995 for every tensor in bf16x3 (the
    near-fp32 step).  The bf16 step's gradients are not held to the fp32 checker here: on this batch fc6's reach cos 0.991
    (measured on an H100), an accuracy of the bf16 step itself, which is the 8-channel step bit for bit (test below) and is
    bounded by tests/test_gpu_train.py."""
    meshes, w, batch, ctx, tr = setup
    out, g, zin, lab = T.forward_backward(w, batch, K, MEANS, input_mask=False)
    try:
        tr.set_precision(precision)
        z = tr.zoom_front(device_batch(batch), K)
        res = tr.forward_backward(z)
        torch.cuda.synchronize()
    finally:
        tr.set_precision("bf16")
    losses = res["losses"].cpu().numpy()
    for i, k in ((0, "flow_loss"), (1, "point_matching_loss")):
        assert abs(losses[i] - out[k].sum()) < 2e-3 * out[k].sum(), k
    assert abs(losses[3] - out["objective"]) < 2e-3 * out["objective"]
    gd = tr.grads_dict()
    assert gd["flow_conv1_weight"].shape == (64, 6, 7, 7) == g["flow_conv1_weight"].shape
    for k in sorted(gd):
        if k in T.FROZEN:
            assert np.abs(gd[k]).max() == 0.0
        elif precision == "bf16x3":
            c = G.cmp(gd[k], g[k])
            assert c["cos"] >= 0.995, (precision, k, c)


def test_gradients_equal_the_eight_channel_step_with_zero_mask_columns(setup):
    """The 8-channel trainer with W6 plus zero mask columns, fed the same batch with its masks: every gradient is
    bit-identical, flow_conv1's mask columns aside (the mask-free table does not have them)."""
    meshes, w, batch, ctx, tr = setup
    w8 = dict(w, flow_conv1_weight=np.concatenate([w["flow_conv1_weight"], np.zeros((64, 2, 7, 7), np.float32)], 1))
    c8 = make_ctx(meshes, True)
    try:
        t8 = Trainer(c8, w8)
        for prec in ("bf16", "bf16x3"):
            tr.set_precision(prec)
            t8.set_precision(prec)
            b = device_batch(batch)
            tr.forward_backward(tr.zoom_front(b, K))
            z8 = t8.zoom_front(b, K)
            assert z8["zoom_mask_observed"].abs().max().item() > 0
            t8.forward_backward(z8)
            torch.cuda.synchronize()
            g6, g8 = tr.grads_dict(), t8.grads_dict()
            assert sorted(g6) == sorted(g8)
            for k in g6:
                want = g8[k][:, :6] if k == "flow_conv1_weight" else g8[k]
                assert np.array_equal(g6[k], want), (prec, k)
    finally:
        tr.set_precision("bf16")
        c8.close()


def test_nomask_training_step_refuses_masks(setup):
    meshes, w, batch, ctx, tr = setup
    z = tr.zoom_front(device_batch(batch), K)
    args = [ctx._h] + [capi.C.c_void_p(z[k].data_ptr()) for k in
                       ("zoom_image_observed", "zoom_image_rendered", "zoom_mask_observed", "zoom_mask_rendered", "zoom_factor")]
    args += [None] * 7 + [B, 0] + [None] * 7 + [None, None, 0]
    rc = capi.lib.dim_train_forward_backward(*args, None, None, None)
    assert rc != 0 and b"takes no mask input" in capi.lib.dim_last_error()
    with pytest.raises(ValueError, match="input channels"):
        Trainer(ctx, synth.make_train_weights(0))


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_nomask_fit_batch_lowers_the_objective(setup, precision):
    meshes = setup[0]
    tctx = make_ctx(meshes, False)
    try:
        batch, cls, tgt, depth_gt = make_device_batch(tctx, meshes, B, SEED, K, MEANS)
        tr = Trainer(tctx, synth.make_train_weights(0, input_mask=False), precision=precision)
        objs = fit_batch(tr, batch, cls, tgt, depth_gt, K, n_inner=4).cpu().numpy()
        assert objs.shape == (4,) and np.isfinite(objs).all()
        assert objs[-1] < objs[0], objs
        assert tr.get_params()["flow_conv1_weight"].shape == (64, 6, 7, 7)
        torch.cuda.synchronize()
    finally:
        tctx.close()
