"""GPU: the training step of the RGB-D network (dim_train_forward_backward on an RGB-D context) against the train oracle
(train_oracle.forward_backward on a batch with depths: train_oracle.graph with the 10-channel input), its parameter table, and
fit_batch carrying the re-render's depth.  Bounds as tests/test_gpu_train.py (bf16 mixed-precision step, fp32 checker)."""
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

from oracle import oracle as O, train_oracle as T  # noqa: E402
from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.trainer import Trainer, fit_batch, make_device_batch, param_table  # noqa: E402
import gpu_train_check as G  # noqa: E402

K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
B, SEED = 2, 11


@pytest.fixture(scope="module")
def setup():
    meshes = [synth.make_cube(), synth.make_blob()]
    w = synth.make_train_weights(0, input_depth=True)
    batch = G.make_batch(meshes, B, SEED)
    # the depths of the same pairs: the observed render's depth plus 2 mm noise, and the update's render depth
    obs, ini = synth.sample_pose_pairs(B, SEED)
    cls = (np.arange(B) % len(meshes)).astype(np.int32)
    depth_gt = np.stack([O.render(meshes[cls[b]], obs[b], K, trunc_u8=False)["depth"] for b in range(B)])[:, None]
    upd = O.train_update(meshes, cls, ini.astype(np.float32), np.tile(np.array([1, 0, 0, 0], np.float32), (B, 1)),
                         np.zeros((B, 3), np.float32), obs.astype(np.float32), depth_gt, K, MEANS)
    noise = np.random.default_rng(4).normal(0, 0.002, depth_gt.shape).astype(np.float32)
    batch["depth_observed"] = np.where(depth_gt > 0, depth_gt + noise, 0).astype(np.float32)
    batch["depth_rendered"] = upd["depth_rendered"]
    ctx = Context(0, max_batch=B, max_classes=2, max_verts=6000, max_faces=11000, input_depth=True)
    for i, m in enumerate(meshes):
        ctx.upload_mesh(i, m)
    tr = Trainer(ctx, w)
    yield meshes, w, batch, ctx, tr
    ctx.close()


def test_rgbd_param_table(setup):
    """The RGB-D table is the RGB one with flow_conv1_weight (64, 10, 7, 7): 6 272 floats more, nothing else moves."""
    meshes, w, batch, ctx, tr = setup
    rgb, rgbd = param_table(False), param_table(True)
    assert sum(n for _, n in rgbd) - sum(n for _, n in rgb) == 64 * 2 * 49 == 6272
    assert int(capi.lib.dim_train_param_count(ctx._h)) == tr.n == sum(n for _, n in rgbd) == 57749164 + 6272
    assert [k for k, _ in rgb] == [k for k, _ in rgbd]
    for (k, n8), (_, n10) in zip(rgb, rgbd):
        assert n10 == (64 * 10 * 49 if k == "flow_conv1_weight" else n8), k
    p = tr.get_params()
    for k in w:
        assert np.array_equal(p[k], w[k]), k


def test_rgbd_training_step_matches_the_checker(setup):
    meshes, w, batch, ctx, tr = setup
    out, g, zin, lab = T.forward_backward(w, batch, K, MEANS)
    b = {k: dev(v) for k, v in batch.items()}
    b["pixel_means_rgb"] = MEANS.astype(np.float32)
    z = tr.zoom_front(b, K)
    for k in ("zoom_depth_observed", "zoom_depth_rendered"):
        assert np.array_equal(z[k].cpu().numpy(), zin[k]), k
    res = tr.forward_backward(z)
    torch.cuda.synchronize()
    losses = res["losses"].cpu().numpy()
    assert abs(losses[0] - out["flow_loss"].sum()) < 2e-3 * out["flow_loss"].sum()
    assert abs(losses[1] - out["point_matching_loss"].sum()) < 2e-3 * out["point_matching_loss"].sum()
    assert abs(losses[3] - out["objective"]) < 2e-3 * out["objective"]
    gd = tr.grads_dict()
    for k in sorted(gd):
        if k in T.FROZEN:
            assert np.abs(gd[k]).max() == 0.0
            continue
        c = G.cmp(gd[k], g[k])
        bad = np.abs(gd[k].astype(np.float64) - g[k]) > 0.15 * np.abs(g[k]).max()
        assert c["cos"] > 0.995 and bad.mean() <= 0.01, (k, c, int(bad.sum()))
    # the depth columns of flow_conv1 on their own
    c = G.cmp(gd["flow_conv1_weight"][:, 6:8], g["flow_conv1_weight"][:, 6:8])
    assert c["cos"] > 0.995 and np.abs(g["flow_conv1_weight"][:, 6:8]).max() > 0, c


def test_training_step_refuses_depth_the_network_does_not_take(setup):
    meshes, w, batch, ctx, tr = setup
    b = {k: dev(v) for k, v in batch.items()}
    b["pixel_means_rgb"] = MEANS.astype(np.float32)
    z = tr.zoom_front(b, K)
    args = [ctx._h] + [capi.C.c_void_p(z[k].data_ptr()) for k in
                       ("zoom_image_observed", "zoom_image_rendered", "zoom_mask_observed", "zoom_mask_rendered", "zoom_factor")]
    args += [None] * 7 + [B, 0] + [None] * 7 + [None, None, 0]
    rc = capi.lib.dim_train_forward_backward(*args, None, None, None)
    assert rc != 0 and b"takes depth input" in capi.lib.dim_last_error()
    with pytest.raises(ValueError, match="input channels"):
        Trainer(ctx, synth.make_train_weights(0))


def test_rgbd_fit_batch_lowers_the_objective(setup):
    meshes, w, _, _, _ = setup
    tctx = Context(0, max_batch=B, max_classes=2, max_verts=6000, max_faces=11000, input_depth=True)
    try:
        for i, m in enumerate(meshes):
            tctx.upload_mesh(i, m)
        batch, cls, tgt, depth_gt = make_device_batch(tctx, meshes, B, SEED, K, MEANS, input_depth=True)
        assert batch["depth_rendered"].abs().max().item() > 0 and batch["depth_observed"].abs().max().item() > 0
        tr = Trainer(tctx, synth.make_train_weights(0, input_depth=True))
        objs = fit_batch(tr, batch, cls, tgt, depth_gt, K, n_inner=4).cpu().numpy()
        assert objs.shape == (4,) and np.isfinite(objs).all()
        assert objs[-1] < objs[0], objs
        torch.cuda.synchronize()
    finally:
        tctx.close()
