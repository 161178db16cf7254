"""GPU: the training step in DIM_PREC_BF16X3 (dim_train_set_precision) -- every activation, activation gradient and operand
pack a bf16 hi / lo pair, three tensor-core passes -- against the fp32 training oracle on the batch of tests/test_gpu_train.py.

Tolerances: parameter gradients must close at least 90 % of the bf16 step's gap to the oracle, tensor by tensor:
1 - cos <= max(0.1 (1 - cos_bf16), GRAD_FLOOR), cos_bf16 being the same context's bf16 step on the same batch.  Forward
maps, outputs and losses: the CPU emulation of the pair storage (tests/bf16x3_emulation.py) deviates from fp32 by the
amounts noted below; the H100 step by 5-100x more, because the tensor cores' fp32 accumulation over K up to 9216 is not the
exact sum the emulation takes (recorded with tools/gpu_train_check.py --precision bf16x3, H100 80GB HBM3 at 400 W).  Each
bound sits about 10x above that device value and is 10x tighter than test_gpu_train.py's bf16 bound for the same quantity."""
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
from deepim_b200.trainer import Trainer, fit_batch, make_device_batch  # noqa: E402
import gpu_train_check as G  # noqa: E402

K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
nhwc = lambda a: np.transpose(a, (0, 2, 3, 1))
B, SEED = 2, 11
# emulation / H100 on this batch -> bound (the bf16 step's bound in test_gpu_train.py)
GRAD_FLOOR = 1e-6     # parameter gradients 1 - cos: emulation <= 1.3e-7; the rule's floor (test_train_bf16x3_emulation)
LOSS_REL = 2e-4       # flow loss 2e-7 / 2.4e-5 relative, objective 3e-7 / 2.2e-5 -> 2e-4 (2e-3)
ROT_ABS, TRANS_ABS = 5e-6, 2e-6           # rot_est_norm 4e-8 / 5.6e-7, trans_est 4e-8 / 2.3e-7 -> (5e-4, 1e-4)
FLOW_EST_REL, MASK_PROB_ABS = 1e-3, 2e-4  # flow_est 7e-6 / 8.6e-5 of max|flow_est|, mask_prob 3e-6 / 1.3e-5 -> (2e-2, 1e-2)
MAP_REL = 1e-3        # flow6/5/4, mask4, concat2/3: max error / max|ref| 1.8e-5 / 1.1e-4 -> (3e-2)
DZ_COS = 0.9999       # data gradient reaching each encoder layer: 1 - cos 1.4e-5 / 5.4e-5 -> (0.98)


def _grad_rule(g3, g16, gref, keys=None):
    for k in sorted(keys or gref):
        if k in T.FROZEN or k.startswith("dz_"):
            continue
        c3, c16 = G.cmp(g3[k], gref[k])["cos"], G.cmp(g16[k], gref[k])["cos"]
        assert 1 - c3 <= max(0.1 * (1 - c16), GRAD_FLOOR), (k, 1 - c3, 1 - c16)


def _pair(tr, tid):
    """hi + lo of a bf16 buffer of the step (debug id, id + 100) -> float32 [B,Hp,Wp,C], (py, px, H, W), hi, lo"""
    hi, geo = tr.debug_tensor(tid)
    lo, _ = tr.debug_tensor(100 + tid)
    return hi + lo, geo, hi, lo


@pytest.fixture(scope="module")
def setup():
    meshes = [synth.make_cube(), synth.make_blob()]
    w = synth.make_train_weights(0)
    batch = G.make_batch(meshes, B, SEED)
    out, g, _, _ = T.forward_backward(w, batch, K, MEANS)
    ctx = Context(0, max_batch=B, max_classes=2, max_verts=6000, max_faces=11000)
    for i, m in enumerate(meshes):
        ctx.upload_mesh(i, m)
    tr = Trainer(ctx, w)
    b = {k: dev(v) for k, v in batch.items()}
    b["pixel_means_rgb"] = MEANS.astype(np.float32)
    z = tr.zoom_front(b, K)
    tr.forward_backward(z)
    torch.cuda.synchronize()
    g16 = tr.grads_dict()
    tr.set_precision("bf16x3")
    yield dict(meshes=meshes, w=w, batch=batch, out=out, g=g, ctx=ctx, tr=tr, z=z, b=b, g16=g16)
    ctx.close()


def test_precision_switch_round_trip(setup):
    tr = setup["tr"]
    assert tr.precision == "bf16x3"
    tr.set_precision(capi.PREC_BF16)
    assert tr.precision == "bf16"
    tr.set_precision("bf16x3")
    assert tr.precision == "bf16x3"


def test_bf16x3_step_matches_the_oracle(setup):
    tr, z, out, g = setup["tr"], setup["z"], setup["out"], setup["g"]
    res = tr.forward_backward(z)
    torch.cuda.synchronize()
    _grad_rule(tr.grads_dict(), setup["g16"], g)
    losses = res["losses"].cpu().numpy()
    assert abs(losses[0] - out["flow_loss"].sum()) < LOSS_REL * out["flow_loss"].sum()
    assert abs(losses[1] - out["point_matching_loss"].sum()) < LOSS_REL * out["point_matching_loss"].sum()
    assert abs(losses[3] - out["objective"]) < LOSS_REL * out["objective"]
    assert np.abs(res["rot_est_norm"].cpu().numpy() - out["rot_est_norm"]).max() < ROT_ABS
    assert np.abs(res["trans_est"].cpu().numpy() - out["trans_est"]).max() < TRANS_ABS
    assert np.abs(res["flow_est"].cpu().numpy() - out["flow_est"]).max() < FLOW_EST_REL * np.abs(out["flow_est"]).max()
    assert np.abs(res["mask_prob"].cpu().numpy() - out["mask_prob"]).max() < MASK_PROB_ABS
    for tid, name in ((0, "flow6"), (1, "flow5"), (2, "flow4"), (3, "mask4")):
        assert G.cmp(tr.debug_tensor(tid), nhwc(out[name]))["rel"] < MAP_REL, name
    for tid, name, C in ((10, "concat2", 1026), (11, "concat3", 770)):
        v, (py, px, H, W), hi, lo = _pair(tr, tid)
        assert G.cmp(v[:, py:py + H, px:px + W, :C], nhwc(out[name]))["rel"] < MAP_REL, name
        assert np.abs(lo[:, py:py + H, px:px + W, :C]).max() > 0, name   # the lo half carries the residual
        for half in (hi, lo):                                             # padding channels and borders stay zero in both halves
            assert np.abs(half[:, py:py + H, px:px + W, C:]).max() == 0.0, name
            assert max(np.abs(half[:, 0]).max(), np.abs(half[:, :, 0]).max(), np.abs(half[:, py + H:]).max(),
                       np.abs(half[:, :, px + W:]).max()) == 0.0, name
    # the data gradient reaching every encoder layer, as hi + lo, zero border intact
    for i, (name, _, _) in enumerate(T.ENC):
        v, (py, px, H, W), hi, lo = _pair(tr, 20 + i)
        assert G.cmp(v[:, py:py + H, px:px + W, :], nhwc(g["dz_" + name]))["cos"] > DZ_COS, name
        assert max(np.abs(v[:, 0]).max(), np.abs(v[:, -1]).max(), np.abs(v[:, :, 0]).max(), np.abs(v[:, :, -1]).max()) == 0.0


def test_bf16x3_forward_only_gives_the_same_outputs(setup):
    tr, z = setup["tr"], setup["z"]
    full = tr.forward_backward(z)
    fwd = tr.forward_backward(z, backward=False)
    torch.cuda.synchronize()
    for k in ("rot_est_norm", "trans_est", "flow_est", "mask_prob", "losses"):
        assert torch.equal(full[k], fwd[k]), k
    # and the test graph's non-FAST_TEST outputs follow the context's precision
    w, batch = setup["w"], setup["batch"]
    b = {k: dev(batch[k]) for k in ("image_observed", "image_rendered", "mask_observed", "mask_rendered", "src_pose")}
    b["pixel_means_rgb"] = MEANS.astype(np.float32)
    got = tr.test_forward_full(b, K)
    ref = T.test_forward_full(w, batch["image_observed"], batch["image_rendered"], batch["mask_observed"], batch["mask_rendered"],
                              batch["src_pose"], K, MEANS)
    se3 = got["se3"].cpu().numpy()
    assert np.abs(se3[:, :4] - ref["se3"][:, :4]).max() < 2e-4 and np.abs(se3[:, 4:] - ref["se3"][:, 4:]).max() < 2e-4  # (2e-2, 2e-3)
    assert np.abs(got["zoom_mask_observed_pred"].cpu().numpy() - ref["zoom_mask_observed_pred"]).max() < MASK_PROB_ABS
    fe, rfe = got["flow_est"].cpu().numpy(), ref["flow_est"]
    assert np.abs(fe - rfe).max() < 2e-3 * max(np.abs(rfe).max(), 1.0)                                                    # (3e-2)


def test_bf16x3_step_is_deterministic(setup):
    tr, z = setup["tr"], setup["z"]
    tr.forward_backward(z)
    a = tr.grads.clone()
    tr.forward_backward(z)
    torch.cuda.synchronize()
    assert torch.equal(a, tr.grads)


def test_switching_precision_leaves_the_bf16_step_unchanged(setup):
    tr, z = setup["tr"], setup["z"]
    tr.set_precision("bf16")
    r0 = tr.forward_backward(z)
    g0 = tr.grads.clone()
    tr.set_precision("bf16x3")
    tr.forward_backward(z)
    tr.set_precision("bf16")
    r1 = tr.forward_backward(z)
    torch.cuda.synchronize()
    assert torch.equal(g0, tr.grads)
    for k in ("rot_est_norm", "trans_est", "flow_est", "mask_prob", "losses"):
        assert torch.equal(r0[k], r1[k]), k
    tr.set_precision("bf16x3")


def test_precision_setter_refuses_other_values(setup):
    ctx = setup["ctx"]
    for bad in (capi.PREC_FP16, 7, -1):
        rc = capi.lib.dim_train_set_precision(ctx._h, bad)
        msg = capi.lib.dim_last_error()
        assert rc != 0 and b"DIM_PREC_BF16" in msg and b"DIM_PREC_BF16X3" in msg, (bad, rc, msg)
    assert setup["tr"].precision == "bf16x3"   # a refused value changes nothing
    with pytest.raises(Exception):
        setup["tr"].set_precision("fp16")
    bare = Context(0, max_batch=1, max_classes=1, max_verts=100, max_faces=100)
    try:
        rc = capi.lib.dim_train_set_precision(bare._h, capi.PREC_BF16X3)
        assert rc != 0 and b"dim_train_create" in capi.lib.dim_last_error()
    finally:
        bare.close()


def test_bf16x3_rgbd_step_matches_the_checker(setup):
    meshes = setup["meshes"]
    w = synth.make_train_weights(0, input_depth=True)
    batch = dict(setup["batch"])
    obs, ini = synth.sample_pose_pairs(B, SEED)
    cls = (np.arange(B) % len(meshes)).astype(np.int32)
    depth_gt = np.stack([O.render(meshes[cls[b]], obs[b], K, trunc_u8=False)["depth"] for b in range(B)])[:, None]
    upd = O.train_update(meshes, cls, ini.astype(np.float32), np.tile(np.array([1, 0, 0, 0], np.float32), (B, 1)),
                         np.zeros((B, 3), np.float32), obs.astype(np.float32), depth_gt, K, MEANS)
    noise = np.random.default_rng(4).normal(0, 0.002, depth_gt.shape).astype(np.float32)
    batch["depth_observed"] = np.where(depth_gt > 0, depth_gt + noise, 0).astype(np.float32)
    batch["depth_rendered"] = upd["depth_rendered"]
    out, g, _, _ = T.forward_backward(w, batch, K, MEANS)
    ctx = Context(0, max_batch=B, max_classes=2, max_verts=6000, max_faces=11000, input_depth=True)
    try:
        for i, m in enumerate(meshes):
            ctx.upload_mesh(i, m)
        tr = Trainer(ctx, w)
        b = {k: dev(v) for k, v in batch.items()}
        b["pixel_means_rgb"] = MEANS.astype(np.float32)
        z = tr.zoom_front(b, K)
        tr.forward_backward(z)
        torch.cuda.synchronize()
        g16 = tr.grads_dict()
        tr.set_precision("bf16x3")
        res = tr.forward_backward(z)
        torch.cuda.synchronize()
        g3 = tr.grads_dict()
        _grad_rule(g3, g16, g)
        losses = res["losses"].cpu().numpy()
        assert abs(losses[3] - out["objective"]) < LOSS_REL * out["objective"]
        # flow_conv1's depth columns on their own
        dcol = lambda d: d["flow_conv1_weight"][:, 6:8]
        c3, c16 = G.cmp(dcol(g3), dcol(g))["cos"], G.cmp(dcol(g16), dcol(g))["cos"]
        assert 1 - c3 <= max(0.1 * (1 - c16), GRAD_FLOOR) and np.abs(dcol(g)).max() > 0, (c3, c16)
    finally:
        ctx.close()


def test_bf16x3_fit_batch_lowers_the_objective(setup):
    meshes = setup["meshes"]
    tctx = Context(0, max_batch=B, max_classes=2, max_verts=6000, max_faces=11000)
    try:
        for i, m in enumerate(meshes):
            tctx.upload_mesh(i, m)
        batch, cls, tgt, depth_gt = make_device_batch(tctx, meshes, B, SEED, K, MEANS)
        tr = Trainer(tctx, synth.make_train_weights(0), precision="bf16x3")
        objs = fit_batch(tr, batch, cls, tgt, depth_gt, K, n_inner=4).cpu().numpy()
        assert objs.shape == (4,) and np.isfinite(objs).all()
        assert objs[-1] < objs[0], objs
        torch.cuda.synchronize()
    finally:
        tctx.close()


def test_bf16x3_sgd_update_feeds_the_bf16x3_inference_path(setup):
    """After an update in bf16x3 the packs' lo halves are current: dim_net_fwd(DIM_PREC_BF16X3) of the same context matches
    the oracle run with the updated master weights at the bf16x3 inference tolerance (test_gpu_train.py)."""
    tr, ctx, z = setup["tr"], setup["ctx"], setup["z"]
    tr.forward_backward(z)
    tr.update(lr=1e-3)
    rot, trans = ctx.net_forward(z["zoom_image_observed"], z["zoom_image_rendered"], z["zoom_mask_observed"], z["zoom_mask_rendered"],
                                 precision=capi.PREC_BF16X3)
    pnow = tr.get_params()
    orot, otrans = O.net_forward(pnow, z["zoom_image_observed"].cpu().numpy(), z["zoom_image_rendered"].cpu().numpy(),
                                 z["zoom_mask_observed"].cpu().numpy(), z["zoom_mask_rendered"].cpu().numpy())
    assert np.abs(rot.cpu().numpy() - orot).max() < 1e-4 and np.abs(trans.cpu().numpy() - otrans).max() < 1e-3
    p0 = setup["w"]
    assert any(not np.array_equal(pnow[k], p0[k]) for k in ("conv2_weight", "deconv5_weight"))
