"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's TRAINING graph (SURVEY 8 row a10 + C4).

Follows deepim/symbols/deepIM_flownet.py:
  get_convs  l.32-167  (encoder, fc6/fc7, decoder Convolution1/deconv5/upsample_flow6to5/Concat2/...)
  get_loss   l.171-365 (Convolution3 + fixed bilinear `upsampling` + Crop(8,8) + flow loss; rot/trans heads,
                        L2Normalization, invZoomTrans, Transform3D point-matching loss; mask_conv3 +
                        mask_upsampling + LogisticRegressionOutput)
  get_train_symbol l.367-545 (ZoomMask / ZoomImageWithFactor / ZoomTrans / ZoomFlow wiring)
and the optimiser call deepim/train.py:296-304 + deepim/core/module.py:1131-1137 (one SGD update after every
inner iteration).  Loss weights from experiments/deepim/cfgs/*.yaml: LW_PM 0.1, NUM_3D_SAMPLE 3000, LW_FLOW 0.25,
LW_MASK 0.03, SE3_PM_LOSS_TYPE L1 (config.py:112), NORMALIZE_FLOW 20, NORMALIZE_3D_POINT 0.1.

PARITY UNPINNED: the arithmetic of Convolution / Deconvolution / Crop / L2Normalization / MakeLoss /
LogisticRegressionOutput / SGD lives in MXNet (un-vendored, `requirements.txt:5` unpinned `mxnet-cu90`,
README pins 1.2.0) and the reference ships no golden vectors for it.  The third-party semantics assumed here are
the ones SURVEY Appendix B items 19-23 record:
  * MakeLoss backward = constant grad_scale per element  ==> total objective = sum(grad_scale * loss_elem)
  * LogisticRegressionOutput backward = grad_scale / num_output * (sigmoid(x) - label), num_output = 480*640
    ==> objective term = grad_scale/num_output * sum BCE-with-logits
  * Deconvolution output (in-1)*s + k, weight (Cin, Cout/group, kh, kw)  (== torch conv_transpose2d)
  * Crop(a, b, offset) = a[:, :, oy:oy+Hb, ox:ox+Wb]
  * L2Normalization(mode=instance) = x / sqrt(sum(x^2) + 1e-10)
  * SGD: mom = momentum*mom - lr*(rescale_grad*grad + wd*w); w += mom; wd only on *_weight, lr_mult 0 on the
    two bilinear upsampling weights
Only Transform3D (forward / custom backward) is pinned by the reference's own self-test (transform3d.py:311-539).
torch autograd (CPU fp32) provides the derivative of everything but Transform3D, whose backward is the
reference's hand-written one (oracle.transform3d_backward)."""
from __future__ import annotations

import numpy as np

from . import oracle as O
from .oracle import ENC

LW_PM, NUM_3D_SAMPLE, LW_FLOW, LW_MASK = 0.1, 3000, 0.25, 0.03
NORMALIZE_FLOW, NORMALIZE_3D_POINT = 20.0, 0.1
FROZEN = ("upsampling_weight", "mask_upsampling_weight")
# deconv5 / deconv4 of the decoder below: 4x4, stride 2, output cropped to the skip connection's size from row / column 1
DECONV_STRIDE, DECONV_CROP = 2, 1


def bilinear_kernel(k=32):
    """mx.init.Initializer._init_bilinear: w[y, x] = (1 - |x/f - c|)(1 - |y/f - c|), f = ceil(k/2),
    c = (2f - 1 - f%2) / (2f)."""
    f = np.ceil(k / 2.0)
    c = (2 * f - 1 - f % 2) / (2.0 * f)
    i = np.arange(k)
    v = 1 - np.abs(i / f - c)
    return np.outer(v, v).astype(np.float32)


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))


def graph(weights, zin, labels, requires_grad=True, num_threads=None, emulate_bf16=False):
    """The network part of the train symbol on already-zoomed inputs.
    zin: zoom_image_observed, zoom_image_rendered (B,3,H,W); zoom_depth_observed, zoom_depth_rendered (B,1,H,W) for the
         RGB-D network; zoom_mask_observed, zoom_mask_rendered (B,1,H,W) unless the network is image-only (O.conv1_input)
    labels: zoom_factor (B,4), zoom_flow (B,2,H,W), zoom_flow_weights (B,2,H,W), zoom_mask_gt_observed (B,1,H,W),
            src_pose (B,3,4), point_cloud_model / point_cloud_weights / point_cloud_observed (B,3,N)
    Returns (outputs dict of numpy arrays, grads dict name -> numpy) ; grads is {} when requires_grad=False.
    emulate_bf16=True rounds what the device step keeps in bf16 -- conv / deconv operand weights, every stored activation
    and every activation gradient -- to bf16 (fp32 accumulation everywhere, fp32 master weights): the resulting deviation
    from the fp32 run is the intrinsic cost of that storage format and calibrates the tolerances of tests/test_gpu_train.py."""
    import torch
    import torch.nn.functional as F

    if num_threads:
        torch.set_num_threads(num_threads)
    P = {k: _t(v).requires_grad_(requires_grad and k not in FROZEN) for k, v in weights.items()}
    rb = (lambda t: t.bfloat16().float()) if emulate_bf16 else (lambda t: t)

    def store(t):  # an activation as the device stores it (+ its gradient on the way back)
        if not emulate_bf16:
            return t
        t = rb(t)
        if t.requires_grad:
            t.register_hook(lambda g: g.bfloat16().float())
        return t

    tc = ("flow_conv1", "conv2", "conv3", "conv3_1", "conv4", "conv4_1", "conv5", "conv5_1", "conv6", "conv6_1", "fc6", "deconv5", "deconv4")
    if emulate_bf16:  # tensor-core operands are bf16; the thin 2-channel heads, fc7, rot, trans read the fp32 master
        P = {k: (rb(v) if k.endswith("_weight") and k[:-7] in tc else v) for k, v in P.items()}
        for k, v in P.items():
            if k.endswith("_weight") and k[:-7] in tc and requires_grad:
                v.retain_grad()
    lrelu = lambda x: store(F.leaky_relu(x, 0.1))
    x = rb(torch.from_numpy(O.conv1_input(zin["zoom_image_observed"], zin["zoom_image_rendered"], zin.get("zoom_depth_observed"),
                            zin.get("zoom_depth_rendered"), zin.get("zoom_mask_observed"), zin.get("zoom_mask_rendered"))))
    feat, pre = {}, {}
    for name, s, p in ENC:
        z = F.conv2d(x, P[name + "_weight"], P[name + "_bias"], stride=s, padding=p)
        if requires_grad:
            z.retain_grad()
        pre[name] = z
        x = lrelu(z)
        feat[name] = x
    r10, r8, r6 = feat["conv6_1"], feat["conv5_1"], feat["conv4_1"]
    h = F.leaky_relu(F.linear(r10.flatten(1), P["fc6_weight"], P["fc6_bias"]), 0.1)   # fc activations stay fp32 on the device
    h = F.leaky_relu(F.linear(h, P["fc7_weight"], P["fc7_bias"]), 0.1)
    rot = F.linear(h, P["rot_weight"], P["rot_bias"])
    ztrans = F.linear(h, P["trans_weight"], P["trans_bias"])
    # decoder (symbol:121-165)
    flow6 = F.conv2d(r10, P["Convolution1_weight"], P["Convolution1_bias"], padding=1)
    d5 = F.conv_transpose2d(r10, P["deconv5_weight"], P["deconv5_bias"],
                            stride=DECONV_STRIDE)[:, :, DECONV_CROP:DECONV_CROP + r8.shape[2], DECONV_CROP:DECONV_CROP + r8.shape[3]]
    up65 = F.conv_transpose2d(flow6, P["upsample_flow6to5_weight"], P["upsample_flow6to5_bias"], stride=2)
    up65 = store(up65[:, :, 1:1 + r8.shape[2], 1:1 + r8.shape[3]])
    cat2 = torch.cat([r8, lrelu(d5), up65], dim=1)
    flow5 = F.conv2d(cat2, P["Convolution2_weight"], P["Convolution2_bias"], padding=1)
    d4 = F.conv_transpose2d(cat2, P["deconv4_weight"], P["deconv4_bias"],
                            stride=DECONV_STRIDE)[:, :, DECONV_CROP:DECONV_CROP + r6.shape[2], DECONV_CROP:DECONV_CROP + r6.shape[3]]
    up54 = F.conv_transpose2d(flow5, P["upsample_flow5to4_weight"], P["upsample_flow5to4_bias"], stride=2)
    up54 = store(up54[:, :, 1:1 + r6.shape[2], 1:1 + r6.shape[3]])
    cat3 = torch.cat([r6, lrelu(d4), up54], dim=1)
    # losses (symbol:171-365)
    Himg, Wimg = zin["zoom_image_observed"].shape[-2:]
    flow4 = F.conv2d(cat3, P["Convolution3_weight"], P["Convolution3_bias"], padding=1)
    flow_full = F.conv_transpose2d(flow4, P["upsampling_weight"], None, stride=16, groups=2)[:, :, 8:8 + Himg, 8:8 + Wimg]
    fw = _t(labels["zoom_flow_weights"])
    flow_loss = fw * (flow_full - _t(labels["zoom_flow"]) / NORMALIZE_FLOW) ** 2
    mask4 = F.conv2d(cat3, P["mask_conv3_weight"], P["mask_conv3_bias"], padding=1)
    mask_logit = F.conv_transpose2d(mask4, P["mask_upsampling_weight"], None, stride=16)[:, :, 8:8 + Himg, 8:8 + Wimg]
    mask_gt = _t(labels["zoom_mask_gt_observed"])
    mask_bce = F.binary_cross_entropy_with_logits(mask_logit, mask_gt, reduction="sum")
    rot_n = rot / torch.sqrt((rot * rot).sum(dim=1, keepdim=True) + 1e-10)
    zf = _t(labels["zoom_factor"])
    trans_est = torch.stack([ztrans[:, 0] * zf[:, 0], ztrans[:, 1] * zf[:, 0], ztrans[:, 2]], dim=1)  # invZoomTrans

    class T3D(torch.autograd.Function):
        @staticmethod
        def forward(ctx, q, t):
            ctx.save_for_backward(q, t)
            return _t(O.transform3d_forward(labels["point_cloud_model"], q.detach().numpy(), t.detach().numpy(),
                                            labels["src_pose"], (0, 0, 0), (1, 1, 1), "camera"))

        @staticmethod
        def backward(ctx, g):
            q, t = ctx.saved_tensors
            rg, tg = O.transform3d_backward(g.numpy(), labels["point_cloud_model"], q.detach().numpy(), t.detach().numpy(),
                                            labels["src_pose"], (0, 0, 0), (1, 1, 1), "camera")
            return _t(rg), _t(tg)

    # b_zoom_grad=False: ZoomTrans backward passes the gradient through unscaled (zoom_trans.py:48-74)
    class InvZoomNoGradScale(torch.autograd.Function):
        @staticmethod
        def forward(ctx, zt):
            return trans_est.detach().clone()

        @staticmethod
        def backward(ctx, g):
            return g

    trans_for_t3d = InvZoomNoGradScale.apply(ztrans)
    pts_est = T3D.apply(rot_n, trans_for_t3d)
    pm = _t(labels["point_cloud_weights"]) * torch.abs((pts_est - _t(labels["point_cloud_observed"])) / NORMALIZE_3D_POINT)
    gs_flow, gs_pm, gs_mask = LW_FLOW / (Himg * Wimg), LW_PM / NUM_3D_SAMPLE, LW_MASK / (Himg * Wimg)
    objective = gs_flow * flow_loss.sum() + gs_pm * pm.sum() + gs_mask * mask_bce
    grads = {}
    if requires_grad:
        objective.backward()
        grads = {k: (v.grad.numpy().copy() if v.grad is not None else np.zeros(v.shape, np.float32)) for k, v in P.items()}
        for name, z in pre.items():  # gradients wrt the pre-activation conv outputs (debugging aid for the device backward)
            grads["dz_" + name] = z.grad.numpy().copy()
    out = {
        "rot_est_norm": rot_n.detach().numpy(), "rot_raw": rot.detach().numpy(), "zoom_trans_est": ztrans.detach().numpy(),
        "trans_est": trans_est.detach().numpy(),
        "flow_est_crop": flow_full.detach().numpy(), "flow_est": (flow_full * NORMALIZE_FLOW).detach().numpy(),
        "flow_loss": flow_loss.detach().numpy(), "mask_prob": torch.sigmoid(mask_logit).detach().numpy(),
        "mask_logit": mask_logit.detach().numpy(), "point_matching_loss": pm.detach().numpy(),
        "points_est": pts_est.detach().numpy(), "objective": float(objective.detach()),
        "flow6": flow6.detach().numpy(), "flow5": flow5.detach().numpy(), "flow4": flow4.detach().numpy(),
        "mask4": mask4.detach().numpy(), "concat2": cat2.detach().numpy(), "concat3": cat3.detach().numpy(),
    }
    return out, grads


def zoom_inputs(batch, K, means_rgb):
    """The zoom front of get_train_symbol (symbol:391-489) via the numpy/C oracle; a batch that carries depth_observed and
    depth_rendered (B,1,H,W metres: the RGB-D network) also gets them zoomed with ZoomDepth by the pair's zoom factor."""
    zo, zg, zr, zf, bbox = O.zoom_mask(batch["mask_observed"], batch["mask_gt_observed"], batch["mask_rendered"],
                                       batch["src_pose"].astype(np.float32), K)
    zio, zir = O.zoom_image_with_factor(zf, batch["image_observed"], batch["image_rendered"],
                                        np.asarray(means_rgb, np.float32))
    zfl, zfw = O.zoom_flow(zf, batch["flow"], batch["flow_weights"], False)
    zin = {"zoom_image_observed": zio, "zoom_image_rendered": zir, "zoom_mask_observed": zo, "zoom_mask_rendered": zr}
    if "depth_observed" in batch:
        zin["zoom_depth_observed"] = O.zoom_depth(zf, batch["depth_observed"])
        zin["zoom_depth_rendered"] = O.zoom_depth(zf, batch["depth_rendered"])
    labels = {"zoom_factor": zf, "zoom_flow": zfl, "zoom_flow_weights": zfw, "zoom_mask_gt_observed": zg,
              "src_pose": batch["src_pose"].astype(np.float32), "bbox": bbox,
              "point_cloud_model": batch["point_cloud_model"], "point_cloud_weights": batch["point_cloud_weights"],
              "point_cloud_observed": batch["point_cloud_observed"],
              "zoom_trans_gt": O.zoom_trans(zf, batch["trans"].astype(np.float32), False)}
    return zin, labels


def forward_backward(weights, batch, K, means_rgb, requires_grad=True, num_threads=None, input_mask=True):
    """The train symbol on a batch: zoom front, graph, unzoomed mask prediction.  input_mask=False is the image-only
    network with PRED_MASK (deepIM_flownet.py:391): the ZoomMask front and the mask labels stay, only conv1's input
    loses the masks.  Returns (outputs, grads, zin, labels); zin holds every zoomed blob, masks included."""
    zin, labels = zoom_inputs(batch, K, means_rgb)
    net_in = zin if input_mask else {k: v for k, v in zin.items() if not k.startswith("zoom_mask_")}
    out, grads = graph(weights, net_in, labels, requires_grad, num_threads)
    out["zoom_factor"] = labels["zoom_factor"]
    out["mask_pred_bin"] = np.round(out["mask_prob"])  # mx.sym.round: half away from zero; prob in (0,1)
    out["unzoomed_mask_pred"] = O.zoom_mask_with_factor(labels["zoom_factor"], out["mask_pred_bin"], True)
    return out, grads, zin, labels


def sgd_update(weights, mom, grads, lr=1e-4, momentum=0.975, wd=5e-4, rescale_grad=1.0):
    """MXNet SGD with momentum (train.py:296-304); in place on `weights` / `mom` (dict name -> float32 array)."""
    for k, w in weights.items():
        if k in FROZEN:
            continue
        g = rescale_grad * grads[k] + (wd * w if k.endswith("_weight") else 0.0)
        mom[k] = (np.float32(momentum) * mom[k] - np.float32(lr) * g).astype(np.float32)
        w += mom[k]


def test_forward_full(weights, image_observed, image_rendered, mask_observed, mask_rendered, src_pose, K, means_rgb):
    """Non-FAST_TEST test graph (get_test_symbol_share, deepIM_flownet.py:548-735): se3, mask_observed_pred (invZoomMask of
    the sigmoid mask, rounded), flow_est (invZoomFlow of the upsampled flow x NORMALIZE_FLOW) and the zoomed intermediates."""
    zo, _, zr, zf, bbox = O.zoom_mask(mask_observed, mask_observed, mask_rendered, src_pose.astype(np.float32), K)
    zio, zir = O.zoom_image_with_factor(zf, image_observed, image_rendered, np.asarray(means_rgb, np.float32))
    B, _, H, W = zio.shape
    zin = {"zoom_image_observed": zio, "zoom_image_rendered": zir, "zoom_mask_observed": zo, "zoom_mask_rendered": zr}
    z1 = np.zeros((B, 3, 1), np.float32)
    labels = {"zoom_factor": zf, "zoom_flow": np.zeros((B, 2, H, W), np.float32), "zoom_flow_weights": np.zeros((B, 2, H, W), np.float32),
              "zoom_mask_gt_observed": np.zeros((B, 1, H, W), np.float32), "src_pose": src_pose.astype(np.float32),
              "point_cloud_model": z1, "point_cloud_weights": z1, "point_cloud_observed": z1}
    out, _ = graph(weights, zin, labels, requires_grad=False)
    mask_pred = np.round(O.zoom_mask_with_factor(zf, out["mask_prob"], True))
    flow_est, _ = O.zoom_flow(zf, out["flow_est"], None, True)
    return {"se3": np.concatenate([out["rot_raw"], out["trans_est"]], axis=1), "zoom_factor": zf, "mask_observed_pred": mask_pred,
            "flow_est": flow_est, "zoom_mask_observed_pred": out["mask_prob"], "zoom_flow_est": out["flow_est"], "bbox": bbox}
