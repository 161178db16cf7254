"""GPU: the training step's prediction heads, losses and pose-head backward, kernel by kernel against float64.

The counterpart of tests/test_gpu_train_kernels.py for the kernels that produce the five tensors every gradient of the
step starts from (dflow4, dmask4, dflow5, dflow6, dh6) and for the forward values they come from.  One forward_backward
per case, then each kernel is recomputed in float64 (torch on the GPU, written from deepIM_flownet.py:120-350 and
transform3d.py, not from the CUDA) from exactly the operands the device stored: the decoder buffers and fp32 maps
(dim_train_debug_tensor ids 0-15), the pose heads' intermediates (ids 30-41), the step's labels and the fp32 master
weights.  Each result is held element by element to |dev - ref| <= rho |ref| + kappa 2^-24 S (tests/kernel_ref.py).

Kernel -> test:
  thin_conv_fwd_kernel<CO, S3>: flow6, flow5, flow4, mask4                        test_thin_conv_forward
  thin_deconv_fwd_kernel: cat2[1024:1026], cat3[768:770]                         test_upsample_flow_forward
  copy_interior_kernel: cat2[:512], cat3[:512], act10b; padding channels zero   test_copied_channels
  fullres_loss_kernel: flow_est, mask_prob, dfull                                test_fullres_heads
  loss_final_kernel (+ the loss partials of fullres_loss / pm_loss)              test_losses
  head_kernel's fc7 / rot / trans in the training forward: h7, rot_raw, ztrans   test_pose_heads_forward
  pose_head_fwd_kernel: rot_n, trans_est                                         test_pose_heads_forward
  transform3d_fwd_kernel (pts_est), pm_loss_kernel (dpts),
  transform3d_bwd_kernel (drot_n, dtrans)                                        test_point_matching
  upsample_bwd_kernel: dflow4, dmask4 (+ the frozen upsampling weights' zero gradient)  test_upsample_backward
  thin_deconv_bwd_kernel: dflow5, dflow6; thin_deconv_wgrad_kernel: upsample_flow5to4 /
  upsample_flow6to5 weight and bias gradients                                    test_upsample_flow_backward
  pose_head_bwd_kernel (drot), fc_heads_bwd_kernel (dh7, dh6),
  fc_wgrad_kernel (rot, trans, fc7 weights and biases)                           test_pose_heads_backward
  pack_thin_kernel and the head parameters that alias the master vector: every forward check of the case after an update
The step's other kernels are held to float64 by tests/test_gpu_train_kernels.py (conv tower data and weight gradients,
deconvolution parity classes, decoder canvases, thin weight gradients, fc6, bias gradients) and the conv tower's forward
by tests/test_gpu_conv1.py.

Cases: the mask network (max_batch 4) in bf16 and bf16x3 at B = 4, B = 3 after B = 4 (image 3 of every buffer is stale
and must not reach a sum over B) and B = 1; B = 16; the image-only and RGB-D networks at B = 3; a non-default
dim_train_config (loss weights, normalisers, trans_means / trans_stds, rot_coord MODEL); a step after one SGD update; and
edge inputs built into the batch: an image with all-zero flow weights, mask logits saturated by mask_conv3_bias = +-40,
point weights of zero on a subset of points, pc_observed equal to the device's own pts_est on another subset (taken from
a first identical step), N = 1000 (not a multiple of 256) and N = 1.  Every pixel of the full-resolution and 1/16 maps
is checked, borders included; a failure names the pixel."""
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

import torch.nn.functional as F  # noqa: E402

import kernel_ref as R  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.trainer import Trainer, make_device_batch  # noqa: E402

K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB

# kappa per kernel family: 4 x the largest (|err| - rho |ref|) / (2^-24 S) observed over every case of this file, rounded
# up to two digits and at least 1 ("obs"; measured on an H100 80GB HBM3 at a 400 W power limit).  The module prints what
# each family needed when it finishes (pytest -s).
KAPPA = {
    "thin_fwd": 4.1,            # obs 1.003  thin_conv_fwd_kernel: flow6, flow5, flow4, mask4
    "thin_deconv": 21,          # obs 5.085  thin_deconv_fwd_kernel (cat2 / cat3 flow channels), thin_deconv_bwd_kernel
    "fullres": 16,              # obs 4.0    fullres_loss_kernel: flow_est, mask_prob, dfull
    "loss": 4.6,                # obs 1.14   fullres_loss / pm_loss partials + loss_final_kernel
    "heads": 7.3,               # obs 1.823  head_kernel's fc7 / rot / trans, pose_head_fwd_kernel
    "transform3d": 8.8,         # obs 2.199  transform3d_fwd_kernel, transform3d_bwd_kernel
    "pm": 1,                    # obs 0.18   pm_loss_kernel: dpts
    "upsample_bwd": 21,         # obs 5.155  upsample_bwd_kernel
    "thin_deconv_wgrad": 7.1,   # obs 1.761  thin_deconv_wgrad_kernel
    "heads_bwd": 30,            # obs 7.287  pose_head_bwd_kernel, fc_heads_bwd_kernel, fc_wgrad_kernel
}

# a dim_train_config far from the defaults; dyadic values, so the fp32 config holds them exactly
CONFIG = {"lw_flow": 0.5, "lw_mask": 0.0625, "lw_pm": 0.375, "num_3d_sample": 1536.0, "normalize_3d_point": 0.25,
          "normalize_flow": 16.0, "trans_means": (0.0625, -0.125, 0.03125), "trans_stds": (0.5, 2.0, 0.75),
          "rot_coord": "MODEL"}

# (context, precision, batch sizes run in order on one context -- the last one is checked, options)
CASES = [("mask", "bf16", (4,), {}), ("mask", "bf16", (4, 3), {}), ("mask", "bf16", (1,), {}),
         ("mask", "bf16x3", (4,), {}), ("mask", "bf16x3", (4, 3), {}), ("mask", "bf16x3", (1,), {}),
         ("mask", "bf16", (4,), {"config": CONFIG}),
         ("mask", "bf16", (4, 4), {"update": True}),
         ("mask16", "bf16", (16,), {}),
         ("nomask", "bf16", (3,), {}), ("rgbd", "bf16", (3,), {}),
         ("sat+", "bf16", (3,), {"edge": True, "N": 1000}),
         ("sat-", "bf16x3", (3,), {"edge": True, "N": 1000}),
         ("sat-", "bf16", (2,), {"N": 1})]
MAXB = {"mask": 4, "mask16": 16, "nomask": 3, "rgbd": 3, "sat+": 4, "sat-": 4}
NET = {"mask16": "mask", "sat+": "mask", "sat-": "mask"}
MASK_BIAS = {"sat+": 40.0, "sat-": -40.0}  # mask_conv3_bias: logits far into both saturated ends of the sigmoid


def case_id(c):
    key, prec, sched, opt = c
    return "%s-%s-B%s%s" % (key, prec, "-".join(map(str, sched)), "".join("-" + k for k in sorted(opt) if k != "N")
                            + ("-N%d" % opt["N"] if "N" in opt else ""))


class Nets:
    """one open context at a time (the cases of a context are consecutive)"""

    def __init__(self):
        self.key, self.ctx, self.tr = None, None, None
        self.meshes = [synth.make_cube(), synth.make_blob()]

    def open(self, key):
        if key != self.key:
            self.close()
            net = NET.get(key, key)
            ctx = Context(0, max_batch=MAXB[key], max_classes=2, max_verts=6000, max_faces=11000,
                          input_mask=net != "nomask", input_depth=net == "rgbd")
            for i, m in enumerate(self.meshes):
                ctx.upload_mesh(i, m)
            w = synth.make_train_weights(0, input_mask=net != "nomask", input_depth=net == "rgbd")
            # the frozen upsampling kernels are the same bilinear kernel in every group; give each group (and the mask) its
            # own, so that a kernel reading another group's weights shows
            rng = np.random.default_rng(7)
            for k in ("upsampling_weight", "mask_upsampling_weight"):
                w[k] = (w[k] * rng.uniform(0.5, 1.5, w[k].shape)).astype(np.float32)
            if key in MASK_BIAS:
                w["mask_conv3_bias"] = np.full_like(w["mask_conv3_bias"], MASK_BIAS[key])
            self.key, self.ctx, self.tr = key, ctx, Trainer(ctx, w)
        return self.ctx, self.tr

    def close(self):
        if self.ctx is not None:
            self.ctx.close()
        self.key, self.ctx, self.tr = None, None, None


@pytest.fixture(scope="module")
def nets():
    n = Nets()
    yield n
    n.close()
    print("\nkernel families, largest kappa needed: " + json.dumps({k: float("%.4g" % v) for k, v in sorted(R.OBSERVED.items())}))


@pytest.fixture(scope="module", params=CASES, ids=[case_id(c) for c in CASES])
def run(request, nets):
    key, prec, sched, opt = request.param
    net = NET.get(key, key)
    ctx, tr = nets.open(key)
    tr.set_precision(prec)
    cfg0 = ctx.get_config()
    if "config" in opt:
        ctx.set_config(**opt["config"])
    try:
        for i, B in enumerate(sched):
            batch = make_device_batch(ctx, nets.meshes, B, 11 + B, K, MEANS, num_points=opt.get("N", 3000),
                                      input_depth=net == "rgbd")[0]
            z = tr.zoom_front(batch, K)
            pts_first = None
            if opt.get("edge"):
                z["zoom_flow_weights"][0].zero_()              # image 0: no flow label at all
                z["point_cloud_weights"][:, :, 0::5] = 0        # a subset of points without weight
                tr.forward_backward(z)                          # the same step once more: its pts_est becomes the label
                torch.cuda.synchronize()
                pts_first = torch.from_numpy(tr.debug_tensor(35)[:B]).cuda()
                z["point_cloud_observed"][:, :, 2::5] = pts_first[:, :, 2::5]
            out = tr.forward_backward(z)
            torch.cuda.synchronize()
            if opt.get("update") and i + 1 < len(sched):
                tr.update(lr=1e-2)  # large enough that a head reading the old weights is off by far more than the bound
                torch.cuda.synchronize()
        r = R.Run(net, prec, sched[-1], ctx, tr)
        r.z, r.out, r.cfg, r.edge, r.pts_first = z, out, ctx.get_config(), bool(opt.get("edge")), pts_first
        yield r
    finally:
        ctx.set_config(**cfg0)
        tr.set_precision("bf16")


def collect(checks):
    """run every check, report all failures together"""
    errs = []
    for f in checks:
        try:
            f()
        except AssertionError as e:
            errs.append(str(e))
    assert not errs, "\n".join(errs)


def tag(run):
    return " (%s, B=%d, %s)" % (run.net, run.B, run.prec)


def label(run, name):
    """a label of the step (zoom_front output) as float64 [B, ...]"""
    return run.z[name][:run.B].to(torch.float64)


def dbg(run, tid):
    """an fp32 pose-head / loss intermediate (ids 30-41) of the batch's images as float64"""
    return R.gpu(run.tbuf(tid)[:run.B])


def where_row(what):
    return lambda idx: "(image %d, %s %d)" % (idx[0], what, idx[1])


def where_point(idx):
    return "(image %d, axis %d, point %d)" % idx


# ------------------------------------------------------------------------------------------------- forward
def test_thin_conv_forward(run):
    """thin_conv_fwd_kernel<CO, S3>: the 3x3 pad-1 convolutions + bias Convolution1 (flow6 from act10b), Convolution2
    (flow5 from cat2[:1026]), Convolution3 and mask_conv3 (flow4, mask4 from cat3[:770]), fp32 weights"""
    def one(name, x, tid):
        ref, S = R.products(lambda a, w: F.conv2d(a, w, padding=1), R.fused(x), run.w32(name + "_weight"))
        b = R.gpu(run.params[name + "_bias"])[None, :, None, None]
        R.check("thin_fwd", name + tag(run), run.fp32(tid), ref + b, S + b.abs(), 0.0, KAPPA["thin_fwd"], R.at_pixel)
    collect([lambda: one("Convolution1", run.pair(15, 0, 1024), 0), lambda: one("Convolution2", run.pair(10, 0, 1026), 1),
             lambda: one("Convolution3", run.pair(11, 0, 770), 2), lambda: one("mask_conv3", run.pair(11, 0, 770), 3)])


def test_upsample_flow_forward(run):
    """thin_deconv_fwd_kernel: cat2[1024:1026] = upsample_flow6to5(flow6) and cat3[768:770] = upsample_flow5to4(flow5),
    k4 s2 deconvolutions + bias cropped by 1, stored as bf16 (bf16x3: a pair)"""
    def one(name, x, cat, c0, hw):
        ref, S = R.deconv_fwd((x, None), run.w32(name + "_weight"), *hw)
        b = R.gpu(run.params[name + "_bias"])[None, :, None, None]
        R.check("thin_deconv", "%s -> buffer %d [%d:%d]%s" % (name, cat, c0, c0 + 2, tag(run)), R.fused(run.pair(cat, c0, c0 + 2))[0],
                ref + b, S + b.abs(), run.rho, KAPPA["thin_deconv"], R.at_pixel)
    collect([lambda: one("upsample_flow6to5", run.fp32(0), 10, 1024, run.sizes[8]),
             lambda: one("upsample_flow5to4", run.fp32(1), 11, 768, run.sizes[6])])


def test_copied_channels(run):
    """copy_interior_kernel: cat2[:512] is act[8], cat3[:512] is act[6] and act10b is act[10], bit for bit in both halves;
    the padding channels cat2[1026:1088] and cat3[770:832] hold exact zeros (whole buffer, both halves)"""
    errs = []
    for tid, c1, i in ((10, 512, 8), (11, 512, 6), (15, 1024, 10)):
        for h, (dev, src) in enumerate(zip(run.pair(tid, 0, c1), run.act(i))):
            if src is not None and not torch.equal(dev, src):
                bad = (dev != src).nonzero()[0].tolist()
                errs.append("buffer %d [:%d] (%s) differs from act[%d] first at %s" % (tid, c1, "lo" if h else "hi", i, R.at_pixel(bad)))
    for tid, c0 in ((10, 1026), (11, 770)):
        for lo in ((False, True) if run.s3 else (False,)):
            if run.tbuf(tid, lo)[0][:run.B, :, :, c0:].any():
                errs.append("buffer %d padding channels %d+ (%s) are not zero" % (tid, c0, "lo" if lo else "hi"))
    assert not errs, "; ".join(errs)


def fullres(run):
    """float64 of fullres_loss_kernel from the stored flow4 / mask4: the upsampled flow v_f and logit v_m with their S,
    the sigmoid and its S (the documented __expf error, 2 + floor(1.173 |x|) ulp, built in), the flow difference"""
    def f():
        H, W = run.ctx.H, run.ctx.W
        wf, wm = R.gpu(run.params["upsampling_weight"]), R.gpu(run.params["mask_upsampling_weight"])
        flow4, mask4 = run.fp32(2), run.fp32(3)
        vf, Svf = R.upsample_fwd(flow4, wf, H, W), R.upsample_fwd(flow4.abs(), wf.abs(), H, W)
        vm, Svm = R.upsample_fwd(mask4, wm, H, W), R.upsample_fwd(mask4.abs(), wm.abs(), H, W)
        ulp_exp = 2 + torch.floor(1.173 * vm.abs())  # __expf(-v), in ulp of its result (<= 2 units of 2^-24 relative)
        sig = torch.sigmoid(vm)
        Ssig = sig * (1 - sig) * (Svm + 2 * ulp_exp) + sig
        nf = run.cfg["normalize_flow"]
        zfl, zfw, lab = label(run, "zoom_flow"), label(run, "zoom_flow_weights"), label(run, "zoom_mask_gt_observed")
        d, Sd = vf - zfl / nf, Svf + zfl.abs() / nf
        return dict(vf=vf, Svf=Svf, vm=vm, Svm=Svm, sig=sig, Ssig=Ssig, ulp_exp=ulp_exp, d=d, Sd=Sd, zfw=zfw, lab=lab, nf=nf,
                    gs_flow=run.cfg["lw_flow"] / (H * W), gs_mask=run.cfg["lw_mask"] / (H * W))
    return run._cached("fullres", f)


def test_fullres_heads(run):
    """fullres_loss_kernel: the grouped bilinear k32 s16 deconvolution cropped at offset 8 -> flow_est (x NORMALIZE_FLOW),
    mask_prob (sigmoid) and dfull: gs_flow 2 w (v - flow / NORMALIZE_FLOW) on the flow channels, gs_mask (sigmoid - y) on
    the mask channel.  An image with all-zero flow weights has an exactly zero flow gradient."""
    r = fullres(run)
    dfull = dbg(run, 41)
    ref = torch.cat([r["gs_flow"] * 2 * r["zfw"] * r["d"], r["gs_mask"] * (r["sig"] - r["lab"])], 1)
    S = torch.cat([r["gs_flow"] * 2 * r["zfw"].abs() * (r["d"].abs() + r["Sd"]), r["gs_mask"] * (r["Ssig"] + (r["sig"] - r["lab"]).abs())], 1)
    checks = [lambda: R.check("fullres", "flow_est" + tag(run), run.out["flow_est"][:run.B], r["vf"] * r["nf"], r["Svf"] * r["nf"], 0.0,
                              KAPPA["fullres"], R.at_pixel),
              lambda: R.check("fullres", "mask_prob" + tag(run), run.out["mask_prob"][:run.B], r["sig"], r["Ssig"], 0.0, KAPPA["fullres"],
                              R.at_pixel),
              lambda: R.check("fullres", "dfull" + tag(run), dfull, ref, S, 0.0, KAPPA["fullres"], R.at_pixel)]
    if run.edge:
        def zero_image():
            assert not r["zfw"][0].any()
            assert not dfull[0, :2].any(), "dfull of the image without flow weights is not zero"
        checks.append(zero_image)
    collect(checks)


def point_matching(run):
    """float64 of the point-matching loss from the stored pts_est: the per-element loss and dpts"""
    def f():
        est, obs, pw = dbg(run, 35), label(run, "point_cloud_observed"), label(run, "point_cloud_weights")
        norm, gs = run.cfg["normalize_3d_point"], run.cfg["lw_pm"] / run.cfg["num_3d_sample"]
        return R.pm_loss(est, obs, pw, norm), R.pm_loss_grad(est, obs, pw, norm, gs)
    return run._cached("pm", f)


def test_losses(run):
    """loss_final_kernel (with the per-block partials of fullres_loss_kernel and pm_loss_kernel): losses = [sum w (v -
    flow / NORMALIZE_FLOW)^2, sum pw |d| / NORMALIZE_3D_POINT, sum BCE-with-logits, gs_flow f + gs_pm p + gs_mask m],
    each bounded by the magnitudes of its summands"""
    r = fullres(run)
    d, Sd, zfw, vm, lab = r["d"], r["Sd"], r["zfw"], r["vm"], r["lab"]
    f, Sf = (zfw * d * d).sum(), (zfw.abs() * (d * d + 2 * d.abs() * Sd)).sum()
    e = torch.exp(-vm.abs())
    m = (vm.clamp_min(0) - vm * lab + torch.log1p(e)).sum()
    Sm = (vm.clamp_min(0) + (vm * lab).abs() + torch.log1p(e) + (r["sig"] - lab).abs() * r["Svm"]
          + 2 * r["ulp_exp"] * e / (1 + e)).sum()
    pm = point_matching(run)[0]
    p, Sp = pm.sum(), pm.abs().sum()
    gs_pm = run.cfg["lw_pm"] / run.cfg["num_3d_sample"]
    ref = torch.stack([f, p, m, r["gs_flow"] * f + gs_pm * p + r["gs_mask"] * m])
    S = torch.stack([Sf, Sp, Sm, r["gs_flow"] * Sf + gs_pm * Sp + r["gs_mask"] * Sm])
    names = ("flow loss", "point-matching loss", "mask BCE", "objective")
    R.check("loss", "losses" + tag(run), run.out["losses"], ref, S, 0.0, KAPPA["loss"], lambda idx: names[idx[0]])


def test_pose_heads_forward(run):
    """the training forward's fc7 / rot / trans (head_kernel, fp32, from the stored h6 and h7), pose_head_fwd_kernel:
    rot_n = L2Normalization(rot_raw) (eps 1e-10 inside the sqrt), trans_est = invZoomTrans(ztrans) (x, y scaled by the
    zoom factor's wx, zoom_trans.py:30-41)"""
    p = {k: R.gpu(v) for k, v in run.params.items() if k.split("_")[0] in ("fc7", "rot", "trans")}
    h6, h7, rot_raw, ztrans = run.fp32(8), dbg(run, 30), dbg(run, 31), dbg(run, 32)

    def fc(name, x, dev, lrelu):
        w, b = p[name + "_weight"], p[name + "_bias"]
        ref, S = x @ w.T + b, x.abs() @ w.abs().T + b.abs()
        R.check("heads", name + tag(run), dev, F.leaky_relu(ref, 0.1) if lrelu else ref, S, 0.0, KAPPA["heads"], where_row("output"))

    def rot_n():
        ref = R.l2_normalize(rot_raw)
        R.check("heads", "rot_n" + tag(run), dbg(run, 33), ref, ref.abs(), 0.0, KAPPA["heads"], where_row("component"))

    def trans_est():
        wx = label(run, "zoom_factor")[:, :1]
        ref = torch.cat([ztrans[:, :2] * wx, ztrans[:, 2:]], 1)
        R.check("heads", "trans_est" + tag(run), dbg(run, 34), ref, ref.abs(), 0.0, KAPPA["heads"], where_row("component"))
    collect([lambda: fc("fc7", h6, h7, True), lambda: fc("rot", h7, rot_raw, False), lambda: fc("trans", h7, ztrans, False),
             rot_n, trans_est])


def test_point_matching(run):
    """Transform3D in the step under the context's trans_means / trans_stds / rot_coord: pts_est from the stored rot_n and
    trans_est (transform3d_fwd_kernel); pm_loss_kernel: dpts = gs_pm w sign(d) / NORMALIZE_3D_POINT, sign(0) = 0; and the
    backward (transform3d_bwd_kernel) drot_n, dtrans from the stored dpts.  Edge case: dpts is exactly zero where the
    weight is zero and where pc_observed is the device's own pts_est."""
    cfg, tg = run.cfg, tag(run)
    P, ps = label(run, "point_cloud_model"), label(run, "src_pose")
    rot_n, trans_est, dpts = dbg(run, 33), dbg(run, 34), dbg(run, 36)
    t3d = (cfg["trans_means"], cfg["trans_stds"], cfg["rot_coord"])

    def forward():
        ref, S = R.transform3d_fwd(P, rot_n, trans_est, ps, *t3d)
        R.check("transform3d", "pts_est" + tg, dbg(run, 35), ref, S, 0.0, KAPPA["transform3d"], where_point)

    def grad():
        ref = point_matching(run)[1]
        R.check("pm", "dpts" + tg, dpts, ref, ref.abs(), 0.0, KAPPA["pm"], where_point)

    def backward():
        (rg, Srg), (tr_, Str) = R.transform3d_bwd(dpts, P, rot_n, trans_est, ps, *t3d)
        R.check("transform3d", "drot_n" + tg, dbg(run, 37), rg, Srg, 0.0, KAPPA["transform3d"], where_row("component"))
        R.check("transform3d", "dtrans" + tg, dbg(run, 38), tr_, Str, 0.0, KAPPA["transform3d"], where_row("component"))
    checks = [forward, grad, backward]
    if run.edge:
        def edge():
            assert torch.equal(dbg(run, 35), run.pts_first.double()), "pts_est differs between two identical steps"
            assert not dpts[:, :, 0::5].any(), "dpts is not zero where the point weight is"
            assert not dpts[:, :, 2::5].any(), "dpts is not zero where pc_observed equals pts_est"
        checks.append(edge)
    collect(checks)


# ------------------------------------------------------------------------------------------------- backward
def test_upsample_backward(run):
    """upsample_bwd_kernel: dflow4 / dmask4 = the adjoint of the upsampling (each 1/16 location sums its 32 x 32 footprint
    of dfull, clipped at the image border); the frozen upsampling kernels get exactly zero gradients"""
    dfull = dbg(run, 41)
    h4, w4 = run.sizes[6]

    def one(name, c0, c1, wname, tid):
        w = R.gpu(run.params[wname])
        ref, S = R.upsample_bwd(dfull[:, c0:c1], w, h4, w4), R.upsample_bwd(dfull[:, c0:c1].abs(), w.abs(), h4, w4)
        R.check("upsample_bwd", name + tag(run), run.fp32(tid), ref, S, 0.0, KAPPA["upsample_bwd"], R.at_pixel)

    def frozen():
        for k in ("upsampling_weight", "mask_upsampling_weight"):
            assert not run.grads[k].any(), k
    collect([lambda: one("dflow4", 0, 2, "upsampling_weight", 4), lambda: one("dmask4", 2, 3, "mask_upsampling_weight", 5), frozen])


def test_upsample_flow_backward(run):
    """thin_deconv_bwd_kernel: dflow5 from the final dcat3[768:770], dflow6 from the final dcat2[1024:1026];
    thin_deconv_wgrad_kernel: upsample_flow5to4 / upsample_flow6to5 weight (from flow5 / flow6) and bias gradients"""
    tg = tag(run)

    def one(name, x, cat, c0, hw, tid):
        d = R.fused(run.pair(cat, c0, c0 + 2))
        ref, S = R.deconv_dgrad(d, run.w32(name + "_weight"), *hw)
        R.check("thin_deconv", "d input of " + name + tg, run.fp32(tid), ref, S, 0.0, KAPPA["thin_deconv"], R.at_pixel)
        ref, S = R.deconv_wgrad((x, None), d)
        R.check("thin_deconv_wgrad", name + "_weight" + tg, run.grads[name + "_weight"], ref, S, 0.0, KAPPA["thin_deconv_wgrad"])
        R.check("thin_deconv_wgrad", name + "_bias" + tg, run.grads[name + "_bias"], d[0].sum((0, 2, 3)), d[0].abs().sum((0, 2, 3)),
                0.0, KAPPA["thin_deconv_wgrad"])
    collect([lambda: one("upsample_flow5to4", run.fp32(1), 13, 768, run.sizes[8], 6),
             lambda: one("upsample_flow6to5", run.fp32(0), 12, 1024, run.sizes[10], 7)])


def test_pose_heads_backward(run):
    """pose_head_bwd_kernel: drot = L2Normalization's backward of drot_n; fc_heads_bwd_kernel: dh7 = mask(h7) (drot W_rot +
    dtrans W_trans) (invZoomTrans passes dtrans through: b_zoom_grad False), dh6 = mask(h6) dh7 W_fc7, the LeakyReLU mask
    from the stored sign; fc_wgrad_kernel: rot / trans / fc7 weight and bias gradients, sums over the batch's B images"""
    tg = tag(run)
    p = {k: R.gpu(v) for k, v in run.params.items() if k.split("_")[0] in ("fc7", "rot", "trans")}
    h6, h7, drot_n, dtrans, drot, dh7 = run.fp32(8), dbg(run, 30), dbg(run, 37), dbg(run, 38), dbg(run, 39), dbg(run, 40)

    def pose():
        rot_raw = dbg(run, 31)
        ref = R.l2_normalize_bwd(rot_raw, drot_n)
        n = torch.sqrt((rot_raw * rot_raw).sum(1, keepdim=True) + R.L2_EPS)
        y = rot_raw / n
        S = (drot_n.abs() + y.abs() * (y * drot_n).abs().sum(1, keepdim=True)) / n
        R.check("heads_bwd", "drot" + tg, drot, ref, S, 0.0, KAPPA["heads_bwd"], where_row("component"))

    def data():
        m7, m6 = R.lrelu_mask(h7), R.lrelu_mask(h6)
        wr, wt, w7 = p["rot_weight"], p["trans_weight"], p["fc7_weight"]
        ref, S = (drot @ wr + dtrans @ wt) * m7, (drot.abs() @ wr.abs() + dtrans.abs() @ wt.abs()) * m7
        R.check("heads_bwd", "dh7" + tg, dh7, ref, S, 0.0, KAPPA["heads_bwd"], where_row("unit"))
        R.check("heads_bwd", "dh6" + tg, run.fp32(9), (dh7 @ w7) * m6, (dh7.abs() @ w7.abs()) * m6, 0.0, KAPPA["heads_bwd"],
                where_row("unit"))

    def wgrad(name, dy, x):
        R.check("heads_bwd", name + "_weight" + tg, run.grads[name + "_weight"], dy.T @ x, dy.abs().T @ x.abs(), 0.0,
                KAPPA["heads_bwd"], lambda idx: "(output %d, input %d)" % idx)
        R.check("heads_bwd", name + "_bias" + tg, run.grads[name + "_bias"], dy.sum(0), dy.abs().sum(0), 0.0, KAPPA["heads_bwd"],
                lambda idx: "output %d" % idx)
    collect([pose, data, lambda: wgrad("rot", drot, h7), lambda: wgrad("trans", dtrans, h7), lambda: wgrad("fc7", dh7, h6)])


def test_debug_ids_of_the_heads(run):
    """dim_train_debug_tensor ids 30-41: fp32 only (100 + id is refused, there is no lo half), requests past the buffer
    are refused, and dim_train_debug_geometry reports zeros for them"""
    import ctypes as C
    from deepim_b200._capi import lib
    h, B = run.ctx._h, run.ctx.max_batch
    sizes = {30: B * 256, 31: B * 4, 32: B * 3, 33: B * 4, 34: B * 3, 37: B * 4, 38: B * 3, 39: B * 4, 40: B * 256,
             41: B * 3 * run.ctx.H * run.ctx.W}
    buf = np.empty(max(sizes.values()) + 1, np.float32)
    p = buf.ctypes.data_as(C.c_void_p)
    for tid, n in sizes.items():
        assert lib.dim_train_debug_tensor(h, tid, p, 4 * n) == 0, tid
        assert lib.dim_train_debug_tensor(h, tid, p, 4 * n + 4) != 0, tid
        assert lib.dim_train_debug_tensor(h, 100 + tid, p, 4) != 0, tid
        geo = (C.c_int32 * 7)()
        lib.dim_train_debug_geometry(h, tid, geo)
        assert list(geo) == [0] * 7, tid
    for tid in (35, 36, 135, 136):
        assert (lib.dim_train_debug_tensor(h, tid, p, 4) == 0) == (tid < 100), tid
