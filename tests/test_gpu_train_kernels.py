"""GPU: the training step's kernels one by one, teacher-forced from the buffers the device stored, against float64.

One forward_backward per case, then every kernel of the backward pass (and the decoder's forward deconvolutions) is
recomputed in float64 from exactly the operands it read: act[i] (dim_debug_activation, hi + lo), the pre-activation
gradients gz[i] and the decoder buffers (dim_train_debug_tensor), the operand packs rounded from the fp32 master as the
repack rounds them, and the stored activation's sign as the LeakyReLU mask.  Each result is held element by element to
|dev - ref| <= rho |ref| + kappa 2^-24 S (tests/kernel_ref.py): no fraction of entries may leave the bound.

Cases: the mask network on a max_batch = 4 context in bf16 and bf16x3 at B = 4, B = 3 after B = 4 (image 3 of every
buffer is stale and must not be read) and B = 1 (the smallest K-slice count); a B = 16 bf16 step (the slice counts of a
full batch); the image-only and the RGB-D network at B = 3 (conv1's weight gradient with its dropped lanes, one encoder
data gradient: their other kernels are the mask network's)."""
import json

import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

import torch.nn.functional as F  # noqa: E402

import kernel_ref as R  # noqa: E402
from oracle import train_oracle as T  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.trainer import Trainer, make_device_batch  # noqa: E402

K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB

# kappa per kernel family: 4 x the largest (|err| - rho |ref| - slack) / (2^-24 S) observed over every case of this file,
# rounded up to two digits and at least 1 ("obs"; measured on an H100 80GB HBM3 at a 400 W power limit).  The module prints what each
# family needed when it finishes (pytest -s).
KAPPA = {
    **R.KAPPA_WGRAD,        # "wgrad", "conv1_wgrad": shared with tests/test_gpu_schedule.py
    "bias": 23,             # obs 5.5    bias_partial / bias_final
    "dgrad": 410,           # obs 100.9  conv_igemm_persistent_kernel, data-gradient parity classes (EPI = 1)
    "deconv_fwd": 70,       # obs 17.4   conv_igemm_persistent_kernel, deconvolution forward parity classes
    "decoder_dgrad": 98,    # obs 24.4   dcat2 / dcat3: deconv4's data gradient, the thin data gradients, the in-place mask
    "thin_wgrad": 47,       # obs 11.6   thin_conv_wgrad (+ final): Convolution1/2/3, mask_conv3
    "fc6": 25,              # obs 6.2    fc6_wgrad_kernel, fc_wgrad (fc6 bias), thin dgrad + fc6_dgrad_kernel into dA10p
    "fc6_fwd": 1.9,         # obs 0.46   fc6_mma_kernel + head_kernel's fc6 sum: h6 (debug id 8) of the training forward
}

# (network, precision, batch sizes run in order on one context; the last one is checked)
CASES = [("mask", "bf16", (4,)), ("mask", "bf16", (4, 3)), ("mask", "bf16", (3, 1)),
         ("mask", "bf16x3", (4,)), ("mask", "bf16x3", (4, 3)), ("mask", "bf16x3", (3, 1)),
         ("mask16", "bf16", (16,)),
         ("nomask", "bf16", (3,)), ("nomask", "bf16x3", (3,)),
         ("rgbd", "bf16", (3,)), ("rgbd", "bf16x3", (3,))]
MAXB = {"mask": 4, "mask16": 16, "nomask": 3, "rgbd": 3}
LAYERS = [(name, s, p) for name, s, p in T.ENC]


class Nets:
    """one open context at a time (the cases of a network are consecutive)"""

    def __init__(self):
        self.key, self.ctx, self.tr = None, None, None
        self.meshes = [synth.make_cube(), synth.make_blob()]

    def open(self, net):
        if net != self.key:
            self.close()
            ctx = Context(0, max_batch=MAXB[net], max_classes=2, max_verts=6000, max_faces=11000,
                          input_mask=net != "nomask", input_depth=net == "rgbd")
            for i, m in enumerate(self.meshes):
                ctx.upload_mesh(i, m)
            w = synth.make_train_weights(0, input_mask=net != "nomask", input_depth=net == "rgbd")
            self.key, self.ctx, self.tr = net, ctx, Trainer(ctx, w)
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


@pytest.fixture(scope="module", params=CASES, ids=["%s-%s-B%s" % (n, p, "-".join(map(str, s))) for n, p, s in CASES])
def run(request, nets):
    net, prec, sched = request.param
    ctx, tr = nets.open(net)
    tr.set_precision(prec)
    for B in sched:
        batch = make_device_batch(ctx, nets.meshes, B, 11 + B, K, MEANS, input_depth=net == "rgbd")[0]
        tr.forward_backward(tr.zoom_front(batch, K))
        torch.cuda.synchronize()
    yield R.Run(net, prec, sched[-1], ctx, tr)
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


def mask_only(run):
    if not run.net.startswith("mask"):
        pytest.skip("the %s network shares this kernel with the mask network" % run.net)


# ------------------------------------------------------------------------------------------------- weight gradients
def test_conv_weight_gradients(run):
    """conv_wgrad_kernel + wgrad_reduce (WG_CONV), conv2 ... conv6_1: dW = conv2d_weight(act[i], gz[i])"""
    mask_only(run)
    collect([lambda i=i: R.check_conv_wgrad(run, i) for i in range(1, 10)])


def test_conv1_weight_gradient(run):
    """flow_conv1's weight gradient (kernel_ref.check_conv1_wgrad): the row-GEMM kernel with WG_CONV1_ROW or, RGB-D, the
    generic kernel with WG_CONV1_RGBD"""
    R.check_conv1_wgrad(run)


def test_bias_gradients(run):
    """bias_partial / bias_final: the sum of a gradient buffer over the batch's pixels (every encoder layer; deconv5 /
    deconv4 over their slices of the final dcat2 / dcat3)"""
    def one(name, g):
        v = R.fused(g)[0]
        R.check("bias", "%s (%s, B=%d, %s)" % (name, run.net, run.B, run.prec), run.grads[name], v.sum((0, 2, 3)),
                v.abs().sum((0, 2, 3)), 0.0, KAPPA["bias"], lambda idx: "channel %d" % idx[0])
    layers = range(10) if run.net.startswith("mask") else (0, 1)
    checks = [lambda i=i: one(LAYERS[i][0] + "_bias", run.pair(20 + i)) for i in layers]
    if run.net.startswith("mask"):
        checks += [lambda: one("deconv5_bias", run.pair(12, 512, 1024)), lambda: one("deconv4_bias", run.pair(13, 512, 768))]
    collect(checks)


def test_deconv_weight_gradients(run):
    """conv_wgrad_kernel + WG_DECONV: deconv5 from act10b and the final dcat2[512:1024], deconv4 from cat2[:1026] and the
    final dcat3[512:768]"""
    mask_only(run)
    collect([lambda n=n: R.check_deconv_wgrad(run, n) for n in ("deconv5_weight", "deconv4_weight")])


def test_thin_weight_gradients(run):
    """thin_conv_wgrad (CUDA cores, fp32 output gradients): Convolution1/2/3 and mask_conv3, weights and biases"""
    mask_only(run)

    def one(name, x, dy):
        ref, S = R.conv_wgrad(R.fused(x), (dy, None), 3, 1, 1)
        tag = " (B=%d, %s)" % (run.B, run.prec)
        R.check("thin_wgrad", name + "_weight" + tag, run.grads[name + "_weight"], ref, S, 0.0, KAPPA["thin_wgrad"])
        R.check("thin_wgrad", name + "_bias" + tag, run.grads[name + "_bias"], dy.sum((0, 2, 3)), dy.abs().sum((0, 2, 3)), 0.0,
                KAPPA["thin_wgrad"])
    collect([lambda: one("Convolution1", run.pair(15, 0, 1024), run.fp32(7)),
             lambda: one("Convolution2", run.pair(10, 0, 1026), run.fp32(6)),
             lambda: one("Convolution3", run.pair(11, 0, 770), run.fp32(4)),
             lambda: one("mask_conv3", run.pair(11, 0, 770), run.fp32(5))])


def test_fc6_gradients(run):
    """fc6 forward (h6 = LeakyReLU(act[10] W_fc6^T + b), the pack's passes), fc6_wgrad_kernel (dW = dh6^T act[10]), the fc6
    bias gradient (sum of dh6) and dA10p = Convolution1's data gradient of dflow6 (thin kernel, stored) + dh6 W_fc6
    (fc6_dgrad_kernel, read-add-store)"""
    mask_only(run)
    B, tag = run.B, " (B=%d, %s)" % (run.B, run.prec)
    dh6 = run.fp32(9)
    flat = lambda v: None if v is None else v.permute(0, 2, 3, 1).reshape(B, 81920)
    a10 = flat(R.fused(run.act(10))[0])

    def forward():
        z, S = R.products(lambda x, w: x @ w.T, tuple(flat(v) for v in run.act(10)), run.w_fc6())
        b = R.gpu(run.params["fc6_bias"])
        R.check("fc6_fwd", "h6" + tag, run.fp32(8), F.leaky_relu(z + b, 0.1), S + b.abs(), 0.0, KAPPA["fc6_fwd"],
                lambda idx: "(image %d, output %d)" % idx)

    def where_w(idx):
        o, kk = idx
        return "(out %d, y %d, x %d, channel %d)" % (o, kk // 10240, (kk // 1024) % 10, kk % 1024)

    def wgrad():
        R.check("fc6", "fc6_weight" + tag, R.fc6_nhwc(run.grads["fc6_weight"]), dh6.T @ a10, dh6.abs().T @ a10.abs(), 0.0,
                KAPPA["fc6"], where_w)

    def bias():
        R.check("fc6", "fc6_bias" + tag, run.grads["fc6_bias"], dh6.sum(0), dh6.abs().sum(0), 0.0, KAPPA["fc6"])

    def dgrad():
        h6, w6 = run.sizes[10]
        t, St = R.conv_dgrad((run.fp32(7), None), run.w32("Convolution1_weight"), (B, 1024, h6, w6), 1, 1)
        wf = R.fused(run.w_fc6())[0]
        nchw = lambda v: v.reshape(B, h6, w6, 1024).permute(0, 3, 1, 2)
        ref, S = t + nchw(dh6 @ wf), St + nchw(dh6.abs() @ wf.abs())
        R.check("fc6", "dA10p" + tag, R.fused(run.pair(14))[0], ref, S, run.rho, KAPPA["fc6"], R.at_pixel, slack=run.rho * t.abs())
    collect([forward, wgrad, bias, dgrad])


# ------------------------------------------------------------------------------------------------- data gradients
def test_encoder_data_gradients(run):
    """conv_igemm_persistent_kernel's data-gradient parity classes, layers 9 ... 1 -> gz[i-1] = mask(act[i]) *
    (conv2d_input(gz[i], W_i) + addend), the addend being dcat2[0:512] for conv6 and dcat3[0:512] for conv5
    (the image-only and RGB-D networks: layer 1)"""
    def one(i):
        name, s, p = LAYERS[i]
        Wi = run.w(name + "_weight")
        ref, S = R.conv_dgrad(run.pair(20 + i), Wi, (run.B, Wi[0].shape[1]) + run.sizes[i], s, p)
        add = {8: 12, 6: 13}.get(i)
        if add is not None:
            a = R.fused(run.pair(add, 0, 512))[0]
            ref, S = ref + a, S + a.abs()
        m = R.lrelu_mask(run.act(i)[0])
        R.check("dgrad", "gz[%d] = %s data gradient (%s, B=%d, %s)" % (i - 1, name, run.net, run.B, run.prec),
                R.fused(run.pair(20 + i - 1))[0], ref * m, S * m, run.rho, KAPPA["dgrad"], R.at_pixel)
    collect([lambda i=i: one(i) for i in (range(9, 0, -1) if run.net.startswith("mask") else (1,))])


def test_deconv5_data_gradient(run):
    """gz[9] = mask(act[10]) * (deconv5's data gradient of the final dcat2[512:1024] + dA10p)"""
    mask_only(run)
    h6, w6 = run.sizes[10]
    ref, S = R.deconv_dgrad(run.pair(12, 512, 1024), run.w("deconv5_weight"), h6, w6)
    a = R.fused(run.pair(14))[0]
    m = R.lrelu_mask(run.act(10)[0])
    R.check("dgrad", "gz[9] (B=%d, %s)" % (run.B, run.prec), R.fused(run.pair(29))[0], (ref + a) * m, (S + a.abs()) * m,
            run.rho, KAPPA["dgrad"], R.at_pixel)


def test_decoder_gradient_canvases(run):
    """The final dcat3 and dcat2, each written by several kernels in order:
    dcat3 = Convolution3's data gradient of dflow4 (stored), + mask_conv3's of dmask4 (read-add-store), then the
    LeakyReLU mask of cat3 on [512:768] in place;  dcat2 = deconv4's data gradient of dcat3[512:768] (stored), +
    Convolution2's of dflow5, then the mask of cat2 on [512:1024].  Every earlier stored value adds its own rounding."""
    mask_only(run)
    B, tag = run.B, " (B=%d, %s)" % (run.B, run.prec)

    def masked(pre, S, slack, cat, c0, c1):
        m = torch.ones_like(pre)
        m[:, c0:c1] = R.lrelu_mask(run.pair(cat, c0, c1)[0])
        stored_before_mask = torch.zeros_like(pre)
        stored_before_mask[:, c0:c1] = pre[:, c0:c1].abs()
        return pre * m, S, slack + run.rho * stored_before_mask

    def dcat3():
        h4, w4 = run.sizes[6]
        t1, S1 = R.conv_dgrad((run.fp32(4), None), run.w32("Convolution3_weight"), (B, 770, h4, w4), 1, 1)
        t2, S2 = R.conv_dgrad((run.fp32(5), None), run.w32("mask_conv3_weight"), (B, 770, h4, w4), 1, 1)
        ref, S, slack = masked(t1 + t2, S1 + S2, run.rho * t1.abs(), 11, 512, 768)
        R.check("decoder_dgrad", "dcat3" + tag, R.fused(run.pair(13, 0, 770))[0], ref, S, run.rho, KAPPA["decoder_dgrad"],
                R.at_pixel, slack=slack)

    def dcat2():
        h5, w5 = run.sizes[8]
        t1, S1 = R.deconv_dgrad(run.pair(13, 512, 768), run.w("deconv4_weight"), h5, w5)
        t2, S2 = R.conv_dgrad((run.fp32(6), None), run.w32("Convolution2_weight"), (B, 1026, h5, w5), 1, 1)
        ref, S, slack = masked(t1 + t2, S1 + S2, run.rho * t1.abs(), 10, 512, 1024)
        R.check("decoder_dgrad", "dcat2" + tag, R.fused(run.pair(12, 0, 1026))[0], ref, S, run.rho, KAPPA["decoder_dgrad"],
                R.at_pixel, slack=slack)
    collect([dcat3, dcat2])


# ------------------------------------------------------------------------------------------------- forward
def test_deconv_forward(run):
    """conv_igemm_persistent_kernel's deconvolution parity classes: cat2[512:1024] = LeakyReLU(deconv5(act10b) + b) and
    cat3[512:768] = LeakyReLU(deconv4(cat2[:1026]) + b), both cropped by 1"""
    mask_only(run)

    def one(name, x, out, c0, c1, hw):
        ref, S = R.deconv_fwd(x, run.w(name + "_weight"), *hw)
        b = R.gpu(run.params[name + "_bias"])[None, :, None, None]
        R.check("deconv_fwd", "%s forward (B=%d, %s)" % (name, run.B, run.prec), R.fused(run.pair(out, c0, c1))[0],
                F.leaky_relu(ref + b, 0.1), S + b.abs(), run.rho, KAPPA["deconv_fwd"], R.at_pixel)
    collect([lambda: one("deconv5", run.pair(15, 0, 1024), 10, 512, 1024, run.sizes[8]),
             lambda: one("deconv4", run.pair(10, 0, 1026), 11, 512, 768, run.sizes[6])])


# ------------------------------------------------------------------------------------------------- borders
def test_buffer_borders_stay_zero(run):
    """the whole zero border (every side, full depth) of the gradient and decoder buffers and of the activations the
    backward pass reads, for the batch's images, both halves"""
    errs = []
    halves = (False, True) if run.s3 else (False,)
    tids = [20 + i for i in range(10)] + ([10, 11, 12, 13, 15] if run.net.startswith("mask") else [])
    for tid in tids:
        for lo in halves:
            buf, geo = run.tbuf(tid, lo)
            if not R.border_is_zero(buf, geo, run.B):
                errs.append("training buffer %d%s" % (tid, " (lo)" if lo else ""))
    for i in range(10):
        for lo in halves:
            buf, geo = run.act_raw(i, lo)
            if i == 0:
                buf = R.s2d_decode(buf).transpose(0, 2, 3, 1)  # the decoded canvas, NHWC
            if not R.border_is_zero(buf, geo, run.B):
                errs.append("act[%d]%s" % (i, " (lo)" if lo else ""))
    assert not errs, "non-zero border in: " + ", ".join(errs)
