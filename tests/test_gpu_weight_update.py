"""GPU: what happens to the weights between two training steps.

dim_train_sgd_update runs sgd_kernel over the flat fp32 master (its weight-decay segments come from a 44-entry end table that
a binary search walks), then repacks every operand pack the forward pass, the backward pass and the inference modes read:
forward hi / lo, dgrad per parity class, deconvolution forward and dgrad, the thin convs, fc6 and fc7^T.  Biases and the
pose heads alias the master.  Packs that only some readers need are refreshed lazily: the bf16x3 'lo' halves and the fp16
packs, the next time net_forward runs in that precision.

(a) The update against float64, element by element, for the mask, image-only and RGB-D parameter tables.
(b) A trained context equals a fresh context loaded with its weights, bit for bit: net_forward in bf16, bf16x3 and fp16,
    refine() at its default fp16, and the training step (losses, outputs, maps and the whole gradient vector, which reads
    the dgrad, deconvolution and thin packs).  The stages vary which reader comes first after an update, so that every
    lazy refresh is the first reader at least once.
(c) Updates and inference on two streams with no host synchronisation in between.
(d) The gradient-bucket readiness events of the overlapped all-reduce."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.trainer import Trainer, make_device_batch, param_table  # noqa: E402

K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
B, SEED, N_ITER = 3, 13, 3
NETS = {"mask": {}, "nomask": {"input_mask": False}, "rgbd": {"input_depth": True}}
PRECS = {"bf16": capi.PREC_BF16, "bf16x3": capi.PREC_BF16X3, "fp16": capi.PREC_FP16}
STEP_OUT = ("losses", "rot_est_norm", "trans_est", "flow_est", "mask_prob")
EPS32 = 2.0 ** -24  # unit roundoff of fp32
_MESHES = []


def meshes():
    if not _MESHES:
        _MESHES.extend([synth.make_cube(), synth.make_blob()])
    return _MESHES


def make_ctx(net):
    c = Context(0, max_batch=B, max_classes=2, max_verts=6000, max_faces=11000, **NETS[net])
    for i, m in enumerate(meshes()):
        c.upload_mesh(i, m)
    return c


def flat(tr, momentum=False):
    """the flat master (or momentum) vector as a device float32 tensor"""
    a = np.empty(tr.n, np.float32)
    capi.check(capi.lib.dim_train_get_params(tr.ctx._h, a.ctypes.data_as(C.c_void_p), tr.n, int(momentum), tr._stream()))
    return torch.from_numpy(a).cuda()


def sgd(tr, lr, momentum, wd, rescale):
    capi.check(capi.lib.dim_train_sgd_update(tr.ctx._h, C.c_void_p(tr.grads.data_ptr()), lr, momentum, wd, rescale, tr._stream()))


# ------------------------------------------------------------------------------------------------- (a) the update itself
def segments(net):
    """[(name, lo, hi)] of the flat vector, and the end of the trainable part (the frozen bilinear kernels follow it)"""
    out, off = [], 0
    for name, n in param_table(**NETS[net]):
        out.append((name, off, off + n))
        off += n
    trainable = [s for s in out if s[0] not in ("upsampling_weight", "mask_upsampling_weight")]
    assert len(trainable) == 44 and trainable[-1][2] == out[-2][1]
    return trainable, trainable[-1][2]


@pytest.mark.parametrize("net", sorted(NETS))
def test_sgd_update_against_float64(net):
    """mom1 = momentum*mom0 - lr*(rescale*g + wd_seg*w0), w1 = w0 + mom1, where wd_seg is wd on every _weight segment and
    0 on every _bias segment.  mom1 within a few fp32 roundings of its terms (six roundings in the kernel's fp32 evaluation,
    each at most EPS32 of the term it rounds); w1 exactly fp32(w0 + mom1) (one add, nothing to contract); the frozen
    bilinear tail untouched in both vectors.  Three updates in a row, so the momentum carries over, with rescale 1 and 1/3.
    First an all-zero gradient on the freshly loaded (zero) momentum: then mom1 is exactly -(lr*(wd*w)) on weights and 0 on
    biases, which pins every segment boundary of the binary search."""
    segs, n_train = segments(net)
    w = synth.make_train_weights(3, **NETS[net])
    rng = np.random.default_rng(4)
    for k in w:  # nonzero biases, so that a bias element decayed like a weight shows
        if k.endswith("_bias"):
            w[k] = (rng.uniform(0.5, 1.5, w[k].shape) * rng.choice([-1.0, 1.0], w[k].shape)).astype(np.float32)
    ctx = make_ctx(net)
    try:
        tr = Trainer(ctx, w)
        wd_seg = torch.zeros(tr.n, dtype=torch.float64, device="cuda")
        is_w = torch.zeros(tr.n, dtype=torch.bool, device="cuda")
        for name, lo, hi in segs:
            if name.endswith("_weight"):
                is_w[lo:hi] = True
        lr, mu, wd = 3e-3, 0.9, 7e-4
        f32 = lambda x: float(np.float32(x))

        # zero gradient on zero momentum
        w0, m0 = flat(tr), flat(tr, True)
        assert not m0.any()
        tr.grads.zero_()
        sgd(tr, lr, mu, wd, 1.0)
        w1, m1 = flat(tr), flat(tr, True)
        want = torch.where(is_w, -((w0 * f32(wd)) * f32(lr)), torch.zeros_like(w0))  # fp32 products, as the kernel rounds them
        want[n_train:] = 0
        for name, lo, hi in segs:  # first and last element of every segment: an off-by-one in the search shows here
            for i in (lo, hi - 1):
                assert m1[i].item() == want[i].item(), (net, name, i, m1[i].item(), want[i].item())
        bad = (m1 != want).nonzero()
        assert bad.numel() == 0, (net, "momentum differs from -(lr*(wd*w)) / 0 at", bad[:8].flatten().tolist())
        assert torch.equal(w1[:n_train], w0[:n_train] + m1[:n_train])
        assert torch.equal(w1[n_train:], w0[n_train:])

        wd_seg[is_w] = f32(wd)
        g = torch.Generator(device="cuda").manual_seed(9)
        for step, rescale in enumerate((1.0, 1.0 / 3.0, 1.0)):
            w0, m0 = w1, m1
            tr.grads.copy_(torch.randn(tr.n, generator=g, device="cuda") * (10.0 ** (step - 1)))
            sgd(tr, lr, mu, wd, rescale)
            w1, m1 = flat(tr), flat(tr, True)
            g64, w64, m64 = tr.grads.double(), w0.double(), m0.double()
            ref = f32(mu) * m64 - f32(lr) * (f32(rescale) * g64 + wd_seg * w64)
            scale = f32(mu) * m64.abs() + f32(lr) * (f32(rescale) * g64.abs() + wd_seg * w64.abs())
            err = (m1.double() - ref).abs()[:n_train]
            bound = (8 * EPS32 * scale + 2.0 ** -126)[:n_train]
            worst = int(torch.argmax(err / bound))
            assert bool((err <= bound).all()), (net, step, worst, err[worst].item(), bound[worst].item())
            assert torch.equal(w1[:n_train], w0[:n_train] + m1[:n_train]), (net, step)
            assert torch.equal(w1[n_train:], w0[n_train:]) and torch.equal(m1[n_train:], m0[n_train:]), (net, step)
            assert (m1[:n_train] != m0[:n_train]).float().mean().item() > 0.99
    finally:
        ctx.close()


# --------------------------------------------------------------------- (b) a trained context equals a freshly loaded one
class World:
    """one network's training context, its Trainer, a fixed training batch (zoom_front output) and a fixed refinement scene"""

    def __init__(self, net, precision="bf16", bucket_mb=32.0):
        self.net = net
        self.ctx = make_ctx(net)
        self.tr = Trainer(self.ctx, synth.make_train_weights(5, **NETS[net]), precision=precision, bucket_mb=bucket_mb)
        batch, cls, _, _ = make_device_batch(self.ctx, meshes(), B, SEED, K, MEANS, input_depth=net == "rgbd")
        self.z = self.tr.zoom_front(batch, K)
        _, ini = synth.sample_pose_pairs(B, SEED)
        self.scene = (batch["image_observed"], cls, torch.from_numpy(np.ascontiguousarray(ini, np.float64)).cuda())
        self.depth_obs = batch.get("depth_observed")
        torch.cuda.synchronize()

    def fwd_args(self):
        z = self.z
        masks = (None, None) if self.net == "nomask" else (z["zoom_mask_observed"], z["zoom_mask_rendered"])
        depths = ({"zoom_depth_observed": z["zoom_depth_observed"], "zoom_depth_rendered": z["zoom_depth_rendered"]}
                  if self.net == "rgbd" else {})
        return (z["zoom_image_observed"], z["zoom_image_rendered"]) + masks, depths

    def update(self, lr=1e-3):
        """one training step and its update on the current stream"""
        self.tr.forward_backward(self.z, want_maps=False)
        self.tr.update(lr=lr)

    def close(self):
        self.ctx.close()


def check_equal_to_fresh(world, order, what=""):
    """E(ctx): the readers in `order` ('bf16', 'bf16x3', 'fp16': net_forward; 'refine': refine() at its default precision;
    'step': forward_backward in the step's current precision) on the trained context give bit for bit what a fresh context
    loaded with its current weights gives.  The trained context runs them in `order`, so the first one is the first reader
    of whatever the last update left stale."""
    tr, net = world.tr, world.net
    p = tr.get_params()
    args, depths = world.fwd_args()
    got = {}
    for r in order:  # the trained context first, in the given order
        if r in PRECS:
            got[r] = world.ctx.net_forward(*args, precision=PRECS[r], **depths)
        elif r == "refine":
            got[r] = world.ctx.refine(*world.scene, K, N_ITER, pixel_means_rgb=MEANS, depth_observed=world.depth_obs)
        else:
            out = tr.forward_backward(world.z)
            got[r] = (out, tr.grads.clone())
    torch.cuda.synchronize()
    fresh = make_ctx(net)
    try:
        fresh.load_weights(p)
        for r in order:
            if r in PRECS:
                rot, trans = fresh.net_forward(*args, precision=PRECS[r], **depths)
                torch.cuda.synchronize()
                assert torch.isfinite(rot).all() and rot.abs().max().item() > 0
                assert torch.equal(got[r][0], rot), (what, net, r, "rot", (got[r][0] - rot).abs().max().item())
                assert torch.equal(got[r][1], trans), (what, net, r, "trans", (got[r][1] - trans).abs().max().item())
            elif r == "refine":
                res = fresh.refine(*world.scene, K, N_ITER, pixel_means_rgb=MEANS, depth_observed=world.depth_obs)
                torch.cuda.synchronize()
                for k in ("poses", "se3"):
                    a, b = got[r][k].cpu().numpy(), res[k].cpu().numpy()
                    assert np.array_equal(a, b), (what, net, "refine", k, np.abs(a - b).max(axis=tuple(range(1, a.ndim))))
    finally:
        fresh.close()
    if "step" not in order:
        return
    fresh = make_ctx(net)
    try:
        tr2 = Trainer(fresh, p, precision=tr.precision)
        out2 = tr2.forward_backward(world.z)
        torch.cuda.synchronize()
        out, grads = got["step"]
        for k in STEP_OUT:
            assert torch.equal(out[k], out2[k]), (what, net, "step", tr.precision, k)
        if not torch.equal(grads, tr2.grads):
            names = [nm for nm, (lo, n) in tr.offsets().items() if not torch.equal(grads[lo:lo + n], tr2.grads[lo:lo + n])]
            raise AssertionError("%s %s step (%s): gradients differ in %s" % (what, net, tr.precision, names))
    finally:
        fresh.close()


def assert_changed(world, before):
    after = world.tr.get_params()
    assert not np.array_equal(after["conv2_weight"], before["conv2_weight"])
    assert not np.array_equal(after["deconv4_weight"], before["deconv4_weight"])
    return after


def test_trained_mask_context_equals_a_freshly_loaded_one():
    w = World("mask")
    try:
        check_equal_to_fresh(w, ["fp16", "bf16", "bf16x3", "refine", "step"], "load")
        p = w.tr.get_params()
        w.update()  # an update with no inference after it: the step reads the packs first
        p = assert_changed(w, p)
        check_equal_to_fresh(w, ["step", "bf16", "refine", "fp16", "bf16x3"], "update, step first")
        w.update()  # the bf16 step left lo stale: fp16 reads first
        p = assert_changed(w, p)
        check_equal_to_fresh(w, ["fp16", "bf16x3", "bf16", "step", "refine"], "update, fp16 first")
        w.update()
        p = assert_changed(w, p)
        check_equal_to_fresh(w, ["bf16x3", "fp16", "refine", "step", "bf16"], "update, bf16x3 first")
        w.tr.set_precision("bf16x3")
        w.update()  # the bf16x3 update refreshes the lo halves itself
        p = assert_changed(w, p)
        check_equal_to_fresh(w, ["refine", "step", "bf16x3", "bf16", "fp16"], "bf16x3 update, refine first")
        w.tr.set_precision("bf16")
        w.update()
        assert_changed(w, p)
        check_equal_to_fresh(w, ["bf16", "step", "fp16", "bf16x3", "refine"], "back to bf16, update")
    finally:
        w.close()


@pytest.mark.parametrize("net", ["nomask", "rgbd"])
def test_trained_context_equals_a_freshly_loaded_one(net):
    w = World(net)
    try:
        check_equal_to_fresh(w, ["fp16", "bf16", "bf16x3", "step"], "load")
        p = w.tr.get_params()
        w.update()
        p = assert_changed(w, p)
        check_equal_to_fresh(w, ["step", "fp16", "bf16x3", "bf16"], "bf16 update")
        w.tr.set_precision("bf16x3")
        w.update()
        assert_changed(w, p)
        check_equal_to_fresh(w, ["bf16x3", "step", "fp16", "bf16"], "bf16x3 update")
    finally:
        w.close()


# --------------------------------------------------------------------------------------------------- (c) two streams
def test_updates_and_inference_on_two_streams():
    """An update on stream A, an fp16 and a bf16x3 forward on stream B (each refreshes packs from the master: fp16 and lo),
    another update on A, a bf16 forward on B, with no host synchronisation until the end; then E with the step and bf16
    first, the readers that refresh nothing.  The second update must wait for B's refreshes to finish reading the master,
    or they write packs from a half-updated master that nothing refreshes again.  Without that ordering this test can still
    pass: it fails only when the streams' timing lets the update overtake a refresh."""
    w = World("mask")
    try:
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        args, _ = w.fwd_args()
        p = w.tr.get_params()
        torch.cuda.synchronize()
        with torch.cuda.stream(a):
            w.update()
        with torch.cuda.stream(b):
            w.ctx.net_forward(*args, precision=capi.PREC_FP16)
            w.ctx.net_forward(*args, precision=capi.PREC_BF16X3)
        with torch.cuda.stream(a):
            w.tr.update(lr=1e-3)
        with torch.cuda.stream(b):
            w.ctx.net_forward(*args, precision=capi.PREC_BF16)
        torch.cuda.synchronize()
        assert_changed(w, p)
        check_equal_to_fresh(w, ["step", "bf16", "fp16", "bf16x3", "refine"], "two streams")
    finally:
        w.close()


# ------------------------------------------------------------------------------------ (d) bucket readiness events
class _Work:
    def wait(self):
        pass


class _Dist:
    """stands in for torch.distributed in Trainer.allreduce_overlapped: snapshots every bucket on the stream it is called on
    (the comm stream, after the bucket's readiness event)"""

    class ReduceOp:
        SUM = "sum"

    def __init__(self):
        self.snaps = []

    def all_reduce(self, t, op=None, async_op=False):
        assert op == self.ReduceOp.SUM and async_op
        self.snaps.append(t.clone())
        return _Work()


def test_gradient_bucket_events_on_one_gpu():
    """forward_backward(overlap=True) records one readiness event per bucket and gives the gradients overlap=False gives;
    every bucket snapshot that allreduce_overlapped takes behind its event equals the bucket's final gradients.  The
    gradients are poisoned with NaN before the step, so a bucket read before its event fired shows, when the timing exposes
    it: an event recorded too early can still pass here."""
    w = World("mask", bucket_mb=0.5)
    try:
        tr = w.tr
        assert len(tr.buckets) >= 12
        first = sorted(tr.bucket_first)
        assert all(i in first for i in range(10)), first  # every encoder layer starts a bucket of its own
        tr.forward_backward(w.z)
        want = tr.grads.clone()
        tr.grads.fill_(float("nan"))
        tr.forward_backward(w.z, overlap=True)
        d = _Dist()
        tr.allreduce_overlapped(d)
        torch.cuda.synchronize()
        assert torch.equal(tr.grads, want)
        assert len(d.snaps) == len(tr.buckets)
        for (lo, hi), s in zip(tr.buckets, d.snaps):
            assert torch.equal(s, tr.grads[lo:hi]), (lo, hi, int(torch.isnan(s).sum()))
    finally:
        w.close()
