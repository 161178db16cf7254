"""GPU: the network's results do not depend on the launch schedule, nor on the batch an instance is run in.

Every output of the inference network is reduced in an order the kernels fix: the K steps of a conv1 row or a conv2 ...
conv6_1 tile, the FC6_SPLITS fc6 partials summed in order by head_kernel, one mma row per instance in fc6.  None of it
depends on how many CTAs the persistent grids have, where conv1's row runs start and end, or which images share a tile.
So an instance's forward results are bit-identical at any SM count, batch size and batch composition.  This file holds
the library to that:

* dim_debug_set_option("sms", n) makes every launch decision use n SMs (the device is not touched).  The sweep SMS runs
  1 and 2 (fewer CTAs than conv1's column tiles: every persistent CTA walks every tile), small odd counts, 64, 114
  (H100 PCIe), 131 and the device's count.  Between them conv1's row runs are odd and even in length and the last run
  ends short (at 132 SMs, B = 16: 59 rows per run, the last 53; at 114: 69 and 24; at 13, B = 1: 41 and 38).
* net_forward of the mask and the RGB-D network in fp16, bf16 and bf16x3 at B = 1, 3, 16 on a max_batch = 16 context:
  act[1..10] (hi, and lo in bf16x3: the whole buffers, borders, virtual rows and the images past the batch), rot and
  trans equal the device-count run bit for bit; at 1 and 7 SMs every layer and fc6 + heads is also held to float64
  (tests/kernel_ref.py bounds), so the file does not lean on a reference only another file checks.  conv1's reference
  input is the stored act[0] (the zoomed blob's 16-bit pack, written before any schedule-dependent kernel runs).
* dim_refine as a captured and replayed CUDA graph at 1, 7 and 114 SMs equals the device count's; setting the key drops
  the graph (dim_debug_graph_count), which is captured again at the new count.
* Batches above 16 (bench.py's C5 configuration batches 128): net_forward on 33 instances equals 16 + 16 + 1;
  dim_refine at B = 33 equals batches of at most 16; PoseRefiner(max_batch=40) equals PoseRefiner(max_batch=16).
* The training step at 1, 7 and 114 SMs: every output except the 12 weight gradients in kernel_ref.SM_DEPENDENT_GRADS is
  bit-identical to the device-count step (see test_train_step_at_other_sm_counts); those 12 are held to float64, each
  kappa scaled by how much longer its K slice is than at the device's count (dim_train_debug_wgrad_slices).
"""
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

import ctypes as C  # noqa: E402

import kernel_ref as R  # noqa: E402
from oracle import oracle as O  # noqa: E402
from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.refiner import PoseRefiner  # noqa: E402
from deepim_b200.trainer import Trainer, make_device_batch  # noqa: E402

DEV = torch.device("cuda", 0)
H, W = 480, 640
K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
DEVICE_SMS = torch.cuda.get_device_properties(0).multi_processor_count
SMS = [n for n in (1, 2, 3, 5, 7, 13, 64, 114, 131) if n < DEVICE_SMS]
FLOAT64_AT = {1: (1, 3), 7: (3, 16)}  # SM count -> the batch sizes whose every layer is also held to float64
MODES = {"fp16": capi.PREC_FP16, "bf16": capi.PREC_BF16, "bf16x3": capi.PREC_BF16X3}
NETS = ("mask", "rgbd")
N_ITER = 4
KAPPA_SEEN = {}  # (family, SM count) -> largest kappa an element needed (DESIGN.md section 6); printed at the end


def set_sms(ctx, n):
    capi.check(capi.lib.dim_debug_set_option(ctx._h, b"sms", n))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def raw_act(ctx, idx, lo=False):
    """the whole 16-bit buffer act[idx] (every image of max_batch, border included) as uint16 [max_batch, rows, cols, C]"""
    g = (C.c_int32 * 8)()
    capi.check(capi.lib.dim_debug_layer_geometry(ctx._h, idx, g))
    shape = (ctx.max_batch, g[0], g[1], g[2])
    buf = np.empty(shape, np.uint16)
    torch.cuda.synchronize()
    capi.check(capi.lib.dim_debug_activation(ctx._h, idx, int(lo), buf.ctypes.data, buf.nbytes))
    return buf, tuple(g)


def as_float(raw, mode):
    return raw.view(np.float16).astype(np.float32) if mode == "fp16" else (raw.astype(np.uint32) << 16).view(np.float32)


@pytest.fixture(scope="module", autouse=True)
def report():
    print("\ndevice: %s, %d SMs" % (torch.cuda.get_device_name(0), DEVICE_SMS))
    yield
    print("\nlargest kappa needed per (family, SMs): " + json.dumps({"%s@%d" % k: float("%.4g" % v) for k, v in sorted(KAPPA_SEEN.items())}))
    print("largest weight-gradient slice growth per (gradient, SMs): " +
          json.dumps({"%s@%d" % k: float("%.4g" % v) for k, v in sorted(GROWTH_SEEN.items())}))


def seen(family, sms, obs):
    KAPPA_SEEN[(family, sms)] = max(KAPPA_SEEN.get((family, sms), 0.0), obs)


GROWTH_SEEN = {}  # (weight gradient, SM count) -> largest growth of its K slice over the device count's


def slices_seen(sms, growth):
    for k, v in growth.items():
        GROWTH_SEEN[(k, sms)] = max(GROWTH_SEEN.get((k, sms), 0.0), v)


@pytest.fixture(scope="module")
def meshes():
    return [synth.make_cube(), synth.make_blob()]


@pytest.fixture(scope="module")
def weights():
    return {"mask": synth.make_weights(0), "rgbd": synth.make_weights(0, input_depth=True)}


class Nets:
    """inference contexts keyed by (network, max_batch), opened on first use"""

    def __init__(self, meshes, weights):
        self.meshes, self.weights, self.open = meshes, weights, {}

    def __call__(self, net, max_batch):
        key = (net, max_batch)
        if key not in self.open:
            c = Context(0, max_batch=max_batch, max_classes=4, max_verts=6000, max_faces=11000, input_depth=net == "rgbd")
            for i, m in enumerate(self.meshes):
                c.upload_mesh(i, m)
            c.load_weights(self.weights[net])
            self.open[key] = c
        c = self.open[key]
        set_sms(c, 0)
        return c

    def close(self):
        for c in self.open.values():
            c.close()
        self.open.clear()


@pytest.fixture(scope="module")
def nets(meshes, weights):
    n = Nets(meshes, weights)
    yield n
    n.close()


# ------------------------------------------------------------------------------------------------- the option
def test_sms_option_range():
    """0 and 1 ... the device's count are accepted; anything else is refused with the range in the message and leaves the
    count as it was: the weight-gradient slicing a step would use (built afresh after the refusal) is the one of the count
    set before it, not the device's"""
    ctx = Context(0, max_batch=2, max_classes=2, max_verts=6000, max_faces=11000)
    try:
        Trainer(ctx, synth.make_train_weights(0))
        for v in (1, DEVICE_SMS, 0):
            set_sms(ctx, v)
        device = R.wgrad_slices(ctx, 2)
        set_sms(ctx, 7)
        for v in (-1, DEVICE_SMS + 1, 1 << 20):
            assert capi.lib.dim_debug_set_option(ctx._h, b"sms", v) == 2
            msg = capi.lib.dim_last_error()
            assert b"sms" in msg and (b"[1, %d]" % DEVICE_SMS) in msg, msg
        after = R.wgrad_slices(ctx, 1)  # B = 1 has no cached launch descriptors yet: sliced for the current count
        set_sms(ctx, 7)
        assert after == R.wgrad_slices(ctx, 1)
        set_sms(ctx, 0)
        assert after != R.wgrad_slices(ctx, 1) and device == R.wgrad_slices(ctx, 2)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------- net_forward
def blobs(net, B, seed):
    g = torch.Generator().manual_seed(seed)
    zio = (torch.rand(B, 3, H, W, generator=g) - 0.5) * 255
    zir = (torch.rand(B, 3, H, W, generator=g) - 0.5) * 255
    zmo = (torch.rand(B, 1, H, W, generator=g) > 0.5).float()
    zmr = (torch.rand(B, 1, H, W, generator=g) > 0.5).float()
    out = [zio, zir, zmo, zmr]
    if net == "rgbd":
        out += [0.5 + 1.5 * torch.rand(B, 1, H, W, generator=g), 0.5 + 1.5 * torch.rand(B, 1, H, W, generator=g)]
    return out


def forward(ctx, net, mode, B, seed):
    t = [x.to(DEV) for x in blobs(net, B, seed)]
    rot, trans = ctx.net_forward(*t[:4], MODES[mode], *t[4:])
    torch.cuda.synchronize()
    return rot.cpu().numpy(), trans.cpu().numpy()


def snapshot(ctx, mode):
    """act[1..10] whole, hi (and lo in bf16x3)"""
    return {(i, lo): raw_act(ctx, i, lo)[0] for i in range(1, 11) for lo in ((False, True) if mode == "bf16x3" else (False,))}


def float64_checks(ctx, weights, net, mode, B, sms):
    """every layer from its stored input, and fc6 + heads from the stored act[10], against float64"""
    from oracle.train_oracle import ENC
    halves = (False, True) if mode == "bf16x3" else (False,)
    acts, geos = {}, {}
    for i in range(11):
        for lo in halves:
            raw, g = raw_act(ctx, i, lo)
            acts[(i, lo)] = as_float(raw, mode if not lo else "bf16")
            geos[i] = g
    sizes = [(H, W)]
    for name, s, p in ENC:
        k = weights[name + "_weight"].shape[-1]
        sizes.append(((sizes[-1][0] + 2 * p - k) // s + 1, (sizes[-1][1] + 2 * p - k) // s + 1))
    pair = lambda i: (acts[(i, False)], acts.get((i, True)))
    tag = ", %d SMs" % sms
    for layer in range(10):
        g_in, g_out = geos[layer], geos[layer + 1]
        geo_in, geo_out = (g_in[3], g_in[4]) + sizes[layer], (g_out[3], g_out[4]) + sizes[layer + 1]
        if layer == 0:  # the decoded space-to-depth input, the weight's input channels (8, or 10 for RGB-D)
            cin = weights["flow_conv1_weight"].shape[1]
            py, px, h, w = geo_in
            x = tuple(None if a is None else R.gpu(R.s2d_decode(a[:B])[:, :cin, py:py + h, px:px + w]) for a in pair(0))
        else:
            x = tuple(None if a is None else R.interior(a, geo_in, B) for a in pair(layer))
        seen("conv1" if layer == 0 else "tower", sms, R.check_conv_layer(weights, mode, layer, B, x, pair(layer + 1), geo_out, tag))
    return pair(10)


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("net", NETS)
def test_forward_bit_identical_at_every_sm_count(nets, weights, net, mode):
    ctx = nets(net, 16)
    w = weights[net]
    errs = []
    for B in (1, 3, 16):
        # before every run each image of the buffers holds another batch's results (written at the device's count), so a
        # store that is missing or lands past the batch shows
        forward(ctx, net, mode, 16, 99)
        ref_rt = forward(ctx, net, mode, B, 7 + B)
        ref = snapshot(ctx, mode)
        for sms in SMS:
            forward(ctx, net, mode, 16, 99)
            set_sms(ctx, sms)
            rot, trans = forward(ctx, net, mode, B, 7 + B)
            got = snapshot(ctx, mode)
            bad = ["act[%d]%s" % (i, " lo" if lo else "") for (i, lo), a in got.items() if not np.array_equal(a, ref[(i, lo)])]
            if not np.array_equal(rot.view(np.uint32), ref_rt[0].view(np.uint32)):
                bad.append("rot")
            if not np.array_equal(trans.view(np.uint32), ref_rt[1].view(np.uint32)):
                bad.append("trans")
            if bad:
                errs.append("%s %s B=%d at %d SMs: %s differ from the %d-SM run" % (net, mode, B, sms, ", ".join(bad), DEVICE_SMS))
            if B in FLOAT64_AT.get(sms, ()):
                a10 = float64_checks(ctx, w, net, mode, B, sms)
                R.check_fc6_heads(w, mode, B, a10, rot, trans, ", %d SMs" % sms)
            set_sms(ctx, 0)
    assert not errs, "\n".join(errs)


# ------------------------------------------------------------------------------------------------- dim_refine
def scene(meshes, B, seed, depth=False, n_frames=None):
    """B observed images (the render at the observed pose composited over noise; RGB-D: a sensor-like depth) and the
    initial poses.  n_frames < B renders that many observed poses and gives the instances past them the same frames with
    their own initial poses."""
    nf = B if n_frames is None else n_frames
    obs, ini = synth.sample_pose_pairs(nf, seed)
    cls = (np.arange(B) % nf % 2).astype(np.int32)  # the class of the instance's frame
    rng = np.random.default_rng(seed)
    u8, dep = [], []
    for f in range(nf):
        r = O.render(meshes[f % 2], obs[f], K, means_rgb=MEANS)
        u8.append(synth.composite_observed(r["bgr"], r["mask"], f))
        if depth:
            d = np.where(r["depth"] > 0, r["depth"], rng.uniform(1.0, 2.0, r["depth"].shape))
            dep.append(np.clip(np.rint(d * 1000.0), 0, 65535).astype(np.uint16))
    idx = np.arange(B) % nf
    ini_all = ini[idx].copy()
    ini_all[:, 2, 3] += 0.004 * (np.arange(B) // nf)  # repeated frames: other initial depths
    u8 = np.stack(u8)[idx]
    out = dict(B=B, cls=cls, ini=ini_all, u8=u8, img=np.stack([synth.transform_image(f) for f in u8]))
    if depth:
        out["u16"] = np.stack(dep)[idx]
        out["depth"] = O.depth_from_u16(out["u16"], 1000.0)[:, None]
    return out


def inputs(sc, lo=0, hi=None):
    """the device tensors of instances lo ... hi - 1.  A graph's key holds the depth buffer's address: a chain replays only
    when called again with the same tensors."""
    hi = sc["B"] if hi is None else hi
    return (dev(sc["img"][lo:hi]), dev(sc["cls"][lo:hi]), dev(sc["ini"][lo:hi]),
            None if "depth" not in sc else dev(sc["depth"][lo:hi]))


def refine(ctx, sc, prec, lo=0, hi=None, out=None, inp=None):
    img, cls, ini, d = inputs(sc, lo, hi) if inp is None else inp
    return ctx.refine(img, cls, ini, K, N_ITER, pixel_means_rgb=MEANS, precision=prec, depth_observed=d, out=out)


def results(ctx, res, B):
    torch.cuda.synchronize()
    r = {k: v.cpu().numpy().copy() for k, v in res.items()}
    r["status"] = ctx.refine_status(B, N_ITER).numpy().copy()
    return r


def same_bits(a, b):
    """names of the results that differ bit for bit (float arrays compared as integers)"""
    return [k for k in a if not np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8))]


REFINE_CASES = [("mask", "fp16"), ("mask", "bf16x3"), ("rgbd", "fp16")]


@pytest.mark.parametrize("net,mode", REFINE_CASES, ids=["%s-%s" % c for c in REFINE_CASES])
def test_refine_graph_at_other_sm_counts(nets, meshes, net, mode):
    """dim_refine with graphs on (a side stream and out=: warm-up, capture, replay) at 1, 7 and 114 SMs equals the
    device count's, poses, se3, bbox, zoom factors and status bit for bit.  Setting the count drops the captured graph
    (dim_debug_graph_count) and the chain is captured again at the new count."""
    ctx = nets(net, 16)
    sc = scene(meshes, 5, 31, depth=net == "rgbd")
    inp = inputs(sc)
    side = torch.cuda.Stream(device=DEV)
    errs = []
    want = None
    for sms in [0] + [n for n in (1, 7, 114) if n < DEVICE_SMS]:
        torch.cuda.synchronize()
        set_sms(ctx, sms)
        assert capi.lib.dim_debug_graph_count(ctx._h) == 0, "setting the SM count keeps a graph of the old schedule"
        out = None
        for rep in range(3):
            with torch.cuda.stream(side):
                out = refine(ctx, sc, MODES[mode], out=out, inp=inp)
            side.synchronize()
            # eager warm-up, then the chain captured at this count and replayed
            assert capi.lib.dim_debug_graph_count(ctx._h) == (0 if rep == 0 else 1), (sms, rep)
            got = results(ctx, out, 5)
            if want is None:
                want = got
            diff = same_bits(got, want)
            if diff:
                errs.append("%d SMs, call %d: %s differ" % (sms or DEVICE_SMS, rep, diff))
    set_sms(ctx, 0)
    assert not want["status"].any()
    assert not errs, "\n".join(errs)


# ------------------------------------------------------------------------------------------------- above 16 instances
@pytest.mark.parametrize("mode", ["fp16", "bf16x3"])
def test_forward_of_33_equals_16_16_1(nets, mode):
    """net_forward on 33 instances (max_batch = 33: three fc6 M chunks) equals the same instances run as 16 + 16 + 1 on a
    max_batch = 16 context: rot, trans and act[10] (hi, and lo in bf16x3) per instance, bit for bit"""
    big, small = nets("mask", 33), nets("mask", 16)
    t = [x.to(DEV) for x in blobs("mask", 33, 5)]
    rot, trans = big.net_forward(*t, MODES[mode])
    torch.cuda.synchronize()
    halves = (False, True) if mode == "bf16x3" else (False,)
    a_big = {lo: raw_act(big, 10, lo)[0] for lo in halves}
    errs = []
    for a, b in ((0, 16), (16, 32), (32, 33)):
        r, tr = small.net_forward(*[x[a:b] for x in t], MODES[mode])
        torch.cuda.synchronize()
        if not torch.equal(r, rot[a:b]) or not torch.equal(tr, trans[a:b]):
            errs.append("rot / trans of instances %d ... %d" % (a, b - 1))
        for lo in halves:
            if not np.array_equal(raw_act(small, 10, lo)[0][:b - a], a_big[lo][a:b]):
                errs.append("act[10]%s of instances %d ... %d" % (" lo" if lo else "", a, b - 1))
    assert not errs, errs


@pytest.mark.parametrize("net,mode", REFINE_CASES, ids=["%s-%s" % c for c in REFINE_CASES])
def test_refine_33_equals_batches_of_16(nets, meshes, net, mode):
    """dim_refine of 33 instances on a max_batch = 33 context equals the same instances in batches of 16, 16 and 1 (and,
    for the composition, 7 + 26), bit for bit in poses, se3, bbox, zoom factors and status"""
    sc = scene(meshes, 33, 41, depth=net == "rgbd", n_frames=11)
    big = nets(net, 33)
    want = results(big, refine(big, sc, MODES[mode]), 33)
    assert not want["status"].any()
    errs = []
    small = nets(net, 16)
    for a, b in ((0, 16), (16, 32), (32, 33)):
        got = results(small, refine(small, sc, MODES[mode], a, b), b - a)
        diff = same_bits(got, {k: v[:, a:b] for k, v in want.items()})
        if diff:
            errs.append("instances %d ... %d (max_batch 16): %s differ" % (a, b - 1, diff))
    for a, b in ((0, 7), (7, 33)):
        got = results(big, refine(big, sc, MODES[mode], a, b), b - a)
        diff = same_bits(got, {k: v[:, a:b] for k, v in want.items()})
        if diff:
            errs.append("instances %d ... %d (max_batch 33): %s differ" % (a, b - 1, diff))
    assert not errs, "\n".join(errs)


def test_pose_refiner_batch_size_does_not_change_poses(meshes, weights):
    """PoseRefiner(max_batch=40, n_slots=2) over 100 instances (batches of 40, 40, 20 in flight two at a time) equals
    PoseRefiner(max_batch=16), pose for pose"""
    sc = scene(meshes, 100, 57, n_frames=20)
    got = {}
    for mb in (40, 16):
        pr = PoseRefiner(meshes, weights["mask"], max_batch=mb, n_slots=2)
        try:
            got[mb] = pr.refine(sc["u8"], sc["cls"], sc["ini"])
        finally:
            for s in pr.slots:
                s["ctx"].close()
    assert got[40].shape == (N_ITER, 100, 3, 4)
    bad = np.nonzero((got[40] != got[16]).reshape(N_ITER, 100, -1).any(axis=(0, 2)))[0]
    assert not len(bad), "instances %s differ between max_batch 40 and 16" % bad.tolist()


# ------------------------------------------------------------------------------------------------- training step
TRAIN_CASES = [("mask", "bf16", 4), ("mask", "bf16", 1), ("mask", "bf16x3", 4), ("mask", "bf16x3", 1), ("rgbd", "bf16", 3)]


def train_state(ctx, tr, out, s3):
    """every output of a step but the SM-dependent weight gradients, as raw bytes keyed by name"""
    st = {"losses": out["losses"], "rot_est_norm": out["rot_est_norm"], "trans_est": out["trans_est"],
          "flow_est": out["flow_est"], "mask_prob": out["mask_prob"]}
    st = {k: v.cpu().numpy().copy() for k, v in st.items()}
    for i in range(11):
        for lo in ((False, True) if s3 else (False,)):
            st["act[%d]%s" % (i, " lo" if lo else "")] = raw_act(ctx, i, lo)[0]
    tids = list(range(10)) + [10, 11, 12, 13, 14, 15] + [20 + i for i in range(10)]
    for tid in tids:
        st["train tensor %d" % tid] = tr.debug_tensor(tid)[0] if tid >= 10 else tr.debug_tensor(tid)
        if s3 and tid >= 10:
            st["train tensor %d lo" % tid] = tr.debug_tensor(tid + 100)[0]
    for k, v in tr.grads_dict().items():
        if k not in R.SM_DEPENDENT_GRADS:
            st["grad " + k] = v
    return st


@pytest.mark.parametrize("net,prec,B", TRAIN_CASES, ids=["%s-%s-B%d" % c for c in TRAIN_CASES])
def test_train_step_at_other_sm_counts(meshes, net, prec, B):
    """One forward_backward at 1, 7 and 114 SMs against the device count's, on the same zoomed batch.

    Bit-identical: the losses, rot / trans / flow / mask outputs, every act (hi and lo), every pre-activation gradient
    gz[0..9], the decoder buffers (cat2, cat3, dcat2, dcat3, dA10p, act10b), the fp32 decoder maps, h6 / dh6, and every
    gradient except the 12 below.  From the code: the forward pass and the data-gradient parity classes run
    conv_igemm_persistent_kernel / conv1_kernel (fixed K order per tile, whatever the grid; run_classes' streams only move
    disjoint classes), bias_partial / thin_conv_wgrad chunk by pixel count, fc6_wgrad_kernel and the thin decoder kernels
    have fixed grids.
    Not bit-identical, held to float64 instead: the weight gradients of flow_conv1, conv2 ... conv6_1, deconv5 and deconv4,
    whose K-slice count make_wgrad / run_wgrad_conv1 derive from the SM count.  Fewer slices mean longer fp32 accumulations,
    so each one's kappa is the calibrated one times kernel_ref.wgrad_slice_growth: its pixel blocks per slice at this
    count over those at the device's count, from the slicing the library reports (dim_train_debug_wgrad_slices).  On a
    132-SM part that is about 66 for conv1 at 1 SM, and 1 for the gradients make_wgrad already gives one slice there (conv6,
    conv6_1, deconv5, deconv4)."""
    ctx = Context(0, max_batch=4 if net == "mask" else 3, max_classes=2, max_verts=6000, max_faces=11000,
                  input_depth=net == "rgbd")
    try:
        for i, m in enumerate(meshes):
            ctx.upload_mesh(i, m)
        tr = Trainer(ctx, synth.make_train_weights(0, input_depth=net == "rgbd"))
        tr.set_precision(prec)
        batch = make_device_batch(ctx, meshes, B, 11 + B, K, MEANS, input_depth=net == "rgbd")[0]
        z = tr.zoom_front(batch, K)
        other = tr.zoom_front(make_device_batch(ctx, meshes, B, 5 + B, K, MEANS, input_depth=net == "rgbd")[0], K)
        errs = []
        want = None
        calibrated = R.wgrad_slices(ctx, B)  # the device count's slicing, which KAPPA_WGRAD was calibrated at
        for sms in [0] + [n for n in (1, 7, 114) if n < DEVICE_SMS]:
            set_sms(ctx, 0)
            tr.forward_backward(other)  # every buffer first holds another batch's step, so a missing store shows
            set_sms(ctx, sms)
            out = tr.forward_backward(z)
            torch.cuda.synchronize()
            got = train_state(ctx, tr, out, prec == "bf16x3")
            if want is None:
                want = got
            else:
                diff = same_bits(got, want)
                if diff:
                    errs.append("%d SMs: %s differ from the %d-SM step" % (sms, ", ".join(diff), DEVICE_SMS))
            run = R.Run(net, prec, B, ctx, tr)
            n = sms or DEVICE_SMS
            g = R.wgrad_slice_growth(R.wgrad_slices(ctx, B), calibrated)
            slices_seen(n, g)
            tag = ", %d SMs" % n
            checks = [("conv1_wgrad", "flow_conv1_weight", lambda: R.check_conv1_wgrad(run, tag, g["flow_conv1_weight"]))]
            checks += [("wgrad", R.SM_DEPENDENT_GRADS[i], lambda i=i: R.check_conv_wgrad(run, i, tag, g[R.SM_DEPENDENT_GRADS[i]]))
                       for i in range(1, 10)]
            checks += [("wgrad", m, lambda m=m: R.check_deconv_wgrad(run, m, tag, g[m])) for m in ("deconv5_weight", "deconv4_weight")]
            for fam, name, f in checks:
                before = R.OBSERVED.get(fam, 0.0)
                R.OBSERVED[fam] = 0.0
                try:
                    f()
                except AssertionError as e:
                    errs.append(str(e))
                # recorded whether or not the check passed: the kappa needed, and that kappa over the slice growth
                seen(fam, n, R.OBSERVED[fam])
                seen(fam + " / growth", n, R.OBSERVED[fam] / g[name])
                R.OBSERVED[fam] = max(before, R.OBSERVED[fam])
        assert not errs, "\n".join(errs)
    finally:
        set_sms(ctx, 0)
        ctx.close()
