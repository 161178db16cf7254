"""Trainer: the device replacement of Module.forward_backward + Module.update for the refiner network
(deepim/core/module.py:1131-1137: one SGD update after each of the TRAIN_ITER_SIZE = 4 inner iterations, with
the batch re-rendered in between by batchUpdaterPyMulti -> Context.train_update).

Data parallel (SURVEY 8(e), training row): one process per GPU, every rank runs forward_backward on its slice
of the batch, the flat fp32 gradient vector is sum-all-reduced with NCCL in buckets (rescale_grad = 1.0, so a
plain sum like kvstore's), then every rank applies the identical SGD update."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _capi as capi
from . import lighting as _lighting
from ._capi import check, lib

NORMALIZE_FLOW = 20.0


def _is_rgbd(weights) -> bool:
    return np.shape(weights["flow_conv1_weight"])[1:2] == (10,)


def _is_nomask(weights) -> bool:
    return np.shape(weights["flow_conv1_weight"])[1:2] == (6,)


def param_table(input_depth=False, input_mask=True):
    """[(tensor name, numel)] in flat order, as the library reports it (dim_train_param_info; input_depth: the RGB-D
    network's table, whose flow_conv1 is (64, 10, 7, 7); input_mask=False: the image-only network's table, whose
    flow_conv1 is (64, 6, 7, 7))."""
    out = []
    for i in range(64):
        name, wn, bn = C.c_char_p(), C.c_int64(), C.c_int64()
        if lib.dim_train_param_info(int(input_depth), int(input_mask), i, C.byref(name), C.byref(wn), C.byref(bn)) != 0:
            break
        out.append((name.value.decode() + "_weight", wn.value))
        if bn.value:
            out.append((name.value.decode() + "_bias", bn.value))
    return out


def flatten_params(weights: dict) -> np.ndarray:
    """The flat vector of the table the weights belong to (RGB-D when flow_conv1_weight has 10 input channels, image-only
    when it has 6)."""
    parts = []
    for name, n in param_table(_is_rgbd(weights), not _is_nomask(weights)):
        a = np.asarray(weights[name], dtype=np.float32)
        if name == "fc6_weight":  # the flat vector keeps fc6 as (out, h*10+w, c): NHWC order of the conv6_1 activation
            a = a.reshape(256, 1024, 80).transpose(0, 2, 1)
        a = np.ascontiguousarray(a).reshape(-1)
        if a.size != n:
            raise ValueError("%s: expected %d values, got %d" % (name, n, a.size))
        parts.append(a)
    return np.concatenate(parts)


def unflatten_params(flat: np.ndarray, like: dict) -> dict:
    out, off = {}, 0
    for name, n in param_table(_is_rgbd(like), not _is_nomask(like)):
        a = np.asarray(flat[off:off + n], np.float32)
        if name == "fc6_weight":  # back to MXNet's (out, c*80 + h*10 + w) (deepIM_flownet.py:110-112)
            a = a.reshape(256, 80, 1024).transpose(0, 2, 1)
        out[name] = np.ascontiguousarray(a).reshape(like[name].shape).copy()
        off += n
    return out


def tensor_sizes(input_depth=False, input_mask=True):
    """[(table index, weight + bias numel)] of the tensors of the flat vector (dim_train_param_info order)."""
    out = []
    for i in range(64):
        nm, wn, bn = C.c_char_p(), C.c_int64(), C.c_int64()
        if lib.dim_train_param_info(int(input_depth), int(input_mask), i, C.byref(nm), C.byref(wn), C.byref(bn)) != 0:
            break
        out.append((i, wn.value + bn.value))
    return out


def make_buckets(bucket_mb=32.0, sizes=None):
    """Gradient buckets for the overlapped all-reduce: contiguous [lo, hi) slices of the flat vector cut along tensor
    boundaries, formed walking the tensors BACKWARDS (the order the backward pass completes them), each at least
    bucket_mb MB (the last one takes the remainder).  Returns (buckets, first) where first[k] = table index of the
    lowest tensor in bucket k: the library records event k once every tensor with index >= first[k] is complete."""
    sizes = tensor_sizes() if sizes is None else sizes
    n = sum(m for _, m in sizes)
    limit = int(bucket_mb * (1 << 20) / 4)
    buckets, first, hi, lo = [], [], n, n
    for idx, m in reversed(sizes):
        lo -= m
        if hi - lo >= limit:
            buckets.append((lo, hi))
            first.append(idx)
            hi = lo
    if hi > 0:
        buckets.append((0, hi))
        first.append(0)
    return buckets, first


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class Trainer:
    def __init__(self, ctx, weights: dict, max_points=3000, lr=1e-4, momentum=0.975, wd=5e-4, bucket_mb=32.0, config=None,
                 precision="bf16"):
        """config: optional dict overriding fields of dim_train_config (lw_flow, lw_mask, lw_pm, num_3d_sample,
        normalize_3d_point, normalize_flow, trans_means, trans_stds, rot_coord = 'MODEL' | 'CAMERA'): the yaml's train.LW_* /
        NUM_3D_SAMPLE / NORMALIZE_* / network.TRANS_MEANS / TRANS_STDS / ROT_COORD.  Default: the shipped LM6d values.
        precision: 'bf16' (bf16 activations and activation gradients) or 'bf16x3' (hi / lo pairs, gradients near fp32) for
        every step of this context -- forward_backward, fit_batch, test_forward_full and the updates (see set_precision)."""
        self.ctx, self.lr, self.momentum, self.wd = ctx, lr, momentum, wd
        self.input_depth = bool(getattr(ctx, "input_depth", False))  # Context(input_depth=True): the RGB-D network
        self.input_mask = bool(getattr(ctx, "input_mask", True))  # Context(input_mask=False): the image-only network
        if _is_rgbd(weights) != self.input_depth or _is_nomask(weights) == self.input_mask:
            raise ValueError("flow_conv1_weight has %d input channels; this context's network takes %d"
                             % (np.shape(weights["flow_conv1_weight"])[1],
                                10 if self.input_depth else (8 if self.input_mask else 6)))
        check(lib.dim_train_create(ctx._h, max_points))
        if config:
            ctx.set_config(**config)
        self.n = int(lib.dim_train_param_count(ctx._h))
        self.table = param_table(self.input_depth, self.input_mask)
        flat = flatten_params(weights)
        assert flat.size == self.n
        self._shapes = {k: np.asarray(v).shape for k, v in weights.items()}
        check(lib.dim_train_load_params(ctx._h, flat.ctypes.data_as(C.c_void_p), self.n, self._stream()))
        torch.cuda.current_stream(ctx.device).synchronize()
        self.set_precision(precision)
        self.grads = torch.zeros(self.n, dtype=torch.float32, device=ctx.device)
        self.buckets, self.bucket_first = make_buckets(bucket_mb, tensor_sizes(self.input_depth, self.input_mask))
        self._events = None
        self._comm_stream = None
        self._last_n = 0

    def set_precision(self, precision):
        """'bf16' | 'bf16x3' (or DIM_PREC_BF16 / DIM_PREC_BF16X3): the precision of this context's training step
        (dim_train_set_precision).  'fp16' is refused: there is no fp16 training step."""
        torch.cuda.current_stream(self.ctx.device).synchronize()  # the switch synchronises the device, not torch's stream
        check(lib.dim_train_set_precision(self.ctx._h, capi.precision_id(precision)))

    @property
    def precision(self) -> str:
        p = C.c_int32()
        check(lib.dim_train_get_precision(self.ctx._h, C.byref(p)))
        return {capi.PREC_BF16: "bf16", capi.PREC_BF16X3: "bf16x3"}[p.value]

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.ctx.device).cuda_stream)

    def offsets(self):
        out, off = {}, 0
        for name, n in self.table:
            out[name] = (off, n)
            off += n
        return out

    def _bucket_events(self):
        if self._events is None:
            self._events = [torch.cuda.Event() for _ in self.buckets]
            for e in self._events:
                e.record()  # forces creation of the underlying cudaEvent_t
            self._ev_handles = (C.c_void_p * len(self._events))(*[e.cuda_event for e in self._events])
            self._ev_first = (C.c_int32 * len(self._events))(*self.bucket_first)
            self._comm_stream = torch.cuda.Stream(device=self.ctx.device)
        return self._ev_handles, self._ev_first

    def forward_backward(self, z, want_maps=True, backward=True, overlap=False):
        """z: dict of device float32 tensors (the outputs of the zoom front of the train symbol + labels):
        zoom_image_observed/rendered (B,3,H,W), zoom_mask_observed/rendered (B,1,H,W), zoom_factor (B,4),
        zoom_flow, zoom_flow_weights (B,2,H,W), zoom_mask_gt_observed (B,1,H,W), src_pose (B,3,4),
        point_cloud_model/weights/observed (B,3,N); RGB-D network: also zoom_depth_observed / zoom_depth_rendered (B,1,H,W).
        The image-only network does not read zoom_mask_observed / zoom_mask_rendered (they may be absent); the GT mask
        label still is."""
        ctx = self.ctx
        B, N = z["zoom_image_observed"].shape[0], z["point_cloud_model"].shape[2]
        self._last_n = N  # the point count of debug_tensor's pts_est / dpts
        zmo, zmr = (z["zoom_mask_observed"], z["zoom_mask_rendered"]) if self.input_mask else (None, None)
        zdo, zdr = (z["zoom_depth_observed"], z["zoom_depth_rendered"]) if self.input_depth else (None, None)
        for k, t in z.items():
            if t.dtype != torch.float32 or not t.is_contiguous() or not t.is_cuda:
                raise TypeError("%s must be a contiguous float32 CUDA tensor" % k)
        out = {"rot_est_norm": ctx._new((B, 4)), "trans_est": ctx._new((B, 3)), "losses": ctx._new((4,)),
               "flow_est": ctx._new((B, 2, ctx.H, ctx.W)) if want_maps else None,
               "mask_prob": ctx._new((B, 1, ctx.H, ctx.W)) if want_maps else None}
        check(lib.dim_train_forward_backward(
            ctx._h, _p(z["zoom_image_observed"]), _p(z["zoom_image_rendered"]), _p(zmo), _p(zmr), _p(z["zoom_factor"]),
            _p(z["zoom_flow"]), _p(z["zoom_flow_weights"]), _p(z["zoom_mask_gt_observed"]), _p(z["src_pose"]),
            _p(z["point_cloud_model"]), _p(z["point_cloud_weights"]), _p(z["point_cloud_observed"]), B, N,
            _p(out["rot_est_norm"]), _p(out["trans_est"]), _p(out["flow_est"]), _p(out["mask_prob"]), _p(out["losses"]),
            _p(self.grads) if backward else None, None,
            *((self._bucket_events() + (len(self.buckets),)) if (backward and overlap) else (None, None, 0)),
            _p(zdo), _p(zdr), self._stream()))
        return out

    def test_forward_full(self, batch, K):
        """The non-FAST_TEST test graph (get_test_symbol_share, deepIM_flownet.py:548-735 with FAST_TEST: False):
        se3 = [rot_raw, invZoomTrans(trans)], mask_observed_pred = round(invZoomMask(sigmoid(mask logits))),
        flow_est = invZoomFlow(upsampled flow x NORMALIZE_FLOW), plus the zoomed intermediates the graph also returns.
        batch: image_observed/rendered (B,3,H,W), mask_observed/rendered (B,1,H,W), src_pose (B,3,4), pixel_means_rgb."""
        ctx = self.ctx
        if self.input_mask:
            zo, zg, zr, zf, bbox, status = ctx.zoom_mask(batch["mask_observed"], batch["mask_observed"], batch["mask_rendered"],
                                                         batch["src_pose"], K)
            zio, zir = ctx.zoom_image_with_factor(zf, batch["image_observed"], batch["image_rendered"], batch["pixel_means_rgb"])
        else:  # the image-only test graph zooms with ZoomImage and feeds no masks (deepIM_flownet.py:562-601)
            zio, zir, zf, bbox, status = ctx.zoom_image(batch["image_observed"], batch["image_rendered"], batch["src_pose"], K,
                                                        batch["pixel_means_rgb"])
            zo = zr = None
        B = zio.shape[0]
        rot, trans = ctx._new((B, 4)), ctx._new((B, 3))
        zflow, zprob = ctx._new((B, 2, ctx.H, ctx.W)), ctx._new((B, 1, ctx.H, ctx.W))
        check(lib.dim_train_forward_backward(ctx._h, _p(zio), _p(zir), _p(zo), _p(zr), _p(zf), None, None, None, None, None, None,
                                             None, B, 0, None, _p(trans), _p(zflow), _p(zprob), None, None, _p(rot), None, None, 0,
                                             None, None, self._stream()))
        mask_pred = torch.round(ctx.zoom_mask_with_factor(zf, zprob, True))
        flow_est, _ = ctx.zoom_flow(zf, zflow, None, True)
        return {"se3": torch.cat([rot, trans], dim=1), "zoom_factor": zf, "mask_observed_pred": mask_pred, "flow_est": flow_est,
                "zoom_mask_observed_pred": zprob, "zoom_flow_est": zflow, "zoom_mask_observed": zo, "zoom_image_observed": zio,
                "zoom_image_rendered": zir, "bbox": bbox}

    def allreduce(self, dist):
        if dist is not None and dist.is_initialized() and dist.get_world_size() > 1:
            for lo, hi in self.buckets:
                dist.all_reduce(self.grads[lo:hi], op=dist.ReduceOp.SUM)

    def update(self, lr=None):
        check(lib.dim_train_sgd_update(self.ctx._h, _p(self.grads), self.lr if lr is None else lr, self.momentum, self.wd,
                                       1.0, self._stream()))

    def allreduce_overlapped(self, dist):
        """Bucket k is all-reduced as soon as its readiness event (recorded inside dim_train_forward_backward) fires,
        i.e. while the backward pass of the lower layers is still running; the update waits for all of them."""
        cur = torch.cuda.current_stream(self.ctx.device)
        works = []
        with torch.cuda.stream(self._comm_stream):
            for k, (lo, hi) in enumerate(self.buckets):
                self._comm_stream.wait_event(self._events[k])
                works.append(dist.all_reduce(self.grads[lo:hi], op=dist.ReduceOp.SUM, async_op=True))
            for w in works:
                w.wait()
        cur.wait_stream(self._comm_stream)

    def step(self, z, dist=None, want_maps=False, overlap=True):
        multi = dist is not None and dist.is_initialized() and dist.get_world_size() > 1
        out = self.forward_backward(z, want_maps=want_maps, overlap=multi and overlap)
        if multi and overlap:
            self.allreduce_overlapped(dist)
        else:
            self.allreduce(dist)
        self.update()
        return out

    def zoom_front(self, batch, K):
        """ZoomMask / ZoomImageWithFactor / ZoomFlow of get_train_symbol (deepIM_flownet.py:391-489) on device tensors."""
        ctx = self.ctx
        zo, zg, zr, zf, _, _ = ctx.zoom_mask(batch["mask_observed"], batch["mask_gt_observed"], batch["mask_rendered"],
                                          batch["src_pose"], K)
        zio, zir = ctx.zoom_image_with_factor(zf, batch["image_observed"], batch["image_rendered"], batch["pixel_means_rgb"])
        zfl, zfw = ctx.zoom_flow(zf, batch["flow"], batch["flow_weights"], False)
        zd = {}
        if self.input_depth:  # ZoomDepth with the pair's zoom factor (deepIM_flownet.py:461-475)
            zdo, zdr = ctx.zoom_depth(zf, batch["depth_observed"], batch["depth_rendered"])
            zd = {"zoom_depth_observed": zdo, "zoom_depth_rendered": zdr}
        return {**zd, "zoom_image_observed": zio, "zoom_image_rendered": zir, "zoom_mask_observed": zo, "zoom_mask_rendered": zr,
                "zoom_factor": zf, "zoom_flow": zfl, "zoom_flow_weights": zfw, "zoom_mask_gt_observed": zg,
                "src_pose": batch["src_pose"], "point_cloud_model": batch["point_cloud_model"],
                "point_cloud_weights": batch["point_cloud_weights"], "point_cloud_observed": batch["point_cloud_observed"]}

    def get_params(self, momentum=False) -> dict:
        flat = np.empty(self.n, np.float32)
        check(lib.dim_train_get_params(self.ctx._h, flat.ctypes.data_as(C.c_void_p), self.n, 1 if momentum else 0, self._stream()))
        return unflatten_params(flat, {k: np.empty(s, np.float32) for k, s in self._shapes.items()})

    def grads_dict(self) -> dict:
        flat = self.grads.cpu().numpy()
        return unflatten_params(flat, {k: np.empty(s, np.float32) for k, s in self._shapes.items()})

    def debug_tensor(self, tid):
        """fp32 maps (id < 8) as [B,h,w,c], h6 / dh6 (8 / 9) as [B,256]; bf16 buffers (10 ... 29) as float32 [B,Hp,Wp,C]
        incl. border; the pose heads (30 ... 40) as [B,256] (h7, dh7), [B,4] / [B,3] (rot_raw, ztrans, rot_n, trans_est,
        drot_n, dtrans, drot) and [B,3,N] (pts_est, dpts, N of the last forward_backward); 41 dfull as [B,3,H,W].
        B is the context's max_batch: images past the last step's batch hold whatever an earlier step left."""
        ctx = self.ctx
        B = ctx.max_batch
        if tid < 10 or 30 <= tid < 42:
            hw = {0: (8, 10, 2), 1: (15, 20, 2), 2: (30, 40, 2), 3: (30, 40, 1), 4: (30, 40, 2), 5: (30, 40, 1), 6: (15, 20, 2),
                  7: (8, 10, 2), 8: (256,), 9: (256,), 30: (256,), 31: (4,), 32: (3,), 33: (4,), 34: (3,), 35: (3, self._last_n),
                  36: (3, self._last_n), 37: (4,), 38: (3,), 39: (4,), 40: (256,), 41: (3, ctx.H, ctx.W)}[tid]
            a = np.empty((B,) + hw, np.float32)
            check(lib.dim_train_debug_tensor(ctx._h, tid, a.ctypes.data_as(C.c_void_p), a.nbytes))
            return a
        geo = (C.c_int32 * 7)()
        check(lib.dim_train_debug_geometry(ctx._h, tid, geo))
        Hp, Wp, py, px, Cc, H, W = list(geo)
        raw = np.empty((B, Hp, Wp, Cc), np.uint16)
        check(lib.dim_train_debug_tensor(ctx._h, tid, raw.ctypes.data_as(C.c_void_p), raw.nbytes))
        return (raw.astype(np.uint32) << 16).view(np.float32), (py, px, H, W)


def make_device_batch(ctx, meshes, B, seed, K, pixel_means_rgb, num_points=3000, init_mask="box_gt", poses=None,
                      image_observed=None, cls_np=None, lighting=None, input_depth=False, background=None, mask_dilate=None):
    """Synthetic training batch built with the device kernels only (config C4: rendered pairs, labels from
    dim_train_update, INIT_MASK box_gt without dilation, 3000 sampled model points as get_point_cloud_model,
    lib/utils/image.py:452-478).  init_mask = "box_gt" (the reference's training config: mask_observed = box of the GT mask)
    or "box_rendered" (the TEST-time convention, yaml:118: box of the rendered mask -- train / test inputs then match).
    poses = (pose_observed, pose_init) [B,3,4] instead of sampling them from `seed`; image_observed = the observed blob to
    train on (float32 [B,3,H,W] RGB - mean, e.g. a render composited over a background) instead of the clean render.
    lighting = None (LINEMOD) or the ModelNet branch's light ({"seed", "offset", "brightness_ratio"} or a
    lighting.LightSource; the meshes' normals must be uploaded to ctx): the observed and the rendered images are lit renders,
    each with a fresh intensity draw.
    input_depth = True adds the RGB-D network's blobs: depth_observed = the observed render's depth, depth_rendered = the
    update's render depth (refined_depth_array, batch_updater_py_multi.py:269).
    background = (augment.BackgroundBank, draws): the observed images are synthetic (data_syn), so each gets the background
    photo the draws name (int32 [B] bank indices, -1 = keep; an int instead of an array seeds
    augment.background_draws(B, RandomState(seed), len(bank))), composited under the GT mask (image.py:96-157).
    mask_dilate = a np.random.RandomState or an int seed: mask_observed is dilated after the box is formed with
    augment.mask_dilate_draws (TRAIN.MASK_DILATE, image.py:289-290).  Both stay fixed across fit_batch's inner iterations.
    Returns (batch dict of CUDA tensors, cls int32[B], tgt_pose f32[B,3,4], depth_gt)."""
    from . import augment, synth
    if background is not None and image_observed is not None:
        raise ValueError("make_device_batch: background replaces the rendered observed image; image_observed would ignore it")
    obs, ini = synth.sample_pose_pairs(B, seed) if poses is None else poses
    dev = ctx.device
    cls_np = (np.arange(B) % len(meshes)).astype(np.int32) if cls_np is None else np.asarray(cls_np, np.int32)
    cls = torch.from_numpy(cls_np).to(dev)
    tgt = torch.from_numpy(obs.astype(np.float32)).to(dev)
    src = torch.from_numpy(ini.astype(np.float32)).to(dev)
    light = _lighting.LightSource.of(lighting)
    want = ("image", "depth", "mask") + (("bgr",) if background is not None else ())
    if light is None:
        r = ctx.render(cls, tgt, K, pixel_means_rgb=pixel_means_rgb, trunc_u8=True, want=want)
    else:
        lp = torch.from_numpy(_lighting.modelnet_light_position(obs)).to(dev)
        r = ctx.render_lit(cls, tgt, K, lp, torch.from_numpy(light.draw(B)).to(dev), light.brightness_ratio,
                           pixel_means_rgb=pixel_means_rgb, want=want)
    if background is not None:
        bank, draws = background
        if np.ndim(draws) == 0:
            draws = augment.background_draws(B, np.random.RandomState(int(draws)), len(bank))
        image_observed = ctx.replace_background(r["bgr"], r["mask"], draws, pixel_means_rgb)
    # the identity update: (0, 0, 0) is the zero translation delta only under T_means = 0, T_stds = 1, so this call keeps
    # train_update's defaults whatever the context's configuration
    ident = torch.tensor([[1.0, 0, 0, 0]] * B, dtype=torch.float32, device=dev)
    upd = ctx.train_update(cls, src, ident, torch.zeros(B, 3, device=dev), tgt, r["depth"], K, pixel_means_rgb=pixel_means_rgb,
                           lighting=_device_lighting(light, B, dev))
    rng = np.random.default_rng(seed)
    pts, pw = np.zeros((B, 3, num_points), np.float32), np.zeros((B, 3, num_points), np.float32)
    for b in range(B):
        v = meshes[cls_np[b]].verts
        keep = rng.permutation(len(v))[:num_points]
        pts[b, :, :len(keep)] = v[keep].T
        pw[b, :, :len(keep)] = 1
    pobs = np.stack([obs[b, :, :3].astype(np.float32) @ pts[b] + obs[b, :, 3:4].astype(np.float32) for b in range(B)]).astype(np.float32)
    box = r["bbox"] if init_mask == "box_gt" else ctx.render(cls, upd["src_pose"], K, pixel_means_rgb=pixel_means_rgb, want=("mask",))["bbox"]
    mask_observed = ctx.update_mask_box(box)
    if mask_dilate is not None:
        rs = mask_dilate if isinstance(mask_dilate, np.random.RandomState) else np.random.RandomState(int(mask_dilate))
        mask_observed = ctx.mask_dilate(mask_observed, augment.mask_dilate_draws(B, rs))
    batch = {"image_observed": r["image"] if image_observed is None else image_observed, "image_rendered": upd["image_rendered"], "mask_observed": mask_observed,
             "mask_gt_observed": r["mask"], "mask_rendered": upd["mask_rendered"], "src_pose": upd["src_pose"], "flow": upd["flow"],
             "flow_weights": upd["flow_weights"], "point_cloud_model": torch.from_numpy(pts).to(dev),
             "point_cloud_weights": torch.from_numpy(pw).to(dev), "point_cloud_observed": torch.from_numpy(pobs).to(dev),
             "pixel_means_rgb": np.asarray(pixel_means_rgb, np.float32)}
    if input_depth:
        batch["depth_observed"], batch["depth_rendered"] = r["depth"], upd["depth_rendered"]
    return batch, cls, tgt, r["depth"]


def _device_lighting(light, B, dev):
    """Context.train_update's lighting for one lit re-render of B instances (a fresh intensity draw), or None"""
    return None if light is None else light.lighting(torch.from_numpy(light.draw(B)).to(dev))


def fit_batch(trainer, batch, cls, tgt_pose, depth_gt, K, n_inner=4, dist=None, update_mask="fixed", lighting=None):
    """One data batch of Module.fit (deepim/core/module.py:1131-1137): n_inner x (forward_backward, update), the
    batch re-rendered at the predicted pose in between (batchUpdaterPyMulti.forward -> Context.train_update).
    lighting = None or the ModelNet branch's light ({"seed", "offset", "brightness_ratio"} or a lighting.LightSource, which
    keeps drawing fresh intensities across calls): the re-renders are lit (batch_updater_py_multi.py:187-229).
    The re-render composes the predicted delta under the context's trans_means / trans_stds / rot_coord, the
    parameterisation the step's Transform3D trained it in (batch_updater_py_multi.py:23-27, 179-180).
    Returns the objective of every inner iteration (device tensor [n_inner])."""
    ctx = trainer.ctx
    light = _lighting.LightSource.of(lighting)
    cfg = ctx.get_config()
    b = dict(batch)
    objs = []
    for it in range(n_inner):
        z = trainer.zoom_front(b, K)
        res = trainer.step(z, dist=dist)
        objs.append(res["losses"][3])
        if it != n_inner - 1:
            upd = ctx.train_update(cls, b["src_pose"], res["rot_est_norm"], res["trans_est"], tgt_pose, depth_gt, K,
                                   pixel_means_rgb=batch["pixel_means_rgb"], T_means=cfg["trans_means"],
                                   T_stds=cfg["trans_stds"], rot_coord=cfg["rot_coord"],
                                   lighting=_device_lighting(light, cls.shape[0], ctx.device))
            for k in ("image_rendered", "mask_rendered", "src_pose", "flow", "flow_weights"):
                b[k] = upd[k]
            if trainer.input_depth:  # the RGB-D network also sees the re-render's depth
                b["depth_rendered"] = upd["depth_rendered"]
            if update_mask == "box_rendered":  # what update_data_batch does at test time (data_pair.py:93-105); the reference's
                # training loop keeps mask_observed fixed (batch_updater_py_multi.py:267-301)
                rb = ctx.render(cls, upd["src_pose"], K, pixel_means_rgb=batch["pixel_means_rgb"], want=("mask",))["bbox"]
                b["mask_observed"] = ctx.update_mask_box(rb)
    return torch.stack(objs)
