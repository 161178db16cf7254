"""PoseRefiner: the batched, device-resident replacement of the per-instance test loop in
deepim/core/tester.py:284-485 (pred_eval's hot loop: predict -> RT_transform -> render ->
update_data_batch -> predict ...).  Also lifts the reference's batch=1 / single-GPU limitation
(tester.py:83, SURVEY 3.1): any number of instances, sharded over ranks.

Two device contexts on two CUDA streams are used round-robin, so the H2D copy of batch k+1 overlaps
the kernels of batch k (instances are independent; nothing else is shared but read-only weights).

lighting={"seed", "offset", "brightness_ratio"} runs the ModelNet branch's lit loop (deepim_b200.lighting): every mesh must
carry `normals`, and each submit draws its light intensities [n_iter, n, 3] from one Generator seeded once
(lighting.sample_intensity), the fresh draw per render of the reference.

input_depth=True runs the RGB-D network (config.network.INPUT_DEPTH; weights with a (64, 10, 7, 7) flow_conv1): submit /
refine then also take the observed depth as the loader's uint16 file values [N,H,W] (LINEMOD's *-depth.png), converted on the
device as float32(u16) / float32(depth_factor).

input_mask=False runs the image-only network (config.network.INPUT_MASK: False; weights with a (64, 6, 7, 7) flow_conv1): the
loop zooms with ZoomImage, boxes from the images' colours.

refine_frames / submit_frames refine instances that share observed frames (several objects in one image, several initial
hypotheses of one object) against one uploaded copy of each frame (dim_refine_host_async with a frame map).

Several cameras in one batch: refine_frames(..., K_frames=[F,3,3]) / submit_frames(..., K_frames=[f,3,3]) give every frame
its own intrinsics, refine(..., K=[N,3,3]) / submit(..., K=[n,3,3]) every instance (no frame map: instance i uses row i);
dim_refine_host_async renders and zooms each instance with its frame's K.  Without them the refiner's K serves every
instance."""
from __future__ import annotations

import numpy as np
import torch

from . import _capi as capi
from . import lighting as _lighting
from . import sharding, synth
from .context import Context


def plan_frame_batches(frame_of, n_frames: int, max_batch: int, lo: int = 0, hi=None, K_frames=None):
    """Device batches of PoseRefiner.refine_frames for instances [lo, hi) (default: all) of frame_of (instance i observes
    frame frame_of[i] of n_frames): the contiguous slices of at most max_batch instances that refine() uses (sharding.chunks),
    each with the frames it observes.  Returns [(a, b, frames, local)]: instances a..b-1, frames = the sorted global indices
    of their frames (at most b - a <= max_batch of them), local int32 [b - a] = each instance's index into `frames`, so
    frames[local[i]] == frame_of[a + i].  Raises ValueError naming the first instance whose frame index is outside
    [0, n_frames).
    K_frames [n_frames,3,3] (one camera per frame): each entry gains a fifth element, the cameras of its frames
    K_frames[frames] (float32 [len(frames),3,3]), so that row local[i] is instance a + i's camera."""
    f = np.asarray(frame_of).reshape(-1)
    hi = len(f) if hi is None else hi
    bad = np.nonzero((f < 0) | (f >= n_frames))[0]
    if len(bad):
        raise ValueError("instance %d has frame index %d: out of range [0,%d)" % (bad[0], f[bad[0]], n_frames))
    if K_frames is not None:
        K_frames = np.asarray(K_frames, np.float32)
        if K_frames.shape != (n_frames, 3, 3):
            raise ValueError("K_frames: expected shape %s, got %s" % ((n_frames, 3, 3), K_frames.shape))
    out = []
    for a, b in sharding.chunks(lo, hi, max_batch):
        frames, local = np.unique(f[a:b], return_inverse=True)
        e = (a, b, frames, local.astype(np.int32).reshape(-1))
        out.append(e if K_frames is None else e + (np.ascontiguousarray(K_frames[frames]),))
    return out


class PoseRefiner:
    def __init__(self, meshes, weights, K=synth.K_LINEMOD, device=0, max_batch=16, n_iter=4,
                 pixel_means_rgb=synth.PIXEL_MEANS_RGB, znear=synth.ZNEAR, zfar=synth.ZFAR, precision="fp16",
                 n_slots=2, lighting=None, input_depth=False, depth_factor=1000.0, input_mask=True):
        self.light = _lighting.LightSource.of(lighting)
        if self.light is not None:
            for i, m in enumerate(meshes):
                if getattr(m, "normals", None) is None:
                    raise ValueError("PoseRefiner(lighting=...): mesh %d has no per-vertex normals" % i)
        self.K = np.asarray(K, np.float32)
        self.n_iter, self.means, self.zn, self.zf = n_iter, np.asarray(pixel_means_rgb, np.float64), znear, zfar
        self.precision = capi.precision_id(precision)
        mv = max(len(m.verts) for m in meshes)
        mf = max(len(m.faces) for m in meshes)
        self.max_batch = max_batch
        self.input_depth, self.depth_factor = bool(input_depth), float(depth_factor)
        self.input_mask = bool(input_mask)
        self.slots = []
        for _ in range(n_slots):
            ctx = Context(device, max_batch=max_batch, max_classes=len(meshes), max_verts=mv, max_faces=mf,
                          input_depth=self.input_depth, input_mask=self.input_mask)
            for i, m in enumerate(meshes):
                ctx.upload_mesh(i, m)
            ctx.load_weights(weights)
            self.slots.append({
                "ctx": ctx, "stream": torch.cuda.Stream(device=ctx.device), "busy": False, "n": 0,
                "poses": torch.empty((n_iter, max_batch, 3, 4), dtype=torch.float64).pin_memory(),
                "se3": torch.empty((n_iter, max_batch, 7), dtype=torch.float32).pin_memory(),
                "status": torch.zeros((min(n_iter, 8) * max_batch,), dtype=torch.int32).pin_memory(),
                "img": None, "cls": None, "pose": None, "depth": None, "frame": None, "K": None,
                "intensity": torch.empty((n_iter, max_batch, 3), dtype=torch.float32).pin_memory() if self.light else None,
            })
        self.ctx = self.slots[0]["ctx"]
        self._next = 0

    # ------------------------------------------------------------------ pipelined submit / result
    def _pinned(self, slot, key, arr, dtype):
        t = arr if isinstance(arr, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(arr))
        if t.dtype != dtype:
            t = t.to(dtype)
        if t.is_pinned() and t.is_contiguous():
            return t
        buf = slot[key]
        if buf is None or buf.shape[1:] != t.shape[1:] or buf.shape[0] < t.shape[0]:
            buf = torch.empty((self.max_batch,) + tuple(t.shape[1:]), dtype=dtype).pin_memory()
            slot[key] = buf
        buf[: t.shape[0]].copy_(t)
        return buf[: t.shape[0]]

    def submit(self, images_bgr_u8, cls_idx, poses_init, depths_u16=None, K=None):
        """Enqueue one batch (<= max_batch instances, host arrays; pinned torch tensors are used in place).
        depths_u16: uint16 [n,H,W], required with input_depth=True.  K: None = the refiner's K; float32 [n,3,3] = each
        instance's own camera.
        Returns a ticket for result().  At most len(slots) batches may be in flight."""
        return self._submit(images_bgr_u8, None, cls_idx, poses_init, depths_u16, K)

    def submit_frames(self, frames_bgr_u8, frame_idx, cls_idx, poses_init, depths_u16=None, K_frames=None):
        """submit() against shared frames: frames_bgr_u8 uint8 [f,H,W,3] (f <= max_batch), frame_idx int [n] (instance i
        observes frames_bgr_u8[frame_idx[i]]; checked before anything is enqueued), depths_u16 uint16 [f,H,W] with
        input_depth=True.  Each frame is uploaded once.  K_frames: None = the refiner's K; float32 [f,3,3] = each frame's
        camera (checked before anything is enqueued)."""
        return self._submit(frames_bgr_u8, frame_idx, cls_idx, poses_init, depths_u16, K_frames)

    def _submit(self, images_bgr_u8, frame_idx, cls_idx, poses_init, depths_u16, K_frames):
        i = self._next
        slot = self.slots[i]
        if slot["busy"]:
            raise RuntimeError("PoseRefiner: slot still in flight; call result() first")
        n = len(cls_idx)
        if n > self.max_batch:
            raise ValueError("batch larger than max_batch")
        if len(images_bgr_u8) > self.max_batch:
            raise ValueError("more frames than max_batch")
        img = self._pinned(slot, "img", images_bgr_u8, torch.uint8)
        cls = self._pinned(slot, "cls", cls_idx, torch.int32)
        pose = self._pinned(slot, "pose", poses_init, torch.float64)
        if (depths_u16 is not None) != self.input_depth:
            raise ValueError("PoseRefiner(input_depth=%s): depths_u16 %s" % (self.input_depth,
                             "is required" if self.input_depth else "belongs to PoseRefiner(input_depth=True)"))
        depth = None if depths_u16 is None else self._pinned(slot, "depth", depths_u16, torch.uint16)
        lit = None
        if self.light is not None:  # a fresh draw per render; the pinned buffer lives until result() of this slot
            inten = slot["intensity"].view(-1)[: self.n_iter * n * 3].view(self.n_iter, n, 3)
            inten.copy_(torch.from_numpy(self.light.draw((self.n_iter, n))))
            lit = self.light.lighting(inten)
        fidx = None if frame_idx is None else self._pinned(slot, "frame", frame_idx, torch.int32)
        K = self.K if K_frames is None else self._pinned(slot, "K", np.asarray(K_frames, np.float32), torch.float32)
        with torch.cuda.stream(slot["stream"]):
            slot["ctx"]._refine_host(img, fidx, cls, pose, K, self.n_iter, self.zn, self.zf, self.means, self.precision,
                                     slot["poses"], slot["se3"], False, lit, depth, self.depth_factor,
                                     ("images_bgr_u8", "depths_u16"))
            slot["ctx"].refine_status(n, self.n_iter, out=slot["status"], sync=False)
        slot["busy"], slot["n"] = True, n
        self._next = (i + 1) % len(self.slots)
        return i

    def result(self, ticket, strict=True):
        """Block until the batch is done; returns poses [n_iter, n, 3, 4] float64 (numpy copy).
        The per-iteration device status is checked: an instance whose object left the view frustum (empty rendered mask;
        the reference crashes in ZoomMask there; image-only network: an observed image with no valid pixel) or whose class
        index is invalid raises DeepIMError when strict, else the flags are left in `self.last_status` ([n_iter, n] int32) for
        the caller.  Bit 2 (image-only network: empty render, the zoom centred on the observed box as the reference does) is
        reported there but does not raise."""
        slot = self.slots[ticket]
        slot["stream"].synchronize()
        slot["busy"] = False
        n, B = slot["n"], self.max_batch
        ni = min(self.n_iter, 8)
        self.last_status = slot["status"][: ni * n].view(ni, n).numpy().copy()
        if strict and (self.last_status & 3).any():
            bad = sorted(set(np.nonzero(self.last_status & 3)[1].tolist()))
            raise capi.DeepIMError("PoseRefiner: instances %s of the batch have a non-zero device status (bit 0: empty rendered "
                                   "mask -- object left the frustum; bit 1: bad class index): %s"
                                   % (bad, self.last_status[:, bad].tolist()))
        # refine_host packs outputs densely as [n_iter, n, ...] at the start of the pinned buffer
        p = slot["poses"].view(-1)[: self.n_iter * n * 12].view(self.n_iter, n, 3, 4)
        return p.numpy().copy()

    # ------------------------------------------------------------------------------ convenience
    def refine(self, images_bgr_u8, cls_idx, poses_init, dist=None, depths_u16=None, K=None):
        """images_bgr_u8 [N,H,W,3] uint8 (cv2 layout), cls_idx [N] int, poses_init [N,3,4] float64 (host); depths_u16 [N,H,W]
        uint16 with input_depth=True; K: None = the refiner's K for every instance, [N,3,3] = each instance's own camera
        (several cameras in one batch; instance i's poses equal refine() by a refiner built with K[i], bit for bit).
        Returns poses [n_iter,N,3,4] float64 (host).  With torch.distributed initialised each rank
        processes its contiguous slice and the poses are all-gathered."""
        n = len(cls_idx)
        if K is not None:
            K = np.asarray(K, np.float32)
            if K.shape != (n, 3, 3):
                raise ValueError("K: expected one camera per instance %s, got %s" % ((n, 3, 3), K.shape))
        rank, world = (dist.get_rank(), dist.get_world_size()) if dist is not None and dist.is_initialized() else (0, 1)
        lo, hi = sharding.shard_range(n, rank, world)
        out = np.zeros((self.n_iter, hi - lo, 3, 4), np.float64)
        pending = []
        for a, b in sharding.chunks(lo, hi, self.max_batch):
            if len(pending) == len(self.slots):
                t, (pa, pb) = pending.pop(0)
                out[:, pa - lo:pb - lo] = self.result(t)
            d = None if depths_u16 is None else depths_u16[a:b]
            k = None if K is None else K[a:b]
            pending.append((self.submit(images_bgr_u8[a:b], cls_idx[a:b], poses_init[a:b], d, k), (a, b)))
        for t, (pa, pb) in pending:
            out[:, pa - lo:pb - lo] = self.result(t)
        return sharding.gather_results(out, n, axis=1, dist=dist, device=self.ctx.device if world > 1 else None)

    def refine_frames(self, frames_bgr_u8, frame_of, cls_idx, poses_init, dist=None, depths_u16=None, K_frames=None):
        """refine() with instances that share observed frames (several objects of one image, several initial hypotheses of
        one object): frames_bgr_u8 [F,H,W,3] uint8, frame_of [N] int (instance i observes frames_bgr_u8[frame_of[i]]),
        cls_idx [N], poses_init [N,3,4] float64; depths_u16 [F,H,W] uint16 with input_depth=True.
        The device batches are refine()'s (plan_frame_batches), each uploading only the frames its instances observe, so the
        result equals refine(frames_bgr_u8[frame_of], ...) bit for bit; keeping the instances of a frame next to each other
        uploads each frame once.  Sharded over instances like refine(): a rank uploads the frames of its slice only.
        K_frames: None = the refiner's K; [F,3,3] = each frame's camera, carried into every device batch with its frames
        (plan_frame_batches), so instance i's poses equal a refiner built with K_frames[frame_of[i]], bit for bit."""
        n = len(cls_idx)
        if len(frame_of) != n:
            raise ValueError("frame_of has %d entries for %d instances" % (len(frame_of), n))
        rank, world = (dist.get_rank(), dist.get_world_size()) if dist is not None and dist.is_initialized() else (0, 1)
        lo, hi = sharding.shard_range(n, rank, world)
        out = np.zeros((self.n_iter, hi - lo, 3, 4), np.float64)
        pending = []
        for a, b, frames, local, *k in plan_frame_batches(frame_of, len(frames_bgr_u8), self.max_batch, lo, hi, K_frames):
            if len(pending) == len(self.slots):
                t, (pa, pb) = pending.pop(0)
                out[:, pa - lo:pb - lo] = self.result(t)
            d = None if depths_u16 is None else depths_u16[frames]
            pending.append((self.submit_frames(frames_bgr_u8[frames], local, cls_idx[a:b], poses_init[a:b], d, *k), (a, b)))
        for t, (pa, pb) in pending:
            out[:, pa - lo:pb - lo] = self.result(t)
        return sharding.gather_results(out, n, axis=1, dist=dist, device=self.ctx.device if world > 1 else None)

    def icp(self, depths_u16, cls_idx, poses, K_frames=None, frame_of=None, n_iter=10, max_dist=0.02, min_points=64):
        """Point-to-plane ICP of poses against the observed depth (Context.icp, dim_icp), typically on refine()'s last poses.
        depths_u16 uint16 [F,H,W] host (the *-depth.png values), converted on the device as float32(u16) /
        float32(depth_factor); cls_idx [N]; poses [N,3,4] float64 host.  frame_of None = instance i observes frame i (F == N),
        else int [N]; K_frames None = the refiner's K, else float32 [F,3,3] = each frame's camera.
        The device batches are refine_frames()'s (plan_frame_batches), pipelined over the slots, so instance i's results
        equal Context.icp's on its batch.  The defaults (10 iterations, 2 cm, 64 points) are starting values and have not
        been tuned.
        Returns host arrays: poses [n_iter,N,3,4] float64, inliers [n_iter,N] int32, rms [n_iter,N] float32 and status
        [n_iter,N] int32 (see Context.icp)."""
        n = len(cls_idx)
        poses = np.asarray(poses, np.float64)
        out = {"poses": np.zeros((n_iter, n, 3, 4)), "inliers": np.zeros((n_iter, n), np.int32),
               "rms": np.zeros((n_iter, n), np.float32), "status": np.zeros((n_iter, n), np.int32)}

        def call(ctx, dev, depth, cls, a, b, K, local):
            return ctx.icp(depth, cls, dev(poses[a:b]), K, n_iter, max_dist, min_points, local)

        return self._depth_batches(depths_u16, cls_idx, K_frames, frame_of, out, 1, call)

    def vsd(self, depths_u16, cls_idx, poses_est, poses_gt, K_frames=None, frame_of=None, delta=0.015, taus=(0.02,),
            visib_mode="sixd17", diameters=None):
        """Visible Surface Discrepancy of poses_est against poses_gt (Context.pose_error_vsd, dim_pose_error_vsd), batched
        and pipelined exactly as icp(): depths_u16, cls_idx, K_frames and frame_of as there, poses_est / poses_gt [N,3,4]
        float64 host; delta and taus in metres (the defaults are the SIXD Challenge 2017's 15 mm and 20 mm).
        visib_mode "bop19" and diameters [N] (metres; taus become fractions of them) give BOP 2019's VSD, as
        Context.pose_error_vsd.
        Returns host arrays: err [N,n_tau] float64 and status [N] int32 (see Context.pose_error_vsd)."""
        n = len(cls_idx)
        poses_est, poses_gt = np.asarray(poses_est, np.float64), np.asarray(poses_gt, np.float64)
        taus = np.asarray(taus, np.float64).reshape(-1)
        diam = None if diameters is None else np.asarray(diameters, np.float64).reshape(-1)
        if diam is not None and len(diam) != n:
            raise ValueError("diameters has %d entries for %d instances" % (len(diam), n))
        out = {"err": np.zeros((n, len(taus))), "status": np.zeros(n, np.int32)}

        def call(ctx, dev, depth, cls, a, b, K, local):
            return ctx.pose_error_vsd(depth, cls, dev(poses_est[a:b]), dev(poses_gt[a:b]), K, delta, taus, local,
                                      self.zn, self.zf, visib_mode, None if diam is None else diam[a:b])

        return self._depth_batches(depths_u16, cls_idx, K_frames, frame_of, out, 0, call)

    def pose_error_sym(self, cls_idx, poses_est, poses_gt, points_per_class, syms_per_class, K=None):
        """BOP 2019's MSSD and MSPD (Context.pose_error_sym, dim_pose_error_sym) of N instances: cls_idx [N], poses_est /
        poses_gt [N,3,4] float64 host, points_per_class[c] [N_c,3] and syms_per_class[c] [S_c,3,4] (bop.symmetry_transforms)
        of every class present; K None = the refiner's K, [3,3] = one camera, [N,3,3] = each instance's own.
        The instances of each class go to the device in slices of max_batch, in their order, on the first slot's context.
        Returns host arrays: err [N,2] float64 (MSSD metres, MSPD pixels) and sym_idx [N,2] int32."""
        cls_idx = np.asarray(cls_idx)
        n = len(cls_idx)
        poses_est, poses_gt = np.asarray(poses_est, np.float64), np.asarray(poses_gt, np.float64)
        Ks = np.asarray(self.K if K is None else K, np.float64)
        Ks = np.broadcast_to(Ks.reshape(3, 3), (n, 3, 3)) if Ks.size == 9 else Ks.reshape(n, 3, 3)
        out = {"err": np.zeros((n, 2)), "sym_idx": np.zeros((n, 2), np.int32)}
        ctx = self.ctx
        dev = lambda x: torch.from_numpy(np.ascontiguousarray(x, np.float64)).to(ctx.device)
        for c in np.unique(cls_idx):
            sel = np.nonzero(cls_idx == c)[0]
            pts, sy = dev(points_per_class[c]), dev(syms_per_class[c])
            for a in range(0, len(sel), self.max_batch):
                s = sel[a:a + self.max_batch]
                r = ctx.pose_error_sym(dev(poses_est[s]), dev(poses_gt[s]), pts, sy, Ks[s])
                for k in out:
                    out[k][s] = r[k].cpu().numpy()
        return out

    def _depth_batches(self, depths_u16, cls_idx, K_frames, frame_of, out, axis, call):
        """icp / vsd over refine_frames()'s device batches (plan_frame_batches), pipelined over the slots: per batch the
        u16 depth of its frames is converted on the device, call(ctx, dev, depth, cls, a, b, K, local) enqueues the
        operation for instances a..b-1 on the slot's stream and returns its CUDA tensors, and out[key] receives them at
        [a:b] along `axis`.  Returns out."""
        depths_u16 = np.asarray(depths_u16, np.uint16)
        n = len(cls_idx)
        if frame_of is None:
            if len(depths_u16) != n:
                raise ValueError("frame_of is None (instance i observes frame i): %d frames for %d instances" % (len(depths_u16), n))
            frame_of = np.arange(n)
        elif len(frame_of) != n:
            raise ValueError("frame_of has %d entries for %d instances" % (len(frame_of), n))
        cls_idx = np.asarray(cls_idx, np.int32)
        pending = []

        def collect(i, a, b, res):
            self.slots[i]["stream"].synchronize()
            self.slots[i]["busy"] = False
            for k in out:
                out[k][(slice(None),) * axis + (slice(a, b),)] = res[k].numpy()

        for a, b, frames, local, *k in plan_frame_batches(frame_of, len(depths_u16), self.max_batch, 0, n, K_frames):
            if len(pending) == len(self.slots):
                collect(*pending.pop(0))
            i = self._next
            slot = self.slots[i]
            if slot["busy"]:
                raise RuntimeError("PoseRefiner: slot still in flight; call result() first")
            ctx = slot["ctx"]
            with torch.cuda.stream(slot["stream"]):
                dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(ctx.device, non_blocking=True)
                depth = ctx.depth_from_u16(dev(depths_u16[frames]), self.depth_factor)
                r = call(ctx, dev, depth, dev(cls_idx[a:b]), a, b, k[0] if k else self.K, dev(local))
                res = {key: torch.empty(v.shape, dtype=v.dtype).pin_memory().copy_(v, non_blocking=True)
                       for key, v in r.items()}
            slot["busy"] = True
            self._next = (i + 1) % len(self.slots)
            pending.append((i, a, b, res))
        for p in pending:
            collect(*p)
        return out

    def close(self):
        for s in self.slots:
            s["ctx"].close()
