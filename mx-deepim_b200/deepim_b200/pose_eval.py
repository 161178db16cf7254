"""ADD / ADI evaluation on the device -- the error metric of the headline benchmark (SURVEY 8 row a15).

Mirrors lib/utils/pose_error.py:72-108 (`add`, `adi`) and the counting / Simpson-AUC part of
LM6D_REFINE.evaluate_pose_add (lib/dataset/LM6D_REFINE.py:372-512): accuracy at 0.02 / 0.05 / 0.10 x diameter and the
area under the accuracy-vs-threshold curve over [0, 0.1 d] with step 1e-4 (scipy.integrate.simps, dx = 1e-4, / 0.1)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from ._capi import check, lib

SYMMETRIC_CLASSES = ("eggbox", "glue", "bowl", "cup")  # LM6D_REFINE.py:418-420


def _p(t):
    return C.c_void_p(t.data_ptr())


def pose_errors(ctx, poses_est, poses_gt, points, symmetric=False):
    """poses_est / poses_gt: [M,3,4] float64 (CUDA tensors or numpy), points [N,3] (float64 on the device).  Returns float64 CUDA [M]."""
    dev = ctx.device
    pe = torch.as_tensor(poses_est, dtype=torch.float64, device=dev).contiguous()
    pg = torch.as_tensor(poses_gt, dtype=torch.float64, device=dev).contiguous()
    pts = torch.as_tensor(np.asarray(points, np.float64), dtype=torch.float64, device=dev).contiguous()
    out = torch.empty(pe.shape[0], dtype=torch.float64, device=dev)
    check(lib.dim_pose_error(ctx._h, _p(pe), _p(pg), pe.shape[0], _p(pts), pts.shape[0], int(symmetric), _p(out),
                             C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return out


def add(ctx, R_est, t_est, R_gt, t_gt, pts):
    """Call-compatible with lib/utils/pose_error.py:add (single pose pair)."""
    pe = np.hstack([np.asarray(R_est, np.float64), np.asarray(t_est, np.float64).reshape(3, 1)])[None]
    pg = np.hstack([np.asarray(R_gt, np.float64), np.asarray(t_gt, np.float64).reshape(3, 1)])[None]
    return float(pose_errors(ctx, pe, pg, pts, False)[0])


def adi(ctx, R_est, t_est, R_gt, t_gt, pts):
    """Call-compatible with lib/utils/pose_error.py:adi."""
    pe = np.hstack([np.asarray(R_est, np.float64), np.asarray(t_est, np.float64).reshape(3, 1)])[None]
    pg = np.hstack([np.asarray(R_gt, np.float64), np.asarray(t_gt, np.float64).reshape(3, 1)])[None]
    return float(pose_errors(ctx, pe, pg, pts, True)[0])


def pose_errors_2d(ctx, poses_est, poses_gt, points, K):
    """[M,3] float64 CUDA: (arp_2d in pixels, rotation distance in degrees, translation distance in metres) per pose pair --
    lib/utils/pose_error.py:55-69 `arp_2d` and lib/pair_matching/RT_transform.py:162-173 `calc_rt_dist_m` on the device."""
    dev = ctx.device
    pe = torch.as_tensor(poses_est, dtype=torch.float64, device=dev).contiguous()
    pg = torch.as_tensor(poses_gt, dtype=torch.float64, device=dev).contiguous()
    pts = torch.as_tensor(np.asarray(points, np.float64), dtype=torch.float64, device=dev).contiguous()
    Kd = torch.as_tensor(np.asarray(K, np.float64).reshape(9), dtype=torch.float64, device=dev).contiguous()
    out = torch.empty((pe.shape[0], 3), dtype=torch.float64, device=dev)
    check(lib.dim_pose_error_2d(ctx._h, _p(pe), _p(pg), pe.shape[0], _p(pts), pts.shape[0], _p(Kd), _p(out),
                                C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return out


def flow_epe(ctx, flow_pred, flow_gt, visible, bg):
    """calc_EPE_one_pair (deepim/core/tester.py:573-589) for a batch on the device: float32 CUDA tensors flow_* [B,2,H,W],
    visible / bg [B,1,H,W].  Returns a dict of float64 numpy arrays [B]: epe_all, num_all, epe_viz, num_viz, epe_vizbg,
    num_vizbg (sums, as the reference accumulates them before dividing)."""
    B = flow_pred.shape[0]
    for t in (flow_pred, flow_gt, visible, bg):
        if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
            raise TypeError("flow_epe expects contiguous float32 CUDA tensors")
    out = torch.empty((B, 6), dtype=torch.float64, device=ctx.device)
    check(lib.dim_flow_epe(ctx._h, _p(flow_pred), _p(flow_gt), _p(visible), _p(bg), B, _p(out),
                           C.c_void_p(torch.cuda.current_stream(ctx.device).cuda_stream)))
    o = out.cpu().numpy()
    return {k: o[:, i] for i, k in enumerate(("epe_all", "num_all", "epe_viz", "num_viz", "epe_vizbg", "num_vizbg"))}


RT_Z_FLIP = np.array([[-1.0, 0, 0, 0], [0, -1.0, 0, 0], [0, 0, 1.0, 0]])  # eggbox: 180 deg about z (LM6D_REFINE.py:304-307)


def _with_eggbox_flip(ctx, est, gt, pts, K, flip):
    """errors [M,3]; where `flip` and the rotation distance exceeds 90 deg the estimate is replaced by est . RT_z first"""
    e = pose_errors_2d(ctx, est, gt, pts, K).cpu().numpy()
    if flip:
        bad = np.nonzero(e[:, 1] > 90.0)[0]
        if len(bad):
            sym = est[bad].copy()
            sym[:, :, :3] = est[bad][:, :, :3] @ RT_Z_FLIP[:, :3]     # se3_mul(est, RT_z): R R_z, translation unchanged (t_z = 0)
            e[bad] = pose_errors_2d(ctx, sym, gt[bad], pts, K).cpu().numpy()
    return e


def evaluate_pose(ctx, poses_est, poses_gt, cls_idx, points_per_class, K, class_names=None):
    """LM6D_REFINE.evaluate_pose (lib/dataset/LM6D_REFINE.py:278-371): rotation / translation / joint accuracy at
    (1..10 deg, 0.01..0.10 m); entry [4] of each = the paper's 5 cm 5 deg.  poses_est [n_iter,M,3,4], poses_gt [M,3,4].
    Returns per class and the mean over valid classes: rot_acc / trans_acc / space_acc [n_iter,10] in percent."""
    poses_est, poses_gt, cls_idx = np.asarray(poses_est, np.float64), np.asarray(poses_gt, np.float64), np.asarray(cls_idx)
    n_iter = poses_est.shape[0]
    rot_th, tr_th = np.arange(1, 11, 1), np.arange(0.01, 0.11, 0.01)
    res = {"classes": {}, "mean": {}}
    acc = {k: [] for k in ("rot_acc", "trans_acc", "space_acc")}
    for c, pts in enumerate(points_per_class):
        sel = np.nonzero(cls_idx == c)[0]
        if len(sel) == 0:
            continue
        flip = class_names is not None and class_names[c] == "eggbox"
        per = {k: np.zeros((n_iter, 10)) for k in acc}
        for it in range(n_iter):
            e = _with_eggbox_flip(ctx, poses_est[it, sel], poses_gt[sel], pts, K, flip)
            for k in range(10):
                r_ok, t_ok = e[:, 1] < rot_th[k], e[:, 2] < tr_th[k]
                per["rot_acc"][it, k] = 100.0 * r_ok.mean()
                per["trans_acc"][it, k] = 100.0 * t_ok.mean()
                per["space_acc"][it, k] = 100.0 * np.logical_and(r_ok, t_ok).mean()
        res["classes"][c] = per
        for k in acc:
            acc[k].append(per[k])
    for k in acc:
        res["mean"][k] = np.mean(acc[k], axis=0) if acc[k] else np.zeros((n_iter, 10))
    res["mean"]["5cm5deg"] = res["mean"]["space_acc"][:, 4].tolist()
    return res


def evaluate_pose_arp_2d(ctx, poses_est, poses_gt, cls_idx, points_per_class, K, class_names=None):
    """LM6D_REFINE.evaluate_pose_arp_2d (lib/dataset/LM6D_REFINE.py:514-): accuracy of the average 2D re-projection error at
    2 / 5 / 10 / 20 px (5 px = the paper's "Proj. 2D") and the Simpson area of the accuracy curve over [0, 50) px, step 0.1."""
    poses_est, poses_gt, cls_idx = np.asarray(poses_est, np.float64), np.asarray(poses_gt, np.float64), np.asarray(cls_idx)
    n_iter = poses_est.shape[0]
    dx = 0.1
    th = np.arange(0, 50, dx).astype(np.float32)
    res = {"classes": {}, "mean": {}}
    sums = {k: np.zeros(n_iter) for k in ("auc", "2", "5", "10", "20")}
    nvalid = 0
    for c, pts in enumerate(points_per_class):
        sel = np.nonzero(cls_idx == c)[0]
        if len(sel) == 0:
            continue
        nvalid += 1
        flip = class_names is not None and class_names[c] == "eggbox"
        per = {k: [] for k in sums}
        for it in range(n_iter):
            e = _with_eggbox_flip(ctx, poses_est[it, sel], poses_gt[sel], pts, K, flip)[:, 0]
            n = float(len(sel))
            for k in ("2", "5", "10", "20"):
                per[k].append(100.0 * float((e < float(k)).sum()) / n)
            curve = np.array([(e < t).sum() for t in th], np.float32) / n
            per["auc"].append(simpson(curve, dx) / 50.0 * 100.0)
        for k in per:
            sums[k] += np.array(per[k])
        res["classes"][c] = per
    for k in sums:
        res["mean"][k] = (sums[k] / max(nvalid, 1)).tolist()
    return res


def evaluate_pose_vsd(errors, cls_idx, n_classes, theta=0.3):
    """Recall of the Visible Surface Discrepancy (Hodan et al., ECCVW 2016; the SIXD Challenge 2017 counts a pose as correct
    when e < theta = 0.3): errors [n_rows,M] float64 (one tau; e.g. PoseRefiner.vsd's err[:, k] per row), cls_idx [M].
    Returns per class and the mean over the classes that have instances: the percentage of instances with e < theta, per
    row (lists of n_rows)."""
    errors, cls_idx = np.asarray(errors, np.float64), np.asarray(cls_idx)
    res = {"classes": {}, "mean": {}}
    per = []
    for c in range(n_classes):
        sel = np.nonzero(cls_idx == c)[0]
        if len(sel) == 0:
            continue
        rec = [100.0 * float((e < theta).sum()) / float(len(sel)) for e in errors[:, sel]]
        res["classes"][c] = rec
        per.append(rec)
    res["mean"]["recall"] = np.mean(per, axis=0).tolist() if per else [0.0] * len(errors)
    return res


def simpson(y, dx):
    """Composite Simpson rule as scipy.integrate.simps(y, dx=dx) with the default even='avg' handling for an even
    number of samples (average of 'first N-2 intervals + trapezoid on the last' and 'trapezoid on the first + last N-2')."""
    y = np.asarray(y, np.float64)
    n = len(y)
    if n % 2 == 1:
        return dx / 3.0 * (y[0] + y[-1] + 4 * y[1:-1:2].sum() + 2 * y[2:-1:2].sum())
    first = simpson(y[:-1], dx) + 0.5 * dx * (y[-1] + y[-2])
    last = simpson(y[1:], dx) + 0.5 * dx * (y[0] + y[1])
    return 0.5 * (first + last)


def evaluate_pose_add(ctx, poses_est, poses_gt, cls_idx, points_per_class, diameters, symmetric_flags):
    """poses_est [n_iter,M,3,4], poses_gt [M,3,4], cls_idx [M]; per class: points [N,3], diameter, symmetric flag.
    Returns dict with per-class and mean accuracies (percent) at 0.02/0.05/0.10 d and the AUC ('mean'), per iteration,
    computed exactly like LM6D_REFINE.evaluate_pose_add (errors come from the device kernel)."""
    poses_est = np.asarray(poses_est, np.float64)
    poses_gt = np.asarray(poses_gt, np.float64)
    cls_idx = np.asarray(cls_idx)
    n_iter = poses_est.shape[0]
    dx = 0.0001
    th = np.arange(0, 0.1, dx).astype(np.float32)
    res = {"classes": {}, "mean": {}}
    sums = {k: np.zeros(n_iter) for k in ("auc", "0.02", "0.05", "0.10")}
    nvalid = 0
    for c, pts in enumerate(points_per_class):
        sel = np.nonzero(cls_idx == c)[0]
        if len(sel) == 0:
            continue
        nvalid += 1
        d = float(diameters[c])
        per = {k: [] for k in ("auc", "0.02", "0.05", "0.10")}
        errs = []
        for it in range(n_iter):
            e = pose_errors(ctx, poses_est[it, sel], poses_gt[sel], pts, bool(symmetric_flags[c])).cpu().numpy()
            errs.append(e)
            n = float(len(sel))
            for k, f in (("0.02", 0.02), ("0.05", 0.05), ("0.10", 0.10)):
                per[k].append(100.0 * float((e < np.float32(f * d)).sum()) / n)
            curve = np.array([(e < t).sum() for t in (th * np.float32(d))], np.float32) / n
            per["auc"].append(simpson(curve, dx) / 0.1 * 100.0)
        for k in per:
            sums[k] += np.array(per[k])
        res["classes"][c] = dict(per, errors=np.stack(errs))
    for k in sums:
        res["mean"][k] = (sums[k] / max(nvalid, 1)).tolist()
    return res
