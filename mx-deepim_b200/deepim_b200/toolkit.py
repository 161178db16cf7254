"""Rendered-pair synthesis on the CUDA rasteriser (SURVEY 8(f) row 3, second half): what toolkit/LM6d_1_gen_rendered_pose.py
and toolkit/LM6d_2_gen_rendered.py do for the LM6d_refine layout -- perturbed "rendered" poses around every observed pose,
their renders, depth maps and pose files, and the observed / rendered pair lists -- with the glumpy renderer replaced by
dim_render, batched.

  gen_rendered_poses   LM6d_1_gen_rendered_pose.py:77-125: euler-angle noise N(0, 15 deg) on the three sxyz angles,
                       translation noise N(0, (1, 1, 5) cm); redrawn while the rotation distance to the observed pose exceeds
                       45 deg or the projected centre is within 16 px of the image border
  write_rendered_set   LM6d_2_gen_rendered.py:60-150: <root>/data/rendered/<cls>/<prefix>_<k>-color.png (uint8 BGR),
                       -depth.png (uint16, metres x 1000), -pose.txt (class-index header + 3x4), and the pair list
                       <root>/image_set/<name>_<cls>.txt with lines "<observed index> <cls>/<prefix>_<k>"

The euler helpers are the static-xyz convention of lib/pair_matching/RT_transform.py:240-360 (R = Rz(ak) Ry(aj) Rx(ai)); they
are pinned to the live reference functions in tests/golden/ref_euler.npz.

The LM6d_refine_syn training set (toolkit/LM6d_ds_0 ... ds_4) and LM6d_refine's gt_observed renders (LM6d_0), with the glumpy
renderers replaced by dim_render_dataset:

  gen_syn_observed_poses  LM6d_ds_0_gen_observed_poses.py: per class the training poses' translation mean / std, the mean
                          of their rotated z axes and the largest angle to it; rejection-sampled normal quaternions and
                          translations inside that cone, centre 48 px inside the border
  syn_light_draws         LM6d_ds_1_gen_observed.py:113-148: per image the light position, colour and brightness ratio
  write_syn_observed_set  LM6d_ds_1 + ds_2: observed (lit) and gt_observed (unlit) images, depth, label, pose, the lists
  write_gt_observed_set   LM6d_0_gen_gt_observed.py: gt_observed pose / depth / label of every real frame
  gen_syn_set             ds_0 ... ds_4 in one call (ds_3 / ds_4 are gen_rendered_poses + write_rendered_set)

The random sequences, file names, pose files and lists are pinned to the live scripts in tests/golden/ref_syn.npz; the
images are compared with the CPU oracle.  PNG encoding runs on a host thread pool (`workers`): the device renders a batch
in a few milliseconds, the encoder is what takes the time."""
from __future__ import annotations

import hashlib
import math
import os
import pickle
import random
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import lm6d_io

# LM6d_ds_*.py / LM6d_0_gen_gt_observed.py constants
K_LM = np.array([[572.4114, 0, 325.2611], [0, 573.57043, 242.04899], [0, 0, 1]])
LM6D_IDX2CLASS = {1: "ape", 2: "benchvise", 4: "camera", 5: "can", 6: "cat", 8: "driller", 9: "duck", 10: "eggbox", 11: "glue",
                  12: "holepuncher", 13: "iron", 14: "lamp", 15: "phone"}
BRIGHTNESS_RATIOS = (0.2, 0.25, 0.3, 0.35, 0.4)     # ds_1 l.98
LIGHT_COLOURS = np.array([[0, 0, 1], [0, 1, 0], [0, 1, 1], [1, 0, 0], [1, 0, 1], [1, 1, 0], [1, 1, 1]])  # ds_1 l.140
LIGHT_OFFSETS = [[1, 0, 1], [1, 1, 1], [0, 1, 1], [-1, 1, 1], [-1, 0, 1], [0, 0, 1]]             # ds_1 l.113-128, idx % 6
GT_OBSERVED_COLOUR_FRAMES = ("000128", "000256", "000512")  # LM6d_0 writes the colour of these frames only
_FLOAT_EPS = np.finfo(float).eps


# ------------------------------------------------------------------------------------ quaternions (RT_transform.py)
def quat2mat(q):
    """RT_transform.quat2mat: the float64 expression order of the reference (unnormalised quaternions allowed)"""
    w, x, y, z = q
    Nq = w * w + x * x + y * y + z * z
    if Nq < _FLOAT_EPS:
        return np.eye(3)
    s = 2.0 / Nq
    X, Y, Z = x * s, y * s, z * s
    wX, wY, wZ = w * X, w * Y, w * Z
    xX, xY, xZ = x * X, x * Y, x * Z
    yY, yZ, zZ = y * Y, y * Z, z * Z
    return np.array([[1.0 - (yY + zZ), xY - wZ, xZ + wY], [xY + wZ, 1.0 - (xX + zZ), yZ - wX], [xZ - wY, yZ + wX, 1.0 - (xX + yY)]])


def mat2quat(M):
    """RT_transform.mat2quat (Bar-Itzhack): the eigenvector of the largest eigenvalue of the symmetric 4x4, w >= 0"""
    Qxx, Qyx, Qzx, Qxy, Qyy, Qzy, Qxz, Qyz, Qzz = np.asarray(M).flat
    Kq = np.array([[Qxx - Qyy - Qzz, 0, 0, 0], [Qyx + Qxy, Qyy - Qxx - Qzz, 0, 0], [Qzx + Qxz, Qzy + Qyz, Qzz - Qxx - Qyy, 0],
                   [Qyz - Qzy, Qzx - Qxz, Qxy - Qyx, Qxx + Qyy + Qzz]]) / 3.0
    vals, vecs = np.linalg.eigh(Kq)
    q = vecs[[3, 0, 1, 2], np.argmax(vals)]
    if q[0] < 0:
        q *= -1
    return q


def se3_q2m(se3_q):
    """RT_transform.se3_q2m: [qw qx qy qz tx ty tz] -> 3x4"""
    se3_q = np.asarray(se3_q)
    m = np.zeros((3, 4))
    m[:, :3] = quat2mat(se3_q[0:4] / np.linalg.norm(se3_q[0:4]))
    m[:, 3] = se3_q[4:]
    return m

_EPS4 = np.finfo(float).eps * 4.0


def euler2mat(ai, aj, ak):
    """static x-y-z euler angles -> rotation matrix (RT_transform.euler2mat, axes='sxyz')"""
    si, sj, sk = math.sin(ai), math.sin(aj), math.sin(ak)
    ci, cj, ck = math.cos(ai), math.cos(aj), math.cos(ak)
    cc, cs, sc, ss = ci * ck, ci * sk, si * ck, si * sk
    return np.array([[cj * ck, sj * sc - cs, sj * cc + ss],
                     [cj * sk, sj * ss + cc, sj * cs - sc],
                     [-sj, cj * si, cj * ci]])


def mat2euler(M):
    """rotation matrix -> static x-y-z euler angles (RT_transform.mat2euler, axes='sxyz')"""
    M = np.asarray(M, np.float64)
    cy = math.sqrt(M[0, 0] * M[0, 0] + M[1, 0] * M[1, 0])
    if cy > _EPS4:
        return math.atan2(M[2, 1], M[2, 2]), math.atan2(-M[2, 0], cy), math.atan2(M[1, 0], M[0, 0])
    return math.atan2(-M[1, 2], M[1, 1]), math.atan2(-M[2, 0], cy), 0.0


def rot_dist_deg(Ra, Rb):
    """rotation part of calc_rt_dist_m (RT_transform.py:162-173): angle of Ra Rb^T in degrees"""
    c = (np.trace(np.asarray(Ra) @ np.asarray(Rb).T) - 1.0) / 2.0
    return math.degrees(math.acos(min(1.0, max(-1.0, c))))


def gen_rendered_poses(poses_observed, K, n_per_observed=10, angle_std=15.0, angle_max=45.0, xyz_std=(0.01, 0.01, 0.05),
                       width=640, height=480, margin=16, seed=2333, max_draws=10000):
    """[N,3,4] observed poses -> [N, n_per_observed, 3, 4] rendered poses.  Rejection rule and noise model as in the
    reference script; the random stream is numpy's legacy RandomState(seed) drawn in the script's order (three angles, then
    x, y, z).  (The script's own sequence is not reproducible beyond its first draw: scipy's logm inside calc_rt_dist_m pulls
    from the same global generator.)"""
    rs = np.random.RandomState(seed)
    K = np.asarray(K, np.float64).reshape(3, 3)
    P = np.asarray(poses_observed, np.float64).reshape(-1, 3, 4)
    out = np.zeros((len(P), n_per_observed, 3, 4))
    for a, src in enumerate(P):
        e = np.array(mat2euler(src[:, :3]))
        for k in range(n_per_observed):
            for draw in range(max_draws):
                te = e + rs.normal(0, angle_std / 180.0 * math.pi, 3)
                tt = src[:, 3] + np.array([rs.normal(0, s, 1)[0] for s in xyz_std])
                R = euler2mat(te[0], te[1], te[2])
                c = K @ tt
                cx, cy = c[0] / c[2], c[1] / c[2]
                if rot_dist_deg(R, src[:, :3]) <= angle_max and margin < cx < width - margin and margin < cy < height - margin:
                    break
            else:
                raise RuntimeError("no admissible rendered pose after %d draws (observed pose %d)" % (max_draws, a))
            out[a, k, :, :3], out[a, k, :, 3] = R, tt
    return out


def write_rendered_set(root, ctx, cls_name, cls_idx, mesh_slot, observed_indices, poses_rendered, K, set_name="train",
                       znear=0.25, zfar=6.0, batch=16, first_only_in_set=False, syn_names=False, workers=1):
    """Render every pose of poses_rendered [N, n, 3, 4] (class `mesh_slot` of `ctx`) and write the rendered half of an
    LM6d_refine directory + the pair list.  observed_indices[i] is the observed index "<video>/<prefix>" of row i.
    first_only_in_set: list only rendered pose 0 of every observed frame (the reference's validation pairs).
    syn_names: the LM6d_refine_syn layout of LM6d_ds_4_gen_rendered.py (l.86-140): files <cls>_<prefix>_<k>-* and the pair
    list sorted.  workers: PNG encoder threads."""
    import torch
    N, n = poses_rendered.shape[:2]
    d = os.path.join(root, "data", "rendered", cls_name)
    os.makedirs(d, exist_ok=True)
    os.makedirs(os.path.join(root, "image_set"), exist_ok=True)
    flat = poses_rendered.reshape(N * n, 3, 4)
    names = [("%s_%s_%d" % (cls_name, observed_indices[i].split("/")[1], k)) if syn_names else
             ("%s_%d" % (observed_indices[i].split("/")[1], k)) for i in range(N) for k in range(n)]
    dev = ctx.device
    with _BatchWriter(workers) as out:
        for lo in range(0, N * n, batch):
            hi = min(N * n, lo + batch)
            cls = torch.full((hi - lo,), mesh_slot, dtype=torch.int32, device=dev)
            r = ctx.render(cls, torch.from_numpy(flat[lo:hi].astype(np.float32)).to(dev), K, znear, zfar, trunc_u8=False,
                           want=("bgr", "depth"))
            bgr, depth = r["bgr"].cpu().numpy(), r["depth"].cpu().numpy()[:, 0]
            for j in range(hi - lo):
                base = os.path.join(d, names[lo + j])
                out.image(base + "-color.png", bgr[j].astype(np.uint8))                 # rgb_gl.astype('uint8') (l.103)
                out.image(base + "-depth.png", (depth[j] * lm6d_io.DEPTH_FACTOR).astype(np.uint16))   # truncation like l.105
                lm6d_io.write_pose(base + "-pose.txt", cls_idx, flat[lo + j])
    lines = ["%s %s/%s" % (observed_indices[i], cls_name, names[i * n + k]) for i in range(N)
             for k in range(1 if first_only_in_set else n)]
    if syn_names:
        lines = sorted(lines)
    with open(os.path.join(root, "image_set", "%s_%s.txt" % (set_name, cls_name)), "w") as f:
        f.write("\n".join(lines) + "\n")
    return lines


class _BatchWriter:
    """cv2.imwrite of every file of a writer, on `workers` host threads (cv2 releases the GIL while it encodes); inline
    for workers <= 1.  Leaving the with-block waits for every file and re-raises the first failure."""

    def __init__(self, workers=1):
        self._cv2 = lm6d_io._cv2()
        self._pool = ThreadPoolExecutor(workers) if workers > 1 else None
        self._pending = []

    def _write(self, path, img):
        if not self._cv2.imwrite(path, img):
            raise IOError("cv2.imwrite failed: %s" % path)

    def image(self, path, img):
        if self._pool is None:
            self._write(path, img)
        else:
            self._pending.append(self._pool.submit(self._write, path, img))
            if len(self._pending) > 4096:
                self._drain(2048)

    def _drain(self, keep=0):
        while len(self._pending) > keep:
            self._pending.pop(0).result()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        try:
            self._drain()
        finally:
            if self._pool is not None:
                self._pool.shutdown(wait=True)
        return False


def _write_pose_txt(path, cls_idx, pose):
    """the scripts' pose file: "{}" of the class index, then "{} {} {} {}" rows of the float64 3x4, no final newline"""
    with open(path, "w") as f:
        f.write("{}\n".format(cls_idx))
        f.write("\n".join(" ".join("{}".format(v) for v in row) for row in np.asarray(pose).reshape(3, 4)))


def _angle(u, v):
    """LM6d_ds_0 angle(): degrees between u and v"""
    c = np.dot(u, v) / (np.linalg.norm(u) * np.linalg.norm(v))
    rad = np.arccos(np.clip(c, -1, 1))
    return rad / np.pi * 180


def gen_syn_observed_poses(train_poses_by_class, K=K_LM, num_images=10000, seed=2333, width=640, height=480, margin=48):
    """LM6d_ds_0_gen_observed_poses.py.  train_poses_by_class {class: [N,3,4] float64} are the real training frames'
    gt_observed poses (np.loadtxt(skiprows=1) of data/gt_observed/<cls>/<prefix>-pose.txt for <cls>_train.txt).  Returns
    {class: [num_images, 7] float64 holding float32 values [qw qx qy qz tx ty tz]}, the script's pickle.
    The classes are sampled in sorted order from one numpy RandomState(seed), drawn as the script draws the global generator,
    with its float64 expressions in its order: one accept / reject decision taken differently would change every later pose."""
    pz = np.array([0, 0, 1])
    K = np.asarray(K, np.float64)
    stats = {}
    for cls_name, poses in train_poses_by_class.items():  # stat_poses
        poses = np.asarray(poses, np.float64).reshape(-1, 3, 4)
        trans = np.zeros((len(poses), 7))
        new_pz = []
        for i, pose in enumerate(poses):
            trans[i, 4:] = pose[:3, 3]
            new_pz.append(np.dot(pose[:3, :3], pz.reshape((-1, 1))).reshape((3,)))
        new_pz = np.array(new_pz)
        pz_mean = np.mean(new_pz, 0)
        deg_max = np.max(np.array([_angle(pz_mean, new_pz[i, :]) for i in range(new_pz.shape[0])]))
        stats[cls_name] = (np.mean(trans[:, 4:], 0), np.std(trans[:, 4:], 0), pz_mean, deg_max)
    rs = np.random.RandomState(seed)
    out = {}
    for cls_name in sorted(train_poses_by_class):  # gen_poses
        trans_mean, trans_std, pz_mean, deg_max = stats[cls_name]
        poses = np.zeros((num_images, 7))
        for i in range(num_images):
            while True:
                tgt_quat = rs.normal(0, 1, 4)
                tgt_quat = tgt_quat / np.linalg.norm(tgt_quat)
                if tgt_quat[0] < 0:
                    tgt_quat *= -1
                tgt_trans = rs.normal(trans_mean, trans_std)
                new_pz = np.dot(quat2mat(tgt_quat), pz.reshape((-1, 1))).reshape((3,))
                deg = _angle(new_pz, pz_mean)
                transform = np.matmul(K, tgt_trans.reshape(3, 1))
                center_x = float(transform[0, 0] / transform[2, 0])
                center_y = float(transform[1, 0] / transform[2, 0])
                if not (deg > deg_max or not (margin < center_x < (width - margin) and margin < center_y < (height - margin))):
                    break
            q = np.zeros((7,), dtype="float32")
            q[:4] = tgt_quat
            q[4:] = tgt_trans
            poses[i, :] = q
        out[cls_name] = poses
    return out


def syn_poses_sha256(syn_poses):
    """SHA-256 over the [N,7] float64 pose arrays in sorted class order"""
    h = hashlib.sha256()
    for c in sorted(syn_poses):
        h.update(np.ascontiguousarray(syn_poses[c], np.float64).tobytes())
    return h.hexdigest()


def syn_light_draws(syn_poses_by_class, seed=2333):
    """The per-image light of LM6d_ds_1_gen_observed.py (l.113-148) over the sorted classes: position = the offset of
    idx % 6 times 0.5 plus (t_x, -t_y, -t_z) (GL camera frame), then np.random.uniform(0.9, 1.1, 3), random.randint(0, 6)
    for the colour and random.randint(0, 4) for the brightness ratio, from numpy's RandomState(seed) and
    random.Random(seed) -- the script's two global generators, interleaved per image.
    Returns {class: {"position" [N,3], "intensity" [N,3] float64, "ratio_k" [N] int}}."""
    rs, rnd = np.random.RandomState(seed), random.Random(seed)
    out = {}
    for cls_name in sorted(syn_poses_by_class):
        q = np.asarray(syn_poses_by_class[cls_name])
        n = len(q)
        pos, inten, rk = np.zeros((n, 3)), np.zeros((n, 3)), np.zeros(n, np.int64)
        for idx in range(n):
            t = se3_q2m(q[idx])[:, 3]
            light = np.array(LIGHT_OFFSETS[idx % 6]) * 0.5
            light[0] += t[0]
            light[1] -= t[1]
            light[2] -= t[2]
            intensity = rs.uniform(0.9, 1.1, size=(3,))
            colour_k = rnd.randint(0, LIGHT_COLOURS.shape[0] - 1)
            pos[idx], inten[idx] = light, LIGHT_COLOURS[colour_k] * intensity
            rk[idx] = rnd.randint(0, len(BRIGHTNESS_RATIOS) - 1)
        out[cls_name] = {"position": pos, "intensity": inten, "ratio_k": rk}
    return out


def _device_batch(ctx, slot, poses32, K, znear, zfar, want, light=None):
    import torch
    dev = ctx.device
    B = len(poses32)
    kw = {}
    if light is not None:
        kw = {"light_position": torch.from_numpy(np.asarray(light[0], np.float32)).to(dev),
              "light_intensity": torch.from_numpy(np.asarray(light[1], np.float32)).to(dev),
              "brightness_ratio": torch.from_numpy(np.asarray(light[2], np.float32)).to(dev)}
    r = ctx.render_dataset(torch.full((B,), slot, dtype=torch.int32, device=dev),
                           torch.from_numpy(np.ascontiguousarray(poses32, np.float32)).to(dev), K, znear, zfar,
                           lm6d_io.DEPTH_FACTOR, want=want, **kw)
    return {k: v.cpu().numpy() for k, v in r.items()}


def write_syn_observed_set(root, ctx, syn_poses_by_class, light_draws, mesh_slots, K=K_LM, znear=0.25, zfar=6.0, batch=16,
                           workers=1):
    """LM6d_ds_1_gen_observed.py + LM6d_ds_2_gen_gt_observed.py: for every class (sorted; mesh_slots[class] = its mesh in
    ctx) and image idx, <root>/data/observed/<cls>/<idx:06d>-{color,depth,label,pose} (the Render_Py_Light render at the
    light of light_draws) and data/gt_observed/<cls>/<idx:06d>-{color,depth,label,pose} (the unlit render), and
    image_set/observed/LM6d_data_syn_train_observed_<cls>.txt.  The pose header is the index in the sorted class list.
    ds_1 renders quat2mat(mat2quat(R)) of the pose se3_q2m(q), ds_2 R itself: where their float32 casts agree (the usual
    case) one render gives both images, otherwise a batch is rendered once per pose."""
    classes = sorted(syn_poses_by_class)
    os.makedirs(os.path.join(root, "image_set", "observed"), exist_ok=True)
    with _BatchWriter(workers) as out:
        for class_idx, cls_name in enumerate(classes):
            q = np.asarray(syn_poses_by_class[cls_name])
            lt = light_draws[cls_name]
            d_obs = os.path.join(root, "data", "observed", cls_name)
            d_gt = os.path.join(root, "data", "gt_observed", cls_name)
            os.makedirs(d_obs, exist_ok=True)
            os.makedirs(d_gt, exist_ok=True)
            index = ["{}/{:06d}".format(cls_name, i + 1) for i in range(len(q))]
            with open(os.path.join(root, "image_set", "observed", "LM6d_data_syn_train_observed_{}.txt".format(cls_name)),
                      "w") as f:
                f.write("".join("{}\n".format(x) for x in index))
            for lo in range(0, len(q), batch):
                hi = min(len(q), lo + batch)
                pose = [se3_q2m(q[i]) for i in range(lo, hi)]
                gt32 = np.stack(pose).astype(np.float32)
                obs32 = np.stack([np.hstack([quat2mat(mat2quat(p[:3, :3])), p[:, -1:]]) for p in pose]).astype(np.float32)
                light = (lt["position"][lo:hi], lt["intensity"][lo:hi],
                         np.array([BRIGHTNESS_RATIOS[k] for k in lt["ratio_k"][lo:hi]]))
                if np.array_equal(obs32, gt32):
                    r_obs = r_gt = _device_batch(ctx, mesh_slots[cls_name], obs32, K, znear, zfar,
                                                 ("lit_bgr", "bgr", "depth", "label"), light)
                else:
                    r_obs = _device_batch(ctx, mesh_slots[cls_name], obs32, K, znear, zfar, ("lit_bgr", "depth", "label"),
                                          light)
                    r_gt = _device_batch(ctx, mesh_slots[cls_name], gt32, K, znear, zfar, ("bgr", "depth", "label"))
                for j, i in enumerate(range(lo, hi)):
                    prefix = index[i].split("/")[1]
                    for d, r, colour in ((d_obs, r_obs, "lit_bgr"), (d_gt, r_gt, "bgr")):
                        base = os.path.join(d, prefix)
                        out.image(base + "-color.png", r[colour][j])
                        out.image(base + "-depth.png", r["depth"][j])
                        # the scripts write a float64 0/1 array, which cv2 stores as this 8-bit image
                        out.image(base + "-label.png", r["label"][j])
                        _write_pose_txt(base + "-pose.txt", class_idx, pose[j])
    return classes


def write_gt_observed_set(lm6d_refine_root, ctx, mesh_slots, idx2class=None, K=K_LM, znear=0.25, zfar=6.0, batch=16,
                          workers=1):
    """LM6d_0_gen_gt_observed.py: for every class of idx2class (its order) and every frame of
    image_set/observed/<cls>_all.txt, the pose of data/observed/<index>-meta.mat (`poses` 3x4, or 3x4xN picked where
    `cls_indexes` is the class id) -> data/gt_observed/<cls>/<prefix>-pose.txt (header: the class id), -depth.png,
    -label.png (uint8 depth != 0) and, for the frames 000128 / 000256 / 000512, -color.png; rendered at
    quat2mat(mat2quat(R)) like the script."""
    import scipy.io as sio
    idx2class = LM6D_IDX2CLASS if idx2class is None else idx2class
    with _BatchWriter(workers) as out:
        for cls_idx, cls_name in idx2class.items():
            with open(os.path.join(lm6d_refine_root, "image_set", "observed", "{}_all.txt".format(cls_name))) as f:
                indices = [line.strip("\r\n") for line in f.readlines()]
            d = os.path.join(lm6d_refine_root, "data", "gt_observed", cls_name)
            os.makedirs(d, exist_ok=True)
            for lo in range(0, len(indices), batch):
                chunk, poses = indices[lo:lo + batch], []
                for observed_idx in chunk:
                    meta = sio.loadmat(os.path.join(lm6d_refine_root, "data", "observed", "{}-meta.mat".format(observed_idx)))
                    inner_id = np.where(np.atleast_1d(np.squeeze(meta["cls_indexes"])) == cls_idx)
                    pose = meta["poses"] if len(meta["poses"].shape) == 2 else np.squeeze(meta["poses"][:, :, inner_id])
                    poses.append(pose)
                    _write_pose_txt(os.path.join(d, "{}-pose.txt".format(observed_idx.split("/")[1])), cls_idx, pose)
                p32 = np.stack([np.hstack([quat2mat(mat2quat(p[:3, :3])), p[:, -1:]]) for p in poses]).astype(np.float32)
                r = _device_batch(ctx, mesh_slots[cls_name], p32, K, znear, zfar, ("bgr", "depth", "label"))
                for j, observed_idx in enumerate(chunk):
                    base = os.path.join(d, observed_idx.split("/")[1])
                    if any(x in observed_idx for x in GT_OBSERVED_COLOUR_FRAMES):
                        out.image(base + "-color.png", r["bgr"][j])
                    out.image(base + "-depth.png", r["depth"][j])
                    out.image(base + "-label.png", r["label"][j])


def read_train_poses(lm6d_refine_root, classes):
    """{class: [N,3,4]} gt_observed poses of image_set/observed/<cls>_train.txt, read as LM6d_ds_0's stat_poses reads them"""
    out = {}
    for cls_name in classes:
        with open(os.path.join(lm6d_refine_root, "image_set", "observed", "{}_train.txt".format(cls_name))) as f:
            prefixes = [line.strip().split("/")[1] for line in f.readlines()]
        out[cls_name] = np.stack([np.loadtxt(os.path.join(lm6d_refine_root, "data", "gt_observed", cls_name,
                                                          "{}-pose.txt".format(p)), skiprows=1) for p in prefixes])
    return out


def gen_syn_set(lm6d_refine_root, syn_root, ctx, classes, mesh_slots=None, num_images=10000, seed=2333, K=K_LM, batch=16,
                workers=None):
    """LM6d_ds_0 ... ds_4 in one call: syn_root gets poses/LM6d_ds_train_observed_pose_all.pkl, the observed and gt_observed
    images (write_syn_observed_set), one rendered pose per observed image (gen_rendered_poses, n_per_observed=1) and its
    render, and the pair lists image_set/train_<cls>.txt (write_rendered_set, syn layout).  classes: the class names, in
    the order of the scripts' idx2class; mesh_slots[class] = its mesh in ctx (default: the position in `classes`).
    workers: PNG encoder threads (default: the CPU count).  Returns the sampled poses."""
    workers = os.cpu_count() if workers is None else workers
    mesh_slots = {c: i for i, c in enumerate(classes)} if mesh_slots is None else mesh_slots
    syn = gen_syn_observed_poses(read_train_poses(lm6d_refine_root, classes), K, num_images, seed)
    os.makedirs(os.path.join(syn_root, "poses"), exist_ok=True)
    with open(os.path.join(syn_root, "poses", "LM6d_ds_train_observed_pose_all.pkl"), "wb") as f:
        pickle.dump(syn, f, 2)
    write_syn_observed_set(syn_root, ctx, syn, syn_light_draws(syn, seed), mesh_slots, K, batch=batch, workers=workers)
    for class_idx, cls_name in enumerate(sorted(syn)):
        index = ["{}/{:06d}".format(cls_name, i + 1) for i in range(len(syn[cls_name]))]
        gt = np.stack([se3_q2m(q) for q in syn[cls_name]])
        rendered = gen_rendered_poses(gt, K, n_per_observed=1, seed=seed)
        write_rendered_set(syn_root, ctx, cls_name, class_idx, mesh_slots[cls_name], index, rendered, K, set_name="train",
                           batch=batch, syn_names=True, workers=workers)
    return syn
