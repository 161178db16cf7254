"""LINEMOD (LM6d_refine) on-disk formats and a batched pred_eval driver (SURVEY 8(f) row 2).

Readers (and, for synthetic fixtures, writers) for what lib/dataset/LM6D_REFINE.py and the renderer consume:

    <root>/models/<cls>/textured.obj, texture_map.png, points.xyz        (render_py_multi.py:69-76, load_object_points.py)
    <root>/models/models_info.txt            "<cls_idx> diameter <mm> ..."                   (LM6D_REFINE.py:112-126)
    <root>/image_set/<set>.txt               "<observed index> <rendered index>" per line   (l.128-138)
    <root>/data/observed/<index>-color.png | -depth.png (uint16, metres * DEPTH_FACTOR 1000) | -label.png   (l.140-182)
    <root>/data/observed/<index>-K.txt       optional: the frame's own 3x3 intrinsics, np.loadtxt   (tester.py:424-427)
    <root>/data/gt_observed/<cls>/<idx>-pose.txt | -depth.png            (1 header line + 3x4, np.loadtxt(skiprows=1), l.184-196)
    <root>/data/rendered/<index>-color.png | -depth.png | -label.png | -pose.txt

textured.obj is un-rolled per face-vertex like glumpy.data.objload (every face corner becomes its own vertex with its
position / texcoord / normal), and the texture is flipped vertically exactly as render_py_multi.py:76 does.
`evaluate` is the B >> 1 replacement of deepim/core/tester.py:pred_eval for this dataset layout: it refines every pair
of the image set with PoseRefiner (4 iterations, device-resident) and scores ADD / ADI on the device (pose_eval)."""
from __future__ import annotations

import os

import numpy as np

from .synth import Mesh

DEPTH_FACTOR = 1000.0


def _cv2():
    import cv2  # image codecs only
    return cv2


# ------------------------------------------------------------------------------------------ models
def load_textured_obj(obj_path, texture_path=None) -> Mesh:
    """OBJ with `v`, `vt`, optional `vn`, triangular (or fan-triangulated polygon) faces `f v/vt[/vn]`."""
    v, vt, vn, corners = [], [], [], []
    with open(obj_path) as f:
        for line in f:
            t = line.split()
            if not t:
                continue
            if t[0] == "v":
                v.append([float(x) for x in t[1:4]])
            elif t[0] == "vt":
                vt.append([float(x) for x in t[1:3]])
            elif t[0] == "vn":
                vn.append([float(x) for x in t[1:4]])
            elif t[0] == "f":
                idx = []
                for c in t[1:]:
                    p = (c.split("/") + ["", ""])[:3]
                    idx.append((int(p[0]), int(p[1]) if p[1] else 0, int(p[2]) if p[2] else 0))
                for k in range(1, len(idx) - 1):  # fan
                    corners += [idx[0], idx[k], idx[k + 1]]
    v, vt, vn = np.asarray(v, np.float32), np.asarray(vt, np.float32), np.asarray(vn, np.float32)
    fix = lambda i, n: i - 1 if i > 0 else n + i  # OBJ indices are 1-based, negative = relative to the end
    pos = np.stack([v[fix(c[0], len(v))] for c in corners])
    uv = np.stack([vt[fix(c[1], len(vt))] if c[1] else np.zeros(2, np.float32) for c in corners])
    faces = np.arange(len(corners), dtype=np.int32).reshape(-1, 3)
    if texture_path is not None:
        tex = _cv2().imread(texture_path, _cv2().IMREAD_COLOR)
        if tex is None:
            raise FileNotFoundError(texture_path)
        tex = tex[::-1, :, ::-1]  # BGR -> RGB and the vertical flip of render_py_multi.py:76
    else:
        tex = np.full((2, 2, 3), 255, np.uint8)
    m = Mesh(pos, uv, faces, np.ascontiguousarray(tex), name=os.path.basename(os.path.dirname(obj_path)))
    if len(vn) and all(c[2] for c in corners):
        m.normals = np.stack([vn[fix(c[2], len(vn))] for c in corners]).astype(np.float32)
    return m


def write_textured_obj(mesh: Mesh, obj_path, texture_path):
    """Inverse of load_textured_obj for synthetic fixtures (indexed v / vt, f v/vt)."""
    os.makedirs(os.path.dirname(obj_path), exist_ok=True)
    with open(obj_path, "w") as f:
        for p in mesh.verts:
            f.write("v %.9g %.9g %.9g\n" % tuple(p))
        for t in mesh.uvs:
            f.write("vt %.9g %.9g\n" % tuple(t))
        for a, b, c in mesh.faces + 1:
            f.write("f %d/%d %d/%d %d/%d\n" % (a, a, b, b, c, c))
    _cv2().imwrite(texture_path, np.ascontiguousarray(mesh.tex[::-1, :, ::-1]))


def load_points_xyz(path):
    return np.loadtxt(path).reshape(-1, 3)


def load_models_info(path, idx2class):
    """{class name: diameter in metres} (LM6D_REFINE.py:112-126: third token, millimetres)."""
    out = {}
    with open(path) as f:
        for line in f:
            t = line.strip().split()
            if len(t) >= 3 and int(t[0]) in idx2class:
                out[idx2class[int(t[0])]] = float(t[2]) / 1000.0
    return out


# ------------------------------------------------------------------------------------------ frames
def read_pose(path):
    return np.loadtxt(path, skiprows=1).reshape(3, 4)


def write_pose(path, cls_idx, pose):
    with open(path, "w") as f:
        f.write("%d\n" % cls_idx)
        for r in np.asarray(pose).reshape(3, 4):
            f.write(" ".join("%.10g" % x for x in r) + "\n")


def read_depth_u16(path):
    """The depth file's uint16 values (metres * DEPTH_FACTOR)."""
    d = _cv2().imread(path, _cv2().IMREAD_UNCHANGED)
    if d is None:
        raise FileNotFoundError(path)
    return d


def read_depth(path):
    return read_depth_u16(path).astype(np.float32) / np.float32(DEPTH_FACTOR)


def write_depth(path, depth_m):
    _cv2().imwrite(path, np.clip(np.round(np.asarray(depth_m, np.float64) * DEPTH_FACTOR), 0, 65535).astype(np.uint16))


def read_color(path):
    im = _cv2().imread(path, _cv2().IMREAD_COLOR)  # BGR uint8, what cv2.imread hands the reference's loader
    if im is None:
        raise FileNotFoundError(path)
    return im


def read_label(path):
    return _cv2().imread(path, _cv2().IMREAD_UNCHANGED)


class LM6DRefine:
    def __init__(self, root, classes, image_set, idx2class=None):
        self.root, self.classes, self.image_set = root, list(classes), image_set
        self.idx2class = idx2class or {i + 1: c for i, c in enumerate(self.classes)}
        self.models_dir = os.path.join(root, "models")
        self.diameters = load_models_info(os.path.join(self.models_dir, "models_info.txt"), self.idx2class)

    def mesh(self, cls):
        d = os.path.join(self.models_dir, cls)
        return load_textured_obj(os.path.join(d, "textured.obj"), os.path.join(d, "texture_map.png"))

    def points(self, cls):
        return load_points_xyz(os.path.join(self.models_dir, cls, "points.xyz"))

    def pairs(self, cls):
        """[(observed index, rendered index)] of `<image_set>_<cls>.txt` (one set file per class as the reference's
        `PoseCNN_val_<cls>` sets)."""
        path = os.path.join(self.root, "image_set", "%s_%s.txt" % (self.image_set, cls))
        with open(path) as f:
            return [tuple(x.strip().split(" ")) for x in f if x.strip()]

    def load_pair(self, cls, pair):
        """What load_render_annotation + the test loader read for one pair (LM6D_REFINE.py:226-262, image.py:297-399), and
        "K" (3x3 float64) from `data/observed/<observed index>-K.txt` where that file exists (tester.py:424-427); a pair
        without one has no "K" and is taken with the dataset's K."""
        obs, ren = pair
        d = os.path.join(self.root, "data")
        rec = {
            "image_observed": read_color(os.path.join(d, "observed", obs + "-color.png")),
            "pose_observed": read_pose(os.path.join(d, "gt_observed", cls, obs.split("/")[1] + "-pose.txt")),
            "pose_rendered": read_pose(os.path.join(d, "rendered", ren + "-pose.txt")),
            "depth_rendered": read_depth(os.path.join(d, "rendered", ren + "-depth.png")),
        }
        k_path = os.path.join(d, "observed", obs + "-K.txt")
        if os.path.exists(k_path):
            rec["K"] = np.loadtxt(k_path).reshape(3, 3)
        return rec


def evaluate(dataset: LM6DRefine, weights, K, symmetric=("eggbox", "glue", "bowl", "cup"), n_iter=4, max_batch=16, device=0,
             precision="fp16", input_depth=False, input_mask=True, icp_iters=0, vsd=False):
    """Batched pred_eval (deepim/core/tester.py:50-527 without its batch = 1 limit): refine every pair of the image set
    and score it the way the reference's dataset class does: ADD / ADI accuracy + AUC (evaluate_pose_add), 5 cm 5 deg
    (evaluate_pose) and Proj. 2D (evaluate_pose_arp_2d); the last two under res["rot_trans"] / res["arp_2d"].
    input_depth=True refines with the RGB-D network (weights with a (64, 10, 7, 7) flow_conv1) and reads each observed frame's
    `-depth.png` as well (image.py:190-219; converted on the device with DEPTH_FACTOR).
    input_mask=False refines with the image-only network (weights with a (64, 6, 7, 7) flow_conv1; ZoomImage).
    A pair whose observed frame has a `-K.txt` (load_pair) is refined with that camera, for the render and the zoom, and the
    other pairs with K, in one set of batches (PoseRefiner.refine with a K per instance).  Proj. 2D projects with K for every
    pair, as the reference's evaluate_pose_arp_2d does with config.dataset.INTRINSIC_MATRIX (LM6D_REFINE.py:526).
    icp_iters > 0 polishes the last refined poses against each pair's observed `-depth.png` with PoseRefiner.icp (icp_iters
    iterations at its default max_dist / min_points, each pair with its own `-K.txt` camera where it has one) and scores
    the result as one more row, the "+ ICP" row of the reference's evaluation (TEST.PRECOMPUTED_ICP): poses_est and every
    table then have n_iter + 1 rows, the last one after ICP.  With icp_iters = 0 nothing changes.
    vsd=True also scores every row (each iteration, and the ICP row) with the Visible Surface Discrepancy against each
    pair's observed `-depth.png` (PoseRefiner.vsd, each pair with its own `-K.txt` camera where it has one, because the
    depth belongs to that camera), with the values of Hodan et al. and the SIXD Challenge 2017: delta 15 mm, tau 20 mm,
    recall at e < 0.3.  res["vsd"] holds evaluate_pose_vsd's per-class and mean recall per row and the errors [rows,M].
    With vsd=False the result is unchanged.
    Returns (evaluate_pose_add result + the two extra tables, poses_est [n_iter,M,3,4], poses_gt)."""
    from . import pose_eval
    from .refiner import PoseRefiner
    meshes = [dataset.mesh(c) for c in dataset.classes]
    ref = PoseRefiner(meshes, weights, K=K, device=device, max_batch=max_batch, n_iter=n_iter, precision=precision,
                      input_depth=input_depth, depth_factor=DEPTH_FACTOR, input_mask=input_mask)
    imgs, cls_idx, init, gt, depths, Ks = [], [], [], [], [], []
    for ci, c in enumerate(dataset.classes):
        for pair in dataset.pairs(c):
            rec = dataset.load_pair(c, pair)
            Ks.append(rec.get("K"))
            imgs.append(rec["image_observed"])
            cls_idx.append(ci)
            init.append(rec["pose_rendered"])
            gt.append(rec["pose_observed"])
            if input_depth or icp_iters > 0 or vsd:
                depths.append(read_depth_u16(os.path.join(dataset.root, "data", "observed", pair[0] + "-depth.png")))
    imgs, cls_idx = np.stack(imgs), np.asarray(cls_idx, np.int32)
    init, gt = np.stack(init).astype(np.float64), np.stack(gt).astype(np.float64)
    K_pairs = None  # one camera for every pair unless some pair has its own
    if any(k is not None for k in Ks):
        K_pairs = np.stack([np.asarray(K if k is None else k, np.float32).reshape(3, 3) for k in Ks])
    depths = np.stack(depths).astype(np.uint16) if depths else None
    poses = ref.refine(imgs, cls_idx, init, depths_u16=depths if input_depth else None, K=K_pairs)
    if icp_iters > 0:
        polished = ref.icp(depths, cls_idx, poses[-1], K_frames=K_pairs, n_iter=icp_iters)["poses"][-1]
        poses = np.concatenate([poses, polished[None]])
    res = pose_eval.evaluate_pose_add(ref.ctx, poses, gt, cls_idx, [dataset.points(c) for c in dataset.classes],
                                      [dataset.diameters[c] for c in dataset.classes], [c in symmetric for c in dataset.classes])
    pts_all = [dataset.points(c) for c in dataset.classes]
    if vsd:
        errs = np.stack([ref.vsd(depths, cls_idx, p, gt, K_frames=K_pairs, delta=0.015, taus=(0.02,))["err"][:, 0]
                         for p in poses])
        res["vsd"] = dict(pose_eval.evaluate_pose_vsd(errs, cls_idx, len(dataset.classes), 0.3), errors=errs)
    res["rot_trans"] = pose_eval.evaluate_pose(ref.ctx, poses, gt, cls_idx, pts_all, K, class_names=list(dataset.classes))
    res["arp_2d"] = pose_eval.evaluate_pose_arp_2d(ref.ctx, poses, gt, cls_idx, pts_all, K, class_names=list(dataset.classes))
    ref.close()
    return res, poses, gt
