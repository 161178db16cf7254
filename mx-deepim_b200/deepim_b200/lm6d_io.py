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


# PLY scalar types and their aliases -> little-endian numpy dtypes
_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "<i2", "int16": "<i2", "ushort": "<u2",
              "uint16": "<u2", "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4", "float": "<f4",
              "float32": "<f4", "double": "<f8", "float64": "<f8"}


def _ply_type(t):
    if t not in _PLY_TYPES:
        raise ValueError("PLY: unknown property type %r" % t)
    return np.dtype(_PLY_TYPES[t])


def _ply_header(data):
    """format, comments and elements [(name, count, [(prop, dtype) or (prop, count dtype, item dtype)])], data offset"""
    end = data.find(b"end_header")
    if not data.startswith(b"ply") or end < 0:
        raise ValueError("PLY: not a PLY file")
    body = data.index(b"\n", end) + 1
    fmt, comments, elements = None, [], []
    for line in data[:end].decode("ascii", "replace").splitlines()[1:]:
        t = line.split()
        if not t:
            continue
        if t[0] == "format":
            fmt = " ".join(t[1:])
        elif t[0] == "comment":
            comments.append(t[1:])
        elif t[0] == "element":
            elements.append((t[1], int(t[2]), []))
        elif t[0] == "property" and elements:
            if t[1] == "list":
                elements[-1][2].append((t[4], _ply_type(t[2]), _ply_type(t[3])))
            else:
                elements[-1][2].append((t[2], _ply_type(t[1])))
    if fmt not in ("ascii 1.0", "binary_little_endian 1.0"):
        raise ValueError("PLY: format %r is not supported (ascii 1.0 and binary_little_endian 1.0 are)" % fmt)
    return fmt == "ascii 1.0", comments, elements, body


def _ply_binary_element(data, pos, count, props):
    """one element of a binary file -> ({scalar prop: [count] array, list prop: [count] list of arrays}, next offset)"""
    if all(len(p) == 2 for p in props):  # fixed-size rows
        dt = np.dtype([(n, t) for n, t in props])
        if pos + dt.itemsize * count > len(data):
            raise ValueError("PLY: file ends inside an element")
        rows = np.frombuffer(data, dt, count, pos)
        return {n: rows[n] for n, _ in props}, pos + dt.itemsize * count
    out = {p[0]: [] for p in props}
    for _ in range(count):
        for p in props:
            if len(p) == 2:
                out[p[0]].append(np.frombuffer(data, p[1], 1, pos)[0])
                pos += p[1].itemsize
            else:
                n = int(np.frombuffer(data, p[1], 1, pos)[0])
                pos += p[1].itemsize
                out[p[0]].append(np.frombuffer(data, p[2], n, pos))
                pos += p[2].itemsize * n
    return {k: (np.array(v) if len(p) == 2 else v) for (k, v), p in zip(out.items(), props)}, pos


def _ply_ascii_element(tokens, pos, count, props):
    out = {p[0]: [] for p in props}
    for _ in range(count):
        for p in props:
            if len(p) == 2:
                out[p[0]].append(tokens[pos])
                pos += 1
            else:
                n = int(tokens[pos])
                out[p[0]].append(np.array(tokens[pos + 1:pos + 1 + n], np.float64).astype(p[2]))
                pos += 1 + n
    return {k: (np.array(v, np.float64).astype(p[1]) if len(p) == 2 else v) for (k, v), p in zip(out.items(), props)}, pos


def load_ply(path, scale=1.0) -> Mesh:
    """A triangle mesh from a PLY file (ascii 1.0 or binary_little_endian 1.0): LINEMOD's obj_xx.ply and BOP's
    models/obj_NNNNNN.ply.  Vertex properties x y z (required), nx ny nz (-> mesh.normals), red green blue (alpha is
    ignored), texture_u texture_v with a `comment TextureFile <file>`; faces from the `vertex_indices` or `vertex_index`
    list of the face element; every other element is skipped.  Positions are float32(float64(x) * scale) (BOP's
    millimetres load with scale=1e-3).  The colour source:
      - a model that names a texture and has UVs: a textured Mesh, the image flipped as load_textured_obj flips it;
      - else per-vertex colours: uchar channels c -> float32(c) / float32(255), float channels as they are (the property
        type decides, unlike the SIXD renderer's "divide by 255 if max > 1", so a dark uchar model is not misread);
      - a model without colours is drawn in the SIXD renderer's 0.5 grey.
    ValueError for big-endian or unknown formats, missing x y z, faces that are not triangles, face indices out of
    range and a texture file that does not exist."""
    with open(path, "rb") as f:
        data = f.read()
    ascii_, comments, elements, pos = _ply_header(data)
    tokens = data[pos:].split() if ascii_ else None
    if ascii_:
        pos = 0
    got = {}
    for name, count, props in elements:
        if ascii_:
            vals, pos = _ply_ascii_element(tokens, pos, count, props)
        else:
            vals, pos = _ply_binary_element(data, pos, count, props)
        got[name] = (vals, {p[0]: p for p in props})
    if "vertex" not in got or not {"x", "y", "z"} <= set(got["vertex"][0]):
        raise ValueError("PLY %s: the vertex element has no x y z" % path)
    vert, vprops = got["vertex"]
    V = len(vert["x"])
    pts = (np.stack([vert[k] for k in "xyz"], 1).astype(np.float64) * float(scale)).astype(np.float32)
    fvals, fprops = got.get("face", ({}, {}))
    key = "vertex_indices" if "vertex_indices" in fvals else "vertex_index"
    if key not in fvals or len(fprops[key]) != 3:
        raise ValueError("PLY %s: no face list vertex_indices / vertex_index" % path)
    lists = fvals[key]
    bad = [i for i, l in enumerate(lists) if len(l) != 3]
    if bad:
        raise ValueError("PLY %s: face %d has %d corners; only triangles are supported" % (path, bad[0], len(lists[bad[0]])))
    faces = np.array(lists, np.int64).reshape(-1, 3)
    if faces.size and (faces.min() < 0 or faces.max() >= V):
        raise ValueError("PLY %s: a face index lies outside [0, %d)" % (path, V))
    faces = faces.astype(np.int32)
    name = os.path.splitext(os.path.basename(path))[0]
    tex_file = [c[1] for c in comments if len(c) >= 2 and c[0] == "TextureFile"]
    if tex_file and {"texture_u", "texture_v"} <= set(vert):
        tex_path = os.path.join(os.path.dirname(os.path.abspath(path)), tex_file[0])
        tex = _cv2().imread(tex_path, _cv2().IMREAD_COLOR) if os.path.exists(tex_path) else None
        if tex is None:
            raise ValueError("PLY %s: texture file %s cannot be read" % (path, tex_path))
        uv = np.stack([vert["texture_u"], vert["texture_v"]], 1).astype(np.float32)
        m = Mesh(pts, uv, faces, np.ascontiguousarray(tex[::-1, :, ::-1]), name=name)
    elif {"red", "green", "blue"} <= set(vert):
        cols = []
        for k in ("red", "green", "blue"):
            t = vprops[k][1]
            if t == np.uint8:
                cols.append(vert[k].astype(np.float32) / np.float32(255))
            elif t.kind == "f":
                cols.append(vert[k].astype(np.float32))
            else:
                raise ValueError("PLY %s: colour property %s of type %s (uchar or float expected)" % (path, k, t))
        m = Mesh(pts, None, faces, None, name=name, colours=np.stack(cols, 1))
    else:
        m = Mesh(pts, None, faces, None, name=name, colours=np.full((V, 3), 0.5, np.float32))
    if {"nx", "ny", "nz"} <= set(vert):
        m.normals = np.stack([vert[k] for k in ("nx", "ny", "nz")], 1).astype(np.float32)
    return m


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
             precision="fp16", input_depth=False, input_mask=True, icp_iters=0, vsd=False, bop=False, models_info_json=None):
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
    bop=True also scores every row with BOP 2019's average recall (pose_eval.evaluate_bop19) into res["bop"], with the
    per-instance errors under res["bop"]["errors"] ("vsd" [rows,M,10], "mssd" and "mspd" [rows,M]): the BOP 2019 VSD
    against each pair's observed `-depth.png` (delta 15 mm, taus relative to the class's diameter from models_info.txt), and
    MSSD / MSPD over each class's symmetries, each pair projected with its own `-K.txt` camera where it has one.  The
    symmetries come from BOP's `models_info.json` (models_info_json; object ids are the dataset's LINEMOD ids, idx2class);
    without it every class has only the identity.  The model points are each class's points.xyz, not BOP's evaluation
    models, so these are not the official BOP numbers.  With bop=False the result is unchanged.
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
            if input_depth or icp_iters > 0 or vsd or bop:
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
    if bop:
        res["bop"] = _evaluate_bop19(dataset, ref, poses, gt, cls_idx, depths, K, K_pairs, pts_all, models_info_json)
    res["rot_trans"] = pose_eval.evaluate_pose(ref.ctx, poses, gt, cls_idx, pts_all, K, class_names=list(dataset.classes))
    res["arp_2d"] = pose_eval.evaluate_pose_arp_2d(ref.ctx, poses, gt, cls_idx, pts_all, K, class_names=list(dataset.classes))
    ref.close()
    return res, poses, gt


def _evaluate_bop19(dataset, ref, poses, gt, cls_idx, depths, K, K_pairs, pts_all, models_info_json):
    """evaluate(bop=True)'s table: BOP 2019 VSD, MSSD and MSPD of every row and their average recall"""
    from . import bop, pose_eval
    info = {} if models_info_json is None else bop.load_models_info_json(models_info_json)
    class2id = {c: i for i, c in dataset.idx2class.items()}
    syms = [bop.symmetry_transforms(info.get(class2id.get(c), {})) for c in dataset.classes]
    diam_cls = np.array([dataset.diameters[c] for c in dataset.classes])
    K_inst = np.broadcast_to(np.asarray(K, np.float32).reshape(3, 3), (len(cls_idx), 3, 3)) if K_pairs is None else K_pairs
    vsd_err, mssd, mspd = [], [], []
    for p in poses:
        vsd_err.append(ref.vsd(depths, cls_idx, p, gt, K_frames=K_pairs, delta=pose_eval.BOP19_VSD_DELTA,
                               taus=pose_eval.BOP19_VSD_TAUS, visib_mode="bop19", diameters=diam_cls[cls_idx])["err"])
        e = ref.pose_error_sym(cls_idx, p, gt, pts_all, syms, K_inst)["err"]
        mssd.append(e[:, 0])
        mspd.append(e[:, 1])
    errors = {"vsd": np.stack(vsd_err), "mssd": np.stack(mssd), "mspd": np.stack(mspd)}
    res = pose_eval.evaluate_bop19(errors["vsd"], errors["mssd"], errors["mspd"], cls_idx, len(dataset.classes), diam_cls,
                                   ref.ctx.W)
    return dict(res, errors=errors)
