"""Writes tests/golden/ref_syn.npz: what the reference's data-preparation scripts do on a fabricated LM6d_refine tree.

Runs the UNMODIFIED scripts toolkit/LM6d_0_gen_gt_observed.py and LM6d_ds_0 ... ds_4 of a checkout of the reference
(mx-DeepIM) with runpy.  The scripts take their data root from abspath(dirname(__file__))/.., so a temporary directory
gets a toolkit/ of symlinks to the scripts and a lib symlink next to it.  glumpy, the two glumpy renderers and
matplotlib.pyplot are replaced in sys.modules by stubs that record every render call (quaternion or matrix, translation,
the live quat2mat of the quaternion, light position / intensity, brightness_k) and return black images, so the scripts'
own cv2.imwrite calls, pose files and lists are written as usual.  The ds_0 pickle is cut to SYN_KEEP images per class
before ds_1 runs (data, not sources).

    python tests/golden/make_golden_syn.py <path of the mx-DeepIM checkout>
"""
import hashlib
import os
import pickle
import runpy
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = sys.argv[1] if len(sys.argv) > 1 else None
IDX2CLASS = {1: "ape", 2: "benchvise", 4: "camera", 5: "can", 6: "cat", 8: "driller", 9: "duck", 10: "eggbox", 11: "glue",
             12: "holepuncher", 13: "iron", 14: "lamp", 15: "phone"}
FRAMES = ["%06d" % i for i in list(range(1, 11)) + [128, 256]]
SYN_KEEP = 8     # ds_0 images per class kept for ds_1 ... ds_4
POSES_KEPT = 300  # ds_0 poses per class stored in the fixture (plus the hash of all of them)
CALLS = {}


def _rot(rs):
    q = rs.normal(0, 1, 4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _stubs():
    from lib.pair_matching.RT_transform import quat2mat  # the live function, after sys.path points at the reference

    black = (np.zeros((480, 640, 3), np.uint8), np.zeros((480, 640), np.float32))

    class Render_Py:
        def __init__(self, *a, **k):
            pass

        def render(self, r, t, r_type="quat", K=None):
            r = np.asarray(r, np.float64)
            CALLS.setdefault(CURRENT, []).append({"r": r, "t": np.asarray(t, np.float64).reshape(3),
                                                  "R": quat2mat(r) if r_type == "quat" else r})
            return black[0].astype(np.float32), black[1].copy()

    class Render_Py_Light:
        def __init__(self, *a, **k):
            pass

        def render(self, r, t, light_position, light_intensity, brightness_k=0, r_type="quat", K=None):
            r = np.asarray(r, np.float64)
            CALLS.setdefault(CURRENT, []).append({
                "r": r, "t": np.asarray(t, np.float64).reshape(3), "R": quat2mat(r) if r_type == "quat" else r,
                "light_position": np.asarray(light_position, np.float64), "light_intensity": np.asarray(light_intensity,
                                                                                                        np.float64),
                "brightness_k": brightness_k})
            return black[0].copy(), black[1].copy()

    m1 = types.ModuleType("lib.render_glumpy.render_py")
    m1.Render_Py = Render_Py
    m2 = types.ModuleType("lib.render_glumpy.render_py_light")
    m2.Render_Py_Light = Render_Py_Light
    sys.modules["lib.render_glumpy.render_py"] = m1
    sys.modules["lib.render_glumpy.render_py_light"] = m2


def _fabricate(lm):
    import cv2
    import scipy.io as sio
    rs = np.random.RandomState(5)
    inputs = {}
    os.makedirs(os.path.join(lm, "image_set", "observed"), exist_ok=True)
    for cls_idx, cls in IDX2CLASS.items():
        video = "%02d" % cls_idx
        os.makedirs(os.path.join(lm, "data", "observed", video), exist_ok=True)
        index = ["%s/%s" % (video, p) for p in FRAMES]
        for name in ("train", "all"):
            with open(os.path.join(lm, "image_set", "observed", "%s_%s.txt" % (cls, name)), "w") as f:
                f.write("".join(x + "\n" for x in index))
        poses = []
        for k, idx in enumerate(index):
            pose = np.hstack([_rot(rs), np.array([[rs.normal(0, 0.03)], [rs.normal(0, 0.03)], [0.9 + rs.normal(0, 0.08)]])])
            poses.append(pose)
            if k % 2:  # a frame with two objects: poses 3x4x2 picked by cls_indexes
                other = np.hstack([_rot(rs), np.array([[0.1], [0.0], [1.0]])])
                meta = {"cls_indexes": np.array([[99], [cls_idx]], np.float64), "poses": np.stack([other, pose], 2)}
            else:
                # numpy 2 refuses np.where on the 0-d squeeze of a 1x1 cls_indexes, so a second (unused) id pads it
                meta = {"cls_indexes": np.array([[cls_idx], [0]], np.float64), "poses": pose}
            sio.savemat(os.path.join(lm, "data", "observed", idx + "-meta.mat"), meta)
            cv2.imwrite(os.path.join(lm, "data", "observed", idx + "-color.png"), np.zeros((480, 640, 3), np.uint8))
        inputs[cls] = np.stack(poses)
    return inputs


def _run(root, script):
    global CURRENT
    CURRENT = script
    runpy.run_path(os.path.join(root, "toolkit", script), run_name="__main__")


def main():
    if REF is None or not os.path.isdir(os.path.join(REF, "toolkit")):
        sys.exit(__doc__)
    tmp = tempfile.mkdtemp(prefix="syn_golden_")
    os.makedirs(os.path.join(tmp, "toolkit"))
    scripts = ["LM6d_0_gen_gt_observed.py", "LM6d_ds_0_gen_observed_poses.py", "LM6d_ds_1_gen_observed.py",
               "LM6d_ds_2_gen_gt_observed.py", "LM6d_ds_3_gen_rendered_pose.py", "LM6d_ds_4_gen_rendered.py"]
    for s in scripts:
        os.symlink(os.path.join(REF, "toolkit", s), os.path.join(tmp, "toolkit", s))
    os.symlink(os.path.join(REF, "lib"), os.path.join(tmp, "lib"))
    sys.path.insert(0, tmp)
    # numpy-2 shim (RT_transform.py:236-237 uses np.float / np.maximum_sctype at import time; LM6d_0 np.int)
    np.float, np.int = float, int
    np.maximum_sctype = lambda t: np.float64
    sys.modules["glumpy"] = types.ModuleType("glumpy")
    sys.modules["matplotlib"] = types.ModuleType("matplotlib")
    sys.modules["matplotlib.pyplot"] = types.ModuleType("matplotlib.pyplot")
    sys.modules["termcolor"] = types.ModuleType("termcolor")  # lib.utils.logger, imported by the dataset classes
    sys.modules["termcolor"].colored = lambda s, *a, **k: s
    _stubs()
    conv = os.path.join(tmp, "data", "LINEMOD_6D", "LM6d_converted")
    lm, syn = os.path.join(conv, "LM6d_refine"), os.path.join(conv, "LM6d_refine_syn")
    inputs = _fabricate(lm)

    _run(tmp, scripts[0])
    _run(tmp, scripts[1])
    pkl = os.path.join(syn, "poses", "LM6d_ds_train_observed_pose_all.pkl")
    with open(pkl, "rb") as f:
        poses_all = pickle.load(f)
    h = hashlib.sha256()
    for c in sorted(poses_all):
        h.update(np.ascontiguousarray(poses_all[c], np.float64).tobytes())
    with open(pkl, "wb") as f:
        pickle.dump({c: v[:SYN_KEEP] for c, v in poses_all.items()}, f, 2)
    for s in scripts[2:]:
        _run(tmp, s)

    rec = {"classes": np.array(sorted(IDX2CLASS.values())), "idx2class_ids": np.array(list(IDX2CLASS)),
           "idx2class_names": np.array(list(IDX2CLASS.values())), "syn_keep": SYN_KEEP,
           "syn_sha256": np.array(h.hexdigest()), "num_images": len(next(iter(poses_all.values())))}
    for c, v in inputs.items():
        rec["input_pose/" + c] = v
    for c, v in poses_all.items():
        rec["syn_pose/" + c] = v[:POSES_KEPT]
    for s, calls in CALLS.items():
        tag = s.split("_gen")[0]
        for key in calls[0]:
            rec["call/%s/%s" % (tag, key)] = np.array([c[key] for c in calls])
    files = []
    for d, _, fs in os.walk(os.path.join(tmp, "data")):
        files += [os.path.relpath(os.path.join(d, f), conv) for f in fs]
    files = sorted(f for f in files if not f.startswith("LM6d_refine/data/observed/"))  # the fabricated input
    rec["files"] = np.array(files)
    texts = [f for f in files if f.endswith(".txt") and "/rendered_poses/" not in f]
    rec["text_names"] = np.array(texts)
    rec["text_values"] = np.array([open(os.path.join(conv, f)).read() for f in texts])

    # what the live dataset class resolves for each pair of the syn training lists
    from lib.dataset.LM6D_REFINE_SYN import LM6D_REFINE_SYN
    res = []
    for c in sorted(IDX2CLASS.values()):
        ds = LM6D_REFINE_SYN(None, "train_%s" % c, tmp, lm, c, result_path=os.path.join(tmp, "cache"))
        for pair in ds.image_set_index:
            r = ds.load_render_annotation(pair)
            res += [os.path.relpath(r[k], conv) for k in ("image_observed", "image_gt_observed", "image_rendered",
                                                          "depth_observed", "depth_gt_observed", "depth_rendered",
                                                          "mask_gt_observed")]
    rec["annotation_paths"] = np.array(sorted(set(res)))
    np.savez_compressed(os.path.join(HERE, "ref_syn.npz"), **rec)
    print("wrote ref_syn.npz: %d files, %d render calls, sha256 %s" % (len(files), sum(map(len, CALLS.values())),
                                                                     h.hexdigest()))


if __name__ == "__main__":
    main()
