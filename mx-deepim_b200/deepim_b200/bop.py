"""BOP 2019 files and symmetries (Hodan et al., "BOP: Benchmark for 6D Object Pose Estimation", ECCV 2018, and the BOP
Challenge 2019 rules): `models_info.json`, the symmetry transforms MSSD / MSPD minimise over, and the results CSV.

Units: the BOP files are in millimetres; everything returned here is in metres, the unit of the rest of this package.

symmetry_transforms follows the published BOP toolkit's get_symmetry_transformations (continuous symmetries discretised into
ceil(pi / max_sym_disc_step) rotations, each combined with every discrete one).  Parity with that toolkit is not pinned by a
fixture; the tests hold the function to its stated contract."""
from __future__ import annotations

import csv
import json
import math

import numpy as np

RESULTS_HEADER = ("scene_id", "im_id", "obj_id", "score", "R", "t", "time")


def load_models_info_json(path):
    """BOP `models_info.json` -> {obj_id: {"diameter": metres, "syms": {"symmetries_discrete": [[4,4] float64 with the
    translation in metres], "symmetries_continuous": [{"axis": [3], "offset": [3] metres}]}}}"""
    with open(path) as f:
        raw = json.load(f)
    out = {}
    for k, v in raw.items():
        disc = []
        for m in v.get("symmetries_discrete", []):
            T = np.asarray(m, np.float64).reshape(4, 4).copy()
            T[:3, 3] /= 1000.0
            disc.append(T)
        cont = [{"axis": np.asarray(c["axis"], np.float64).reshape(3),
                 "offset": np.asarray(c.get("offset", [0.0, 0.0, 0.0]), np.float64).reshape(3) / 1000.0}
                for c in v.get("symmetries_continuous", [])]
        out[int(k)] = {"diameter": float(v["diameter"]) / 1000.0,
                       "syms": {"symmetries_discrete": disc, "symmetries_continuous": cont}}
    return out


def rotation_about(axis, angle):
    """[3,3] rotation by `angle` (radians) about `axis` (normalised here), Rodrigues' formula"""
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    c, s = math.cos(angle), math.sin(angle)
    cross = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return c * np.eye(3) + s * cross + (1.0 - c) * np.outer(a, a)


def symmetry_transforms(info, max_sym_disc_step=0.01):
    """f64 [S,3,4] symmetry transforms of one object, the identity at row 0.  info: an entry of load_models_info_json (or
    its "syms" dict); without symmetries S = 1.
    Each continuous symmetry becomes n = ceil(pi / max_sym_disc_step) rotations R_k by 2 pi k / n about its axis with
    t_k = -R_k offset + offset, k = 1 .. n - 1 (k = 0 is the identity).  Every discrete transform D (the identity first) is
    combined with every continuous one C (the identity first): R = R_C R_D, t = R_C t_D + t_C."""
    syms = info.get("syms", info)
    disc = [(np.eye(3), np.zeros(3))]
    disc += [(np.asarray(T, np.float64)[:3, :3], np.asarray(T, np.float64)[:3, 3]) for T in syms.get("symmetries_discrete", [])]
    cont = [(np.eye(3), np.zeros(3))]
    for c in syms.get("symmetries_continuous", []):
        n = int(math.ceil(math.pi / max_sym_disc_step))
        off = np.asarray(c["offset"], np.float64).reshape(3)
        for k in range(1, n):
            R = rotation_about(c["axis"], 2.0 * math.pi * k / n)
            cont.append((R, -R @ off + off))
    out = np.empty((len(disc) * len(cont), 3, 4))
    i = 0
    for Rd, td in disc:
        for Rc, tc in cont:
            out[i, :, :3] = Rc @ Rd
            out[i, :, 3] = Rc @ td + tc
            i += 1
    return out


def write_results_csv(path, rows):
    """BOP 2019 results file: rows of dicts with scene_id, im_id, obj_id, score, R [3,3], t [3] metres and optionally time
    (seconds; -1 = not measured).  R is written as 9 space-separated values, row-major; t in millimetres."""
    with open(path, "w", newline="") as f:
        w = csv.writer(f, lineterminator="\n")
        w.writerow(RESULTS_HEADER)
        for r in rows:
            R = np.asarray(r["R"], np.float64).reshape(9)
            t = np.asarray(r["t"], np.float64).reshape(3) * 1000.0
            w.writerow([int(r["scene_id"]), int(r["im_id"]), int(r["obj_id"]), repr(float(r["score"])),
                        " ".join(repr(float(x)) for x in R), " ".join(repr(float(x)) for x in t),
                        repr(float(r.get("time", -1.0)))])


def read_results_csv(path):
    """write_results_csv's inverse: a list of dicts with R [3,3] float64 and t [3] metres"""
    out = []
    with open(path, newline="") as f:
        rd = csv.reader(f)
        if tuple(next(rd)) != RESULTS_HEADER:
            raise ValueError("%s: not a BOP 2019 results file (header %s expected)" % (path, ",".join(RESULTS_HEADER)))
        for row in rd:
            if not row:
                continue
            out.append({"scene_id": int(row[0]), "im_id": int(row[1]), "obj_id": int(row[2]), "score": float(row[3]),
                        "R": np.array([float(x) for x in row[4].split()]).reshape(3, 3),
                        "t": np.array([float(x) for x in row[5].split()]) / 1000.0, "time": float(row[6])})
    return out
