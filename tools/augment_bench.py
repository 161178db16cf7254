"""Train-time augmentation cost per batch: background replacement + observed-mask dilation on the device
(dim_replace_background + dim_mask_dilate, CUDA events over many batches) against the reference's host path on the same
inputs, one instance after the other on one core (image.py:108-157: crop, cv2.resize INTER_LINEAR, composite, transform;
mask_dilate.py).  Prints one JSON line with the card's name and power limit.

    python tools/augment_bench.py [--iters 200] [--out augment_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "mx-deepim_b200"))
from deepim_b200 import augment  # noqa: E402
from deepim_b200.context import Context  # noqa: E402

H, W = 480, 640
MEANS_RGB = (123.68, 116.779, 103.939)
MEANS_BGR = MEANS_RGB[::-1]
PHOTO_SHAPES = [(375, 500), (500, 333), (333, 500), (500, 375), (400, 400), (281, 500), (500, 400), (375, 500)]  # VOC-like


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:  # the numbers are still device times; say what could not be read
        return torch.cuda.get_device_name(0), "unknown (%s)" % type(e).__name__


def host_instance(cv2, obs_u8, mask_gt, mask_obs, photo, draws):
    """the reference's per-instance host work, restated: crop + resize + composite + transform + dilation"""
    bh, bw = photo.shape[:2]
    ch, cw, dh, dw, fx = augment.background_geometry(H, W, bh, bw)
    r = cv2.resize(photo[:ch, :cw], None, None, fx=fx, fy=fx, interpolation=cv2.INTER_LINEAR)
    res = np.zeros((H, W, 3), np.uint8)
    res[:r.shape[0], :r.shape[1]] = r
    fg = np.dstack([mask_gt] * 3) != 0
    res[fg] = obs_u8[fg]
    t = np.zeros((1, 3, H, W))
    for i in range(3):
        t[0, i] = res[:, :, 2 - i] - MEANS_BGR[2 - i]
    m = mask_obs.astype(np.float64)  # the reference's mask_observed is float64
    out = m.copy()
    td, tu, tr, tl = draws[1:]
    if td:
        out[td:] += np.logical_and(m[:-td] != 0, m[td:] == 0)
    if tu:
        out[:-tu] += np.logical_and(m[tu:] != 0, m[:-tu] == 0)
    if tr:
        out[:, tr:] += np.logical_and(m[:, :-tr] != 0, m[:, tr:] == 0)
    if tl:
        out[:, :-tl] += np.logical_and(m[:, tl:] != 0, m[:, :-tl] == 0)
    out[out > 1] = 1
    return t.astype(np.float32), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--host-iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("augment_bench needs a CUDA device: there is no CPU measurement of the device path")
    rng = np.random.default_rng(0)
    photos = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in PHOTO_SHAPES]
    ctx = Context(0, max_batch=16, max_classes=1, max_verts=100, max_faces=100)
    bank = augment.BackgroundBank(ctx, photos)
    name, power = card()
    res = {"metric": "augment_ms_per_batch", "gpu": name, "power_limit": power, "iters": a.iters, "batches": {}}
    yy, xx = np.mgrid[0:H, 0:W]
    for B in (4, 16):
        obs_u8 = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
        mask_gt = np.stack([(((yy - 240) / (80 + 5 * b)) ** 2 + ((xx - 320) / 120.0) ** 2 < 1) for b in range(B)]).astype(np.uint8)
        mask_obs = np.zeros((B, H, W), np.float32)
        mask_obs[:, 150:330, 190:450] = 1
        idx = augment.background_draws(B, np.random.RandomState(B), len(bank))
        draws = augment.mask_dilate_draws(B, np.random.RandomState(B))
        d_obs = torch.from_numpy(obs_u8.astype(np.float32)).cuda()
        d_mgt = torch.from_numpy(mask_gt.astype(np.float32)[:, None]).cuda()
        d_mo = torch.from_numpy(mask_obs[:, None]).cuda()
        d_draws = torch.from_numpy(draws).cuda()
        for _ in range(10):  # warm-up
            ctx.replace_background(d_obs, d_mgt, idx, MEANS_RGB)
            ctx.mask_dilate(d_mo, d_draws)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            ctx.replace_background(d_obs, d_mgt, idx, MEANS_RGB)
            ctx.mask_dilate(d_mo, d_draws)
        e1.record()
        torch.cuda.synchronize()
        dev_ms = e0.elapsed_time(e1) / a.iters
        row = {"device_ms": round(dev_ms, 4)}
        try:
            import cv2
            cv2.setNumThreads(1)
            t0 = time.perf_counter()
            for _ in range(a.host_iters):
                for b in range(B):
                    host_instance(cv2, obs_u8[b], mask_gt[b], mask_obs[b], photos[idx[b]], draws[b])
            host_ms = (time.perf_counter() - t0) * 1e3 / a.host_iters
            row.update(host_ms_one_core=round(host_ms, 2), speedup=round(host_ms / dev_ms, 1))
        except ImportError:
            row["host_ms_one_core"] = "not measured (cv2 missing)"
        res["batches"][str(B)] = row
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
