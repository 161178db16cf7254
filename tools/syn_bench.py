"""Data-preparation renders on the GPU: dim_render_dataset per batch, and toolkit.gen_syn_set end to end.

    python tools/syn_bench.py [--batches 300] [--images 400] [--threads N] [--out DIR]

1. Device ms per B = 16 batch (CUDA events over --batches batches after a warm-up): dim_render_dataset with every output
   (lit colour, unlit colour, u16 depth, label) against dim_render (float BGR + depth) on the same poses.
2. gen_syn_set on 2 classes x --images images in a temporary directory, with 1 PNG encoder thread and with --threads:
   images/s, split into pose sampling (host), device time (render + copy back, synchronous) and encode / write time.
Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "mx-deepim_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from deepim_b200 import synth, toolkit  # noqa: E402
from deepim_b200.context import Context  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # the numbers still carry the torch device name
        return torch.cuda.get_device_name(0), "unknown (%s)" % type(e).__name__


def batch_ms(ctx, fn, n):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=300)
    ap.add_argument("--images", type=int, default=400)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "syn_bench needs a GPU"
    name, power = card()
    meshes = [synth.make_blob(nlat=100, nlon=200, tex_size=512, seed=s) for s in (1, 2)]
    for m in meshes:
        m.normals = synth.vertex_normals(m)
    ctx = Context(0, max_batch=16, max_classes=2, max_verts=max(len(m.verts) for m in meshes),
                  max_faces=max(len(m.faces) for m in meshes))
    for i, m in enumerate(meshes):
        ctx.upload_mesh(i, m)
    K = toolkit.K_LM.astype(np.float32)
    rs = np.random.RandomState(0)
    B = 16
    poses = np.stack([np.hstack([synth.random_rotation(rs), [[rs.normal(0, 0.05)], [rs.normal(0, 0.05)], [0.7 + rs.rand() * 0.3]]])
                      for _ in range(B)]).astype(np.float32)
    cls = torch.from_numpy((np.arange(B) % 2).astype(np.int32)).cuda()
    pose = torch.from_numpy(poses).cuda()
    lp = torch.from_numpy(np.stack([[p[0, 3], -p[1, 3], -p[2, 3]] for p in poses]).astype(np.float32) + 0.5).cuda()
    li = torch.from_numpy(toolkit.LIGHT_COLOURS[np.arange(B) % 7].astype(np.float32)).cuda()
    ratio = torch.from_numpy(np.array([toolkit.BRIGHTNESS_RATIOS[b % 5] for b in range(B)], np.float32)).cuda()
    res = {"card": name, "power_limit": power, "B": B, "H": 480, "W": 640, "verts_per_mesh": len(meshes[0].verts)}
    res["render_dataset_ms"] = batch_ms(ctx, lambda: ctx.render_dataset(
        cls, pose, K, light_position=lp, light_intensity=li, brightness_ratio=ratio,
        want=("lit_bgr", "bgr", "depth", "label")), a.batches)
    res["render_ms"] = batch_ms(ctx, lambda: ctx.render(cls, pose, K, trunc_u8=False, want=("bgr", "depth")), a.batches)

    # gen_syn_set: training poses of two classes, then the whole ds_0 ... ds_4 chain
    work = a.out or tempfile.mkdtemp(prefix="syn_bench_")
    lm = os.path.join(work, "LM6d_refine")
    classes = ["ape", "can"]
    os.makedirs(os.path.join(lm, "image_set", "observed"), exist_ok=True)
    for ci, c in enumerate(classes):
        os.makedirs(os.path.join(lm, "data", "gt_observed", c), exist_ok=True)
        idx = ["%02d/%06d" % (ci + 1, i + 1) for i in range(50)]
        with open(os.path.join(lm, "image_set", "observed", "%s_train.txt" % c), "w") as f:
            f.write("".join(x + "\n" for x in idx))
        for x in idx:
            p = np.hstack([synth.random_rotation(rs), [[rs.normal(0, 0.03)], [rs.normal(0, 0.03)], [0.8 + rs.normal(0, 0.05)]]])
            toolkit._write_pose_txt(os.path.join(lm, "data", "gt_observed", c, x.split("/")[1] + "-pose.txt"), ci + 1, p)
    timers = {"device": 0.0, "sampling": 0.0}
    dev_batch, render, sample = toolkit._device_batch, ctx.render, toolkit.gen_syn_observed_poses

    def timed(key, fn):
        def w(*args, **kw):
            t = time.perf_counter()
            try:
                return fn(*args, **kw)
            finally:
                torch.cuda.synchronize()
                timers[key] += time.perf_counter() - t
        return w

    toolkit._device_batch = timed("device", dev_batch)
    toolkit.gen_syn_observed_poses = timed("sampling", sample)
    ctx.render = timed("device", render)
    n_img = len(classes) * a.images
    for threads in (1, a.threads):
        syn = os.path.join(work, "syn_%d" % threads)
        timers.update(device=0.0, sampling=0.0)
        t = time.perf_counter()
        toolkit.gen_syn_set(lm, syn, ctx, classes, num_images=a.images, workers=threads)
        wall = time.perf_counter() - t
        res["gen_syn_set_threads_%d" % threads] = {
            "images": n_img, "wall_s": wall, "images_per_s": n_img / wall, "sampling_s": timers["sampling"],
            "device_s": timers["device"], "encode_write_s": wall - timers["device"] - timers["sampling"]}
        shutil.rmtree(syn)
    if a.out is None:
        shutil.rmtree(work)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
