"""Several instances per observed frame: the frame-indexed host entry against duplicating the frame per instance; and
several cameras in one batch: the per-frame-intrinsics host entry against splitting the batch by camera.

    python tools/frames_bench.py [--steps 4] [--warmup 1] [--rounds 3] [--batch 16] [--slots 4] [--out FILE]

C2 inputs (the 5k-vert blob, 4 iterations, fp16, random-init weights), device batches of `batch` instances, `slots` batches
in flight through PoseRefiner (as bench.py's e2e arm), pinned host u8 frames.  Every device batch observes batch / k frames,
k instances per frame (an initial hypothesis each: the frame's object pose perturbed as synth.sample_pose_pairs does), over
3 rotating input sets.  Three passes alternate `rounds` times:
  dup       dim_refine_host_async without a frame map, each frame copied once per instance (k = 8): `batch` frames
            uploaded and packed
  frames8   dim_refine_host_async with a frame map, k = 8: batch / 8 frames uploaded and packed
  frames2   dim_refine_host_async with a frame map, k = 2: batch / 2 frames
  cams_mixed  dim_refine_host_async with a frame map and K_frames: `batch` instances, 2 per frame, over batch / 2 frames
              from 4 cameras (each frame rendered with its own camera), one batch with one K per frame
  cams_split  the same instances split by camera into 4 batches of batch / 4 through dim_refine_host_async with a frame
              map and K9, what a caller without per-frame intrinsics has to do
  cams_one    the same poses, every frame rendered with the first camera: one batch of `batch` through
              dim_refine_host_async with a frame map and K9
Reported per pass: refinements/s end to end (host wall clock around `steps` x 32 batches of `batch` instances, results
consumed; best round), host-to-device bytes per batch (computed from the shapes), and for dup / frames8 / frames2, from a
pass of one batch at a time on one context with the stage events on (dim_profile_enable) the batch time, the chain's four
stages and their difference: the upload + pack (+ the 8 KB result download) of the batch.  dup and frames8 observe the same
frames: their poses are checked to be equal; so are cams_mixed's and cams_split's.
The card's name and power limit are reported with the numbers.  Prints one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "mx-deepim_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from deepim_b200 import synth  # noqa: E402
from deepim_b200.refiner import PoseRefiner  # noqa: E402
from variant_bench import card  # noqa: E402

N_ITER, STEP_BATCHES, N_SETS, H, W = 4, 32, 3, 480, 640
N_CAMS = 4
CAMERAS = np.array([[[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]],  # LINEMOD
                    [[1066.778, 0.0, 312.9869], [0.0, 1067.487, 241.3109], [0.0, 0.0, 1.0]],    # YCB-Video camera 1
                    [[1077.836, 0.0, 323.7872], [0.0, 1078.189, 279.6921], [0.0, 0.0, 1.0]],    # YCB-Video camera 2
                    [[800.0, 0.0, 410.5], [0.0, 790.0, 190.25], [0.0, 0.0, 1.0]]], np.float32)  # off-centre


def observed_u8(ctx, poses, K, seed, dev):
    """the blob at `poses` rendered with camera K over uniform noise: BGR u8 [n,H,W,3] on the host"""
    n = len(poses)
    r = ctx.render(torch.zeros(n, dtype=torch.int32, device=dev), torch.from_numpy(poses.astype(np.float32)).to(dev), K,
                   want=("bgr", "mask"))
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    bg = torch.randint(0, 256, r["bgr"].shape, generator=g, device=dev, dtype=torch.int32).to(torch.uint8)
    return torch.where(r["mask"].permute(0, 2, 3, 1) > 0, r["bgr"].to(torch.uint8), bg).cpu()


def make_camera_sets(ctx, B, seed, dev):
    """N_SETS input sets of B instances, 2 per frame, over B // 2 frames from N_CAMS cameras (the frames of camera c
    contiguous): "frames" rendered with their own cameras and "K" one row per frame, "frames_one" the same poses all
    rendered with CAMERAS[0], and "split" the sub-batch of each camera (its frames and instances, pinned on their own)"""
    F, per = B // 2, B // 2 // N_CAMS
    frame_of = np.repeat(np.arange(F, dtype=np.int32), 2)
    cam = np.repeat(np.arange(N_CAMS), per)
    sets = []
    for s in range(N_SETS):
        fobs, _ = synth.sample_pose_pairs(F, seed + 100 * s)
        pobs, pini = synth.sample_pose_pairs(B, seed + 100 * s + 1)
        ini = pini.copy()
        ini[:, :, 3] = fobs[frame_of][:, :, 3] + (pini[:, :, 3] - pobs[:, :, 3])
        u8 = torch.cat([observed_u8(ctx, fobs[cam == c], CAMERAS[c], seed + 10 * s + c, dev) for c in range(N_CAMS)])
        one = observed_u8(ctx, fobs, CAMERAS[0], seed + 10 * s, dev)
        cls, pose = torch.zeros(B, dtype=torch.int32), torch.from_numpy(ini)
        split = [{"frames": u8[c * per:(c + 1) * per].contiguous().pin_memory(),
                  "frame_of": torch.from_numpy(frame_of[:2 * per].copy()).pin_memory(),
                  "cls": cls[:2 * per].clone().pin_memory(), "pose": pose[c * 2 * per:(c + 1) * 2 * per].clone().pin_memory(),
                  "K9": CAMERAS[c]} for c in range(N_CAMS)]
        sets.append({"frames": u8.pin_memory(), "frames_one": one.pin_memory(), "K": torch.from_numpy(CAMERAS[cam]).pin_memory(),
                     "frame_of": torch.from_numpy(frame_of).pin_memory(), "cls": cls.pin_memory(), "pose": pose.pin_memory(),
                     "split": split})
    return sets


def make_sets(ctx, mesh, B, k, seed, dev):
    """N_SETS pinned input sets of B instances over B // k frames composited over noise"""
    F = B // k
    frame_of = np.repeat(np.arange(F, dtype=np.int32), k)
    sets = []
    for s in range(N_SETS):
        fobs, _ = synth.sample_pose_pairs(F, seed + 100 * s)
        pobs, pini = synth.sample_pose_pairs(B, seed + 100 * s + 1)
        ini = pini.copy()
        ini[:, :, 3] = fobs[frame_of][:, :, 3] + (pini[:, :, 3] - pobs[:, :, 3])
        r = ctx.render(torch.zeros(F, dtype=torch.int32, device=dev), torch.from_numpy(fobs.astype(np.float32)).to(dev),
                       synth.K_LINEMOD, want=("bgr", "mask"))
        g = torch.Generator(device=dev)
        g.manual_seed(seed + s)
        bg = torch.randint(0, 256, r["bgr"].shape, generator=g, device=dev, dtype=torch.int32).to(torch.uint8)
        u8 = torch.where(r["mask"].permute(0, 2, 3, 1) > 0, r["bgr"].to(torch.uint8), bg).cpu()
        sets.append({"frames": u8.pin_memory(), "dup": u8[torch.from_numpy(frame_of).long()].contiguous().pin_memory(),
                     "frame_of": torch.from_numpy(frame_of).pin_memory(),
                     "cls": torch.zeros(B, dtype=torch.int32).pin_memory(), "pose": torch.from_numpy(ini).pin_memory()})
    return sets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--slots", type=int, default=4)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frames_bench.py: no CUDA device; the product path has no CPU fallback")
    B = a.batch
    if B % 8:
        raise SystemExit("frames_bench.py: --batch must be a multiple of 8")  # also 2 instances per frame, 4 cameras
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    K, means = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
    mesh = synth.make_blob()
    ref = PoseRefiner([mesh], synth.make_weights(0), K, device=0, max_batch=B, n_iter=N_ITER, precision="fp16",
                      n_slots=a.slots)
    ctx0 = ref.ctx
    sets = {8: make_sets(ctx0, mesh, B, 8, 3000, dev), 2: make_sets(ctx0, mesh, B, 2, 4000, dev)}
    cam_sets = make_camera_sets(ctx0, B, 5000, dev)
    torch.cuda.synchronize()

    def with_k(K9, submit):  # the single-camera entries take the refiner's K, read when the batch is enqueued
        def f(s):
            ref.K = K9
            return submit(s)
        return f
    frames_submit = lambda s: ref.submit_frames(s["frames"], s["frame_of"], s["cls"], s["pose"])  # noqa: E731
    passes = {  # name -> (input sets, submit of one device batch, device batches per batch of B instances)
        "dup": (sets[8], with_k(K, lambda s: ref.submit(s["dup"], s["cls"], s["pose"])), 1),
        "frames8": (sets[8], with_k(K, frames_submit), 1),
        "frames2": (sets[2], with_k(K, frames_submit), 1),
        "cams_mixed": (cam_sets, lambda s: ref.submit_frames(s["frames"], s["frame_of"], s["cls"], s["pose"], K_frames=s["K"]),
                       1),
        "cams_split": ([sub for s in cam_sets for sub in s["split"]], lambda s: with_k(s["K9"], frames_submit)(s), N_CAMS),
        "cams_one": (cam_sets, with_k(CAMERAS[0], lambda s: ref.submit_frames(s["frames_one"], s["frame_of"], s["cls"],
                                                                             s["pose"])), 1),
    }

    def run(name, n_batches):
        ss, submit, per = passes[name]
        pending, last = [], None
        for k in range(n_batches * per):
            if len(pending) == len(ref.slots):
                last = ref.result(pending.pop(0))
            pending.append(submit(ss[k % len(ss)]))
        for t in pending:
            last = ref.result(t)
        return last

    def e2e(name, n_steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(name, n_steps * STEP_BATCHES)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    # same frames, same instances: the duplicated and the frame-indexed upload refine identically
    p_dup = run("dup", 1)
    p_fr = run("frames8", 1)
    assert np.array_equal(p_dup, p_fr), "a frame map differs from duplicated frames (dim_refine_host_async)"
    p_mixed = run("cams_mixed", 1)
    p_split = []
    for sub in cam_sets[0]["split"]:
        p_split.append(ref.result(passes["cams_split"][1](sub)))
    assert np.array_equal(p_mixed, np.concatenate(p_split, axis=1)), \
        "K_frames differs from K9 on the per-camera batches (dim_refine_host_async)"
    for name in passes:  # every (slot, input set) argument set: eager run, then graph capture
        run(name, 2 * N_SETS * N_CAMS * len(ref.slots))
        e2e(name, a.warmup)
    best = {}
    for _ in range(a.rounds):
        for name in passes:
            ms = e2e(name, a.steps)
            best[name] = min(best.get(name, ms), ms)

    def stage_pass(name, n=STEP_BATCHES):
        """one batch at a time on slot 0's context and stream, the stage events on (the chain runs eagerly)"""
        ss = passes[name][0]
        st = ref.slots[0]["stream"]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        ctx0.profile_enable(True)
        total = 0.0
        out = dict(poses_out=ref.slots[0]["poses"], se3_out=ref.slots[0]["se3"], sync=False)  # pinned
        with torch.cuda.stream(st):
            for k in range(n):
                s = ss[k % len(ss)]
                e0.record(st)
                if name == "dup":
                    ctx0.refine_host(s["dup"], s["cls"], s["pose"], K, N_ITER, pixel_means_rgb=means, precision=ref.precision,
                                     **out)
                else:
                    ctx0.refine_frames_host(s["frames"], s["frame_of"], s["cls"], s["pose"], K, N_ITER, pixel_means_rgb=means,
                                            precision=ref.precision, **out)
                e1.record(st)
                e1.synchronize()
                total += e0.elapsed_time(e1)
        stages, _ = ctx0.profile_read()
        ctx0.profile_enable(False)
        chain = sum(stages.values())
        return {"batch_ms": round(total / n, 4), "chain_ms": round(chain / n, 4),
                "upload_pack_ms": round((total - chain) / n, 4),
                "chain_stages_ms": {k: round(v / n, 4) for k, v in stages.items()}}

    stage_pass("dup", 4)  # warm the eager chain
    n_ref = B * STEP_BATCHES * a.steps
    P = H * W
    res = {"metric": "480x640 4-iter pose refinements/sec, several instances per observed frame, host u8 frames in",
           "unit": "refinements/s", "gpu": torch.cuda.get_device_name(dev), "card": card(), "batch": B, "slots": a.slots,
           "steps": a.steps, "rounds": a.rounds, "precision": "fp16", "weights": "random-init", "workload": "C2"}
    for name, (ss, _, per) in passes.items():
        F = B if name == "dup" else int(ss[0]["frames"].shape[0]) * per
        # frames + cls + pose (+ frame indices) (+ the cameras: 36 B per frame)
        h2d = F * P * 3 + B * (4 + 96) + (0 if name == "dup" else 4 * B) + (36 * F if name == "cams_mixed" else 0)
        res[name] = {"frames_per_batch": F, "device_batches_per_batch": per, "value": round(n_ref / (best[name] / 1e3), 2),
                     "ms_per_step": round(best[name] / a.steps, 4), "h2d_bytes_per_batch": h2d}
        if not name.startswith("cams"):
            res[name]["one_batch_at_a_time"] = stage_pass(name)
    for name in ("frames8", "frames2"):
        res[name]["over_dup"] = round(res[name]["value"] / res["dup"]["value"], 4)
    res["cams_mixed"]["over_split"] = round(res["cams_mixed"]["value"] / res["cams_split"]["value"], 4)
    res["cams_mixed"]["over_one"] = round(res["cams_mixed"]["value"] / res["cams_one"]["value"], 4)
    ref.close()
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
