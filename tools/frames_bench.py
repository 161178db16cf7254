"""Several instances per observed frame: the frame-indexed host entry against duplicating the frame per instance.

    python tools/frames_bench.py [--steps 4] [--warmup 1] [--rounds 3] [--batch 16] [--slots 4] [--out FILE]

C2 inputs (the 5k-vert blob, 4 iterations, fp16, random-init weights), device batches of `batch` instances, `slots` batches
in flight through PoseRefiner (as bench.py's e2e arm), pinned host u8 frames.  Every device batch observes batch / k frames,
k instances per frame (an initial hypothesis each: the frame's object pose perturbed as synth.sample_pose_pairs does), over
3 rotating input sets.  Three passes alternate `rounds` times:
  dup       dim_refine_host_async with each frame copied once per instance (k = 8): `batch` frames uploaded and packed
  frames8   dim_refine_frames_host_async, k = 8: batch / 8 frames uploaded and packed
  frames2   dim_refine_frames_host_async, k = 2: batch / 2 frames
Reported per pass: refinements/s end to end (host wall clock around `steps` x 32 batches, results consumed; best round),
host-to-device bytes per batch (computed from the shapes), and from a pass of one batch at a time on one context with
the stage events on (dim_profile_enable) the batch time, the chain's four stages and their difference: the upload + pack
(+ the 8 KB result download) of the batch.  dup and frames8 observe the same frames: their poses are checked to be equal.
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
        raise SystemExit("frames_bench.py: --batch must be a multiple of 8")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    K, means = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
    mesh = synth.make_blob()
    ref = PoseRefiner([mesh], synth.make_weights(0), K, device=0, max_batch=B, n_iter=N_ITER, precision="fp16",
                      n_slots=a.slots)
    ctx0 = ref.ctx
    sets = {8: make_sets(ctx0, mesh, B, 8, 3000, dev), 2: make_sets(ctx0, mesh, B, 2, 4000, dev)}
    torch.cuda.synchronize()
    passes = {  # name -> (input sets, submit of one batch)
        "dup": (sets[8], lambda s: ref.submit(s["dup"], s["cls"], s["pose"])),
        "frames8": (sets[8], lambda s: ref.submit_frames(s["frames"], s["frame_of"], s["cls"], s["pose"])),
        "frames2": (sets[2], lambda s: ref.submit_frames(s["frames"], s["frame_of"], s["cls"], s["pose"])),
    }

    def run(name, n_batches):
        ss, submit = passes[name]
        pending, last = [], None
        for k in range(n_batches):
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
    assert np.array_equal(p_dup, p_fr), "dim_refine_frames_host differs from dim_refine_host on duplicated frames"
    for name in passes:  # every (slot, input set) argument set: eager run, then graph capture
        run(name, 2 * N_SETS * len(ref.slots))
        e2e(name, a.warmup)
    best = {}
    for _ in range(a.rounds):
        for name in passes:
            ms = e2e(name, a.steps)
            best[name] = min(best.get(name, ms), ms)

    def stage_pass(name, n=STEP_BATCHES):
        """one batch at a time on slot 0's context and stream, the stage events on (the chain runs eagerly)"""
        ss, _ = passes[name]
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
    for name, (ss, _) in passes.items():
        F = B if name == "dup" else int(ss[0]["frames"].shape[0])
        h2d = F * P * 3 + B * (4 + 96) + (0 if name == "dup" else 4 * B)  # frames + cls + pose (+ frame indices)
        res[name] = {"frames_per_batch": F, "value": round(n_ref / (best[name] / 1e3), 2),
                     "ms_per_step": round(best[name] / a.steps, 4), "h2d_bytes_per_batch": h2d,
                     "one_batch_at_a_time": stage_pass(name)}
    for name in ("frames8", "frames2"):
        res[name]["over_dup"] = round(res[name]["value"] / res["dup"]["value"], 4)
    ref.close()
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
