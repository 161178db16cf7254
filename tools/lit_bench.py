"""Cost of the ModelNet branch's lit refinement loop against the unlit loop on the headline workload (config C2).

    python tools/lit_bench.py [--steps 10] [--warmup 2] [--rounds 2] [--batch 16] [--slots 4]

Same inputs, pass shape and precision (fp16) as bench.py's device-resident `value`: one step = 32 device batches of `batch`
instances, `slots` batches in flight on as many contexts / streams, 3 rotating input sets.  The lit loop is dim_refine with
a dim_lighting (Lambert-lit render; light = (0, .5, .5) + (t_x, -t_y, -t_z) of the float64 pose, brightness ratio 0.7), normals from
synth.vertex_normals, light intensities [4, batch, 3] drawn once from default_rng(2024).  The unlit and lit passes alternate
`rounds` times so that clock drift under a power cap hits both alike; the best round of each is reported, plus the stage
times (render / zoom / conv / head) of a single-stream pass with CUDA events between the stages.  Random-init weights: the
timed work does not depend on the weight values.  Prints one JSON line."""
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

import bench  # noqa: E402  (input sets and the clock sampler of the headline benchmark)
from deepim_b200 import lighting, synth  # noqa: E402
from deepim_b200.refiner import PoseRefiner  # noqa: E402

N_ITER, STEP_BATCHES, N_SETS, SEED = 4, 32, 3, 2024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--slots", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lit_bench.py: no CUDA device; the product path has no CPU fallback")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, K, means = a.batch, synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
    mesh = synth.make_blob()
    mesh.normals = synth.vertex_normals(mesh)
    refiner = PoseRefiner([mesh], synth.make_weights(0), K, device=0, max_batch=B, n_iter=N_ITER, n_slots=a.slots)
    ctxs = [s["ctx"] for s in refiner.slots]
    streams = [s["stream"] for s in refiner.slots]
    sets = bench.make_inputs(ctxs[0], synth, mesh, B, N_SETS, 1000, dev, torch)
    lit_arg = {"intensity": torch.from_numpy(lighting.sample_intensity(np.random.default_rng(SEED), (N_ITER, B))).to(dev),
               "offset": lighting.OFFSET, "brightness_ratio": lighting.BRIGHTNESS_RATIO}
    outs = {False: {}, True: {}}  # persistent result tensors per (mode, slot): the library replays its CUDA graphs

    def batch(k, i, lit, ctx):
        s = sets[k % len(sets)]
        o = outs[lit is not None]
        o[i] = ctx.refine(s["img_dev"], s["cls_dev"], s["pose_dev"], K, N_ITER, pixel_means_rgb=means, out=o.get(i), lighting=lit)

    def device_pass(lit, n_steps, sampler=None):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.time()
        e0.record()
        for st in streams:
            st.wait_event(e0)
        for k in range(n_steps * STEP_BATCHES):
            i = k % len(streams)
            with torch.cuda.stream(streams[i]):
                batch(k, i, lit, ctxs[i])
        for st in streams:
            torch.cuda.current_stream().wait_stream(st)
        e1.record()
        torch.cuda.synchronize()
        clocks = sampler.stop(t0, time.time()) if sampler else None
        return e0.elapsed_time(e1), clocks

    def stage_pass(lit):
        torch.cuda.synchronize()
        ctxs[0].profile_enable(True)
        for k in range(STEP_BATCHES):
            batch(k, 0, lit, ctxs[0])
        torch.cuda.synchronize()
        stages, _ = ctxs[0].profile_read()
        ctxs[0].profile_enable(False)
        return {k: round(v / STEP_BATCHES, 4) for k, v in stages.items()}

    for lit in (None, lit_arg):  # first sight of every argument set runs eagerly, the next one captures the graphs
        for k in range(2 * len(streams)):
            i = k % len(streams)
            with torch.cuda.stream(streams[i]):
                batch(k, i, lit, ctxs[i])
        device_pass(lit, a.warmup)
    best = {False: None, True: None}
    for _ in range(a.rounds):
        for lit in (None, lit_arg):
            sampler = bench.ClockSampler(0)
            sampler.start()
            time.sleep(0.3)
            ms, clocks = device_pass(lit, a.steps, sampler)
            key = lit is not None
            if best[key] is None or ms < best[key][0]:
                best[key] = (ms, clocks)
    stages = {False: stage_pass(None), True: stage_pass(lit_arg)}
    n_ref = B * STEP_BATCHES * a.steps
    res = {"metric": "480x640 4-iter pose refinements/sec, unlit vs lit (ModelNet) loop", "unit": "refinements/s",
           "gpu": torch.cuda.get_device_name(dev), "batch": B, "slots": a.slots, "steps": a.steps, "rounds": a.rounds,
           "precision": "fp16", "weights": "random-init"}
    for key, name in ((False, "unlit"), (True, "lit")):
        ms, clocks = best[key]
        res[name] = {"value": round(n_ref / (ms / 1e3), 2), "ms_per_step": round(ms / a.steps, 4), "clocks": clocks,
                     "stages_ms_per_batch_single_stream": stages[key]}
    res["lit_over_unlit"] = round(res["lit"]["value"] / res["unlit"]["value"], 4)
    refiner.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
