"""Cost of the RGB-D network (INPUT_DEPTH: 10-channel conv1) against the RGB network on the headline workload (config C2).

    python tools/rgbd_bench.py [--steps 10] [--warmup 2] [--rounds 2] [--batch 16] [--slots 4]

Same inputs, pass shape and precision (fp16) as bench.py's device-resident `value`: one step = 32 device batches of `batch`
instances, `slots` batches in flight on as many contexts / streams, 3 rotating input sets.  The RGB passes run dim_refine on
RGB contexts, the RGB-D passes dim_refine on RGB-D contexts (Context(input_depth=True)) with a fixed observed depth per
input set.  The two alternate `rounds` times so that clock drift under a power cap hits both alike; the best round of
each is reported, plus the stage times (render / zoom / conv / head) of a single-stream pass with CUDA events between the
stages and the per-layer conv times of one forward pass.  Random-init weights: the timed work does not depend on the weight
or depth values.  Prints one JSON line."""
import argparse
import ctypes
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
from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402

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
        raise SystemExit("rgbd_bench.py: no CUDA device; the product path has no CPU fallback")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, K, means = a.batch, synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
    mesh = synth.make_blob()
    w8 = synth.make_weights(0)
    w10 = synth.make_weights(0, input_depth=True)
    ctxs, streams = {}, [torch.cuda.Stream(dev) for _ in range(a.slots)]
    for depth, w in ((False, w8), (True, w10)):
        ctxs[depth] = []
        for _ in range(a.slots):
            c = Context(0, max_batch=B, max_classes=1, max_verts=6000, max_faces=11000, input_depth=depth)
            c.upload_mesh(0, mesh)
            c.load_weights(w)
            ctxs[depth].append(c)
    sets = bench.make_inputs(ctxs[False][0], synth, mesh, B, N_SETS, 1000, dev, torch)
    rng = np.random.default_rng(SEED)
    for s in sets:
        s["depth_dev"] = torch.from_numpy(rng.uniform(0.5, 1.5, (B, 1, 480, 640)).astype(np.float32)).to(dev)
    outs = {False: {}, True: {}}  # persistent result tensors per (mode, slot): the library replays its CUDA graphs

    def batch(k, i, depth, ctx):
        s = sets[k % len(sets)]
        o = outs[depth]
        o[i] = ctx.refine(s["img_dev"], s["cls_dev"], s["pose_dev"], K, N_ITER, pixel_means_rgb=means, out=o.get(i),
                          depth_observed=s["depth_dev"] if depth else None)

    def device_pass(depth, n_steps, sampler=None):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.time()
        e0.record()
        for st in streams:
            st.wait_event(e0)
        for k in range(n_steps * STEP_BATCHES):
            i = k % len(streams)
            with torch.cuda.stream(streams[i]):
                batch(k, i, depth, ctxs[depth][i])
        for st in streams:
            torch.cuda.current_stream().wait_stream(st)
        e1.record()
        torch.cuda.synchronize()
        clocks = sampler.stop(t0, time.time()) if sampler else None
        return e0.elapsed_time(e1), clocks

    def stage_pass(depth):
        c = ctxs[depth][0]
        torch.cuda.synchronize()
        c.profile_enable(True)
        for k in range(STEP_BATCHES):
            batch(k, 0, depth, c)
        torch.cuda.synchronize()
        stages, _ = c.profile_read()
        c.profile_enable(False)
        ms10 = (ctypes.c_float * 10)()
        capi.check(capi.lib.dim_debug_layer_profile(c._h, 1, None))
        layers = np.zeros(10)
        for k in range(8):
            batch(k, 0, depth, c)
            capi.check(capi.lib.dim_debug_layer_profile(c._h, 1, ms10))
            if k >= 3:  # the layer times of the call's last forward pass
                layers += np.array(ms10[:])
        capi.check(capi.lib.dim_debug_layer_profile(c._h, 0, None))
        layers /= 5
        return {k: round(v / STEP_BATCHES, 4) for k, v in stages.items()}, [round(float(x), 4) for x in layers]

    for depth in (False, True):  # first sight of every argument set runs eagerly, the next one captures the graphs
        for k in range(2 * N_SETS * len(streams)):
            i = k % len(streams)
            with torch.cuda.stream(streams[i]):
                batch(k, i, depth, ctxs[depth][i])
        device_pass(depth, a.warmup)
    best = {False: None, True: None}
    for _ in range(a.rounds):
        for depth in (False, True):
            sampler = bench.ClockSampler(0)
            sampler.start()
            time.sleep(0.3)
            ms, clocks = device_pass(depth, a.steps, sampler)
            if best[depth] is None or ms < best[depth][0]:
                best[depth] = (ms, clocks)
    stages = {d: stage_pass(d) for d in (False, True)}
    n_ref = B * STEP_BATCHES * a.steps
    res = {"metric": "480x640 4-iter pose refinements/sec, RGB vs RGB-D (INPUT_DEPTH) network", "unit": "refinements/s",
           "gpu": torch.cuda.get_device_name(dev), "batch": B, "slots": a.slots, "steps": a.steps, "rounds": a.rounds,
           "precision": "fp16", "weights": "random-init"}
    for depth, name in ((False, "rgb"), (True, "rgbd")):
        ms, clocks = best[depth]
        res[name] = {"value": round(n_ref / (ms / 1e3), 2), "ms_per_step": round(ms / a.steps, 4), "clocks": clocks,
                     "stages_ms_per_batch_single_stream": stages[depth][0],
                     "conv_layer_ms_per_forward": stages[depth][1]}
    res["rgbd_over_rgb"] = round(res["rgbd"]["value"] / res["rgb"]["value"], 4)
    for cs in ctxs.values():
        for c in cs:
            c.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
