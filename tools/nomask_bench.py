"""Cost of the image-only network (INPUT_MASK: False, 6-channel conv1, ZoomImage) against the mask network on the headline
workload (config C2).

    python tools/nomask_bench.py [--steps 10] [--warmup 2] [--rounds 2] [--batch 16] [--slots 4]

Same inputs, pass shape and precision (fp16) as bench.py's device-resident `value`: one step = 32 device batches of `batch`
instances, `slots` batches in flight on as many contexts / streams, 3 rotating input sets.  The mask passes run dim_refine on
the default contexts, the mask-free passes dim_refine on Context(input_mask=False) contexts with the same observed images
(the observed box of those is then the full frame: bench.py composites over noise).  The two alternate `rounds` times so that clock drift under a power cap hits both alike; the best round of
each is reported, plus the stage times (render / zoom / conv / head) of a single-stream pass with CUDA events between the
stages and the per-layer conv times of one forward pass.  Random-init weights: the timed work does not depend on the weight
values.  The card's name and power limit are reported with the numbers.  Prints one JSON line."""
import argparse
import ctypes
import json
import os
import subprocess
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

N_ITER, STEP_BATCHES, N_SETS = 4, 32, 3


def card():
    q = "name,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        f = [x.strip() for x in out.split(",")]
        return {"name": f[0], "power_limit_w": float(f[1])}
    except Exception as e:  # noqa: BLE001  (a report field, not a measurement)
        return {"error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--slots", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nomask_bench.py: no CUDA device; the product path has no CPU fallback")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, K, means = a.batch, synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
    mesh = synth.make_blob()
    w8 = synth.make_weights(0)
    w6 = dict(w8, flow_conv1_weight=np.ascontiguousarray(w8["flow_conv1_weight"][:, :6]))
    ctxs, streams = {}, [torch.cuda.Stream(dev) for _ in range(a.slots)]
    for nomask, w in ((False, w8), (True, w6)):
        ctxs[nomask] = []
        for _ in range(a.slots):
            c = Context(0, max_batch=B, max_classes=1, max_verts=6000, max_faces=11000, input_mask=not nomask)
            c.upload_mesh(0, mesh)
            c.load_weights(w)
            ctxs[nomask].append(c)
    sets = bench.make_inputs(ctxs[False][0], synth, mesh, B, N_SETS, 1000, dev, torch)
    outs = {False: {}, True: {}}  # persistent result tensors per (mode, slot): the library replays its CUDA graphs

    def batch(k, i, nomask, ctx):
        s = sets[k % len(sets)]
        o = outs[nomask]
        o[i] = ctx.refine(s["img_dev"], s["cls_dev"], s["pose_dev"], K, N_ITER, pixel_means_rgb=means, out=o.get(i))

    def device_pass(nomask, n_steps, sampler=None):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.time()
        e0.record()
        for st in streams:
            st.wait_event(e0)
        for k in range(n_steps * STEP_BATCHES):
            i = k % len(streams)
            with torch.cuda.stream(streams[i]):
                batch(k, i, nomask, ctxs[nomask][i])
        for st in streams:
            torch.cuda.current_stream().wait_stream(st)
        e1.record()
        torch.cuda.synchronize()
        clocks = sampler.stop(t0, time.time()) if sampler else None
        return e0.elapsed_time(e1), clocks

    def stage_pass(nomask):
        c = ctxs[nomask][0]
        torch.cuda.synchronize()
        c.profile_enable(True)
        for k in range(STEP_BATCHES):
            batch(k, 0, nomask, c)
        torch.cuda.synchronize()
        stages, _ = c.profile_read()
        c.profile_enable(False)
        ms10 = (ctypes.c_float * 10)()
        capi.check(capi.lib.dim_debug_layer_profile(c._h, 1, None))
        layers = np.zeros(10)
        for k in range(8):
            batch(k, 0, nomask, c)
            capi.check(capi.lib.dim_debug_layer_profile(c._h, 1, ms10))
            if k >= 3:  # the layer times of the call's last forward pass
                layers += np.array(ms10[:])
        capi.check(capi.lib.dim_debug_layer_profile(c._h, 0, None))
        layers /= 5
        return {k: round(v / STEP_BATCHES, 4) for k, v in stages.items()}, [round(float(x), 4) for x in layers]

    for nomask in (False, True):  # first sight of every argument set runs eagerly, the next one captures the graphs
        for k in range(2 * N_SETS * len(streams)):
            i = k % len(streams)
            with torch.cuda.stream(streams[i]):
                batch(k, i, nomask, ctxs[nomask][i])
        device_pass(nomask, a.warmup)
    best = {False: None, True: None}
    for _ in range(a.rounds):
        for nomask in (False, True):
            sampler = bench.ClockSampler(0)
            sampler.start()
            time.sleep(0.3)
            ms, clocks = device_pass(nomask, a.steps, sampler)
            if best[nomask] is None or ms < best[nomask][0]:
                best[nomask] = (ms, clocks)
    stages = {d: stage_pass(d) for d in (False, True)}
    n_ref = B * STEP_BATCHES * a.steps
    res = {"metric": "480x640 4-iter pose refinements/sec, mask vs image-only (INPUT_MASK: False) network",
           "unit": "refinements/s", "gpu": torch.cuda.get_device_name(dev), "card": card(), "batch": B, "slots": a.slots,
           "steps": a.steps, "rounds": a.rounds, "precision": "fp16", "weights": "random-init"}
    for nomask, name in ((False, "mask"), (True, "nomask")):
        ms, clocks = best[nomask]
        res[name] = {"value": round(n_ref / (ms / 1e3), 2), "ms_per_step": round(ms / a.steps, 4), "clocks": clocks,
                     "stages_ms_per_batch_single_stream": stages[nomask][0],
                     "conv_layer_ms_per_forward": stages[nomask][1]}
    res["nomask_over_mask"] = round(res["nomask"]["value"] / res["mask"]["value"], 4)
    for cs in ctxs.values():
        for c in cs:
            c.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
