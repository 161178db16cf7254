"""Cost of a network variant against the baseline loop on the headline workload (config C2).

    python tools/variant_bench.py --variant {lit,rgbd,nomask} [--steps 10] [--warmup 2] [--rounds 2] [--batch 16] [--slots 4]

  lit     the ModelNet branch's lit loop: dim_refine with a dim_lighting (Lambert-lit render; light = (0, .5, .5) +
          (t_x, -t_y, -t_z) of the float64 pose, brightness ratio 0.7), normals from synth.vertex_normals, light
          intensities [4, batch, 3] drawn once from default_rng(2024); baseline: the unlit loop
  rgbd    the RGB-D network (INPUT_DEPTH: 10-channel conv1) on Context(input_depth=True) contexts with a fixed observed
          depth per input set, uniform in [0.5, 1.5) m from default_rng(2024); baseline: the RGB network
  nomask  the image-only network (INPUT_MASK: False, 6-channel conv1, ZoomImage) on Context(input_mask=False) contexts;
          bench.py composites its observed images over noise, so their observed box is the full frame; baseline: the
          mask network

Same inputs, pass shape and precision (fp16) as bench.py's device-resident `value`: one step = 32 device batches of `batch`
instances, `slots` batches in flight on as many contexts / streams, 3 rotating input sets.  Baseline and variant each get
their own `slots` contexts, built alike, and every (input set, slot) argument set of both is warmed up (eager, then graph
capture) before anything is timed.  The two alternate `rounds` times so that clock drift under a power cap hits both
alike; the best round of each is reported, plus the stage times (render / zoom / conv / head) of a single-stream pass with
CUDA events between the stages and the per-layer conv times of one forward pass.  Random-init weights: the timed work does
not depend on the weight, depth or intensity values.  The card's name and power limit are reported with the numbers.
Prints one JSON line."""
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
from deepim_b200 import lighting, synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402

N_ITER, STEP_BATCHES, N_SETS, SEED = 4, 32, 3, 2024
# variant -> (what the metric compares, baseline pass name, variant pass name)
VARIANTS = {"lit": ("unlit vs lit (ModelNet) loop", "unlit", "lit"),
            "rgbd": ("RGB vs RGB-D (INPUT_DEPTH) network", "rgb", "rgbd"),
            "nomask": ("mask vs image-only (INPUT_MASK: False) network", "mask", "nomask")}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        f = [x.strip() for x in out.split(",")]
        return {"name": f[0], "power_limit_w": float(f[1])}
    except Exception as e:  # noqa: BLE001  (a report field, not a measurement)
        return {"error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", required=True, choices=sorted(VARIANTS))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--slots", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("variant_bench.py: no CUDA device; the product path has no CPU fallback")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, K, means = a.batch, synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
    mesh = synth.make_blob()
    mesh.normals = synth.vertex_normals(mesh)
    streams = [torch.cuda.Stream(dev) for _ in range(a.slots)]

    def contexts(weights, **network):
        cs = []
        for _ in range(a.slots):
            c = Context(0, max_batch=B, max_classes=1, max_verts=6000, max_faces=11000, **network)
            c.upload_mesh(0, mesh)
            c.load_weights(weights)
            cs.append(c)
        return cs

    w8 = synth.make_weights(0)
    base = contexts(w8)
    sets = bench.make_inputs(base[0], synth, mesh, B, N_SETS, 1000, dev, torch)
    rng = np.random.default_rng(SEED)
    if a.variant == "lit":
        lit = {"intensity": torch.from_numpy(lighting.sample_intensity(rng, (N_ITER, B))).to(dev),
               "offset": lighting.OFFSET, "brightness_ratio": lighting.BRIGHTNESS_RATIO}
        var, var_args = contexts(w8), lambda s: {"lighting": lit}
    elif a.variant == "rgbd":
        for s in sets:
            s["depth_dev"] = torch.from_numpy(rng.uniform(0.5, 1.5, (B, 1, 480, 640)).astype(np.float32)).to(dev)
        var = contexts(synth.make_weights(0, input_depth=True), input_depth=True)
        var_args = lambda s: {"depth_observed": s["depth_dev"]}
    else:
        w6 = dict(w8, flow_conv1_weight=np.ascontiguousarray(w8["flow_conv1_weight"][:, :6]))
        var, var_args = contexts(w6, input_mask=False), lambda s: {}
    modes = [(base, lambda s: {}), (var, var_args)]
    outs = [{}, {}]  # persistent result tensors per (mode, slot): the library replays its CUDA graphs

    def batch(k, i, m):
        s = sets[k % len(sets)]
        ctxs, args = modes[m]
        outs[m][i] = ctxs[i].refine(s["img_dev"], s["cls_dev"], s["pose_dev"], K, N_ITER, pixel_means_rgb=means,
                                    out=outs[m].get(i), **args(s))

    def device_pass(m, n_steps, sampler=None):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.time()
        e0.record()
        for st in streams:
            st.wait_event(e0)
        for k in range(n_steps * STEP_BATCHES):
            i = k % len(streams)
            with torch.cuda.stream(streams[i]):
                batch(k, i, m)
        for st in streams:
            torch.cuda.current_stream().wait_stream(st)
        e1.record()
        torch.cuda.synchronize()
        clocks = sampler.stop(t0, time.time()) if sampler else None
        return e0.elapsed_time(e1), clocks

    def stage_pass(m):
        c = modes[m][0][0]
        torch.cuda.synchronize()
        c.profile_enable(True)
        for k in range(STEP_BATCHES):
            batch(k, 0, m)
        torch.cuda.synchronize()
        stages, _ = c.profile_read()
        c.profile_enable(False)
        ms10 = (ctypes.c_float * 10)()
        capi.check(capi.lib.dim_debug_layer_profile(c._h, 1, None))
        layers = np.zeros(10)
        for k in range(8):
            batch(k, 0, m)
            capi.check(capi.lib.dim_debug_layer_profile(c._h, 1, ms10))
            if k >= 3:  # the layer times of the call's last forward pass
                layers += np.array(ms10[:])
        capi.check(capi.lib.dim_debug_layer_profile(c._h, 0, None))
        layers /= 5
        return {k: round(v / STEP_BATCHES, 4) for k, v in stages.items()}, [round(float(x), 4) for x in layers]

    for m in (0, 1):  # first sight of every argument set runs eagerly, the next one captures the graphs
        for k in range(2 * N_SETS * len(streams)):
            i = k % len(streams)
            with torch.cuda.stream(streams[i]):
                batch(k, i, m)
        device_pass(m, a.warmup)
    best = [None, None]
    for _ in range(a.rounds):
        for m in (0, 1):
            sampler = bench.ClockSampler(0)
            sampler.start()
            time.sleep(0.3)
            ms, clocks = device_pass(m, a.steps, sampler)
            if best[m] is None or ms < best[m][0]:
                best[m] = (ms, clocks)
    stages = [stage_pass(m) for m in (0, 1)]
    n_ref = B * STEP_BATCHES * a.steps
    title, *names = VARIANTS[a.variant]
    res = {"metric": "480x640 4-iter pose refinements/sec, " + title, "unit": "refinements/s", "variant": a.variant,
           "gpu": torch.cuda.get_device_name(dev), "card": card(), "batch": B, "slots": a.slots, "steps": a.steps,
           "rounds": a.rounds, "precision": "fp16", "weights": "random-init"}
    for m, name in enumerate(names):
        ms, clocks = best[m]
        res[name] = {"value": round(n_ref / (ms / 1e3), 2), "ms_per_step": round(ms / a.steps, 4), "clocks": clocks,
                     "stages_ms_per_batch_single_stream": stages[m][0], "conv_layer_ms_per_forward": stages[m][1]}
    res["variant_over_baseline"] = round(res[names[1]]["value"] / res[names[0]]["value"], 4)
    for ctxs, _ in modes:
        for c in ctxs:
            c.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
