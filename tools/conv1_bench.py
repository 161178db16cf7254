"""Per-layer conv tower times of the RGB network's forward pass, and flow_conv1's tensor-core rate against the card's clock.

    python tools/conv1_bench.py [--forwards 200] [--warmup 20] [--batch 16] [--precision fp16]

Runs dim_net_fwd on fixed seeded zoomed blobs (random-init weights: the timed work does not depend on the values) with
the per-layer events of dim_debug_layer_profile, and averages each layer's time over `forwards` passes.  conv1's
executed FLOP count is what conv1_kernel issues (every virtual row, 25 K steps of 16 per row and column tile, three
wgmmas per K step in bf16x3), the useful count is 2 * B * Ho * Wo * 64 * 8 * 7 * 7.  conv2 ... conv6_1 get the same executed / useful counts (igemm_flops)
and rates.  All rates are set against the dense fp16 / bf16 tensor rate at the SM clock
sampled during the timed passes (132 SMs x 4096 FLOP per clock).  The card's name, power limit and clocks are read in the
same run.  Prints one JSON line."""
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

import bench  # noqa: E402  (the clock sampler of the headline benchmark)
from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402

H, W, HO, WO, HQ = 480, 640, 240, 320, 243  # conv1 output rows per image incl. the 3 virtual rows of the strip schedule
NAMES = ["flow_conv1", "conv2", "conv3", "conv3_1", "conv4", "conv4_1", "conv5", "conv5_1", "conv6", "conv6_1"]
PREC = {"fp16": capi.PREC_FP16, "bf16": capi.PREC_BF16, "bf16x3": capi.PREC_BF16X3}
# (Cout, Cin, k, stride, pad) of conv2 ... conv6_1 (deepIM_flownet.py:63-107)
IGEMM = [(128, 64, 5, 2, 2), (256, 128, 5, 2, 2), (256, 256, 3, 1, 1), (512, 256, 3, 2, 1), (512, 512, 3, 1, 1),
         (512, 512, 3, 2, 1), (512, 512, 3, 1, 1), (1024, 512, 3, 2, 1), (1024, 1024, 3, 1, 1)]


def igemm_flops(B, passes):
    """(executed, useful) FLOP of conv2 ... conv6_1 per forward.  Executed is what conv_igemm_persistent_kernel issues: every
    128-row M tile over the virtual rows of the batch (net.cu build_geometry: BW x BH pixels, BW | Wo, unused tile rows and
    rows past the batch included) x BLOCK_N x the whole K."""
    h, w, out = HO, WO, []
    for cout, cin, k, s, pad in IGEMM:
        ho, wo = (h + 2 * pad - k) // s + 1, (w + 2 * pad - k) // s + 1
        hp = h + 2 * pad
        hp += hp & 1 if s == 2 else 0
        hq = hp // 2 if s == 2 else hp
        bw = max((d for d in range(8, min(wo, 128) + 1) if wo % d == 0), key=lambda d: d * (128 // d) * 1000 + d)
        bh = 128 // bw
        bn = 256 if cout >= 256 else 128
        tiles = -(-B * hq // bh) * (wo // bw) * (cout // bn)
        out.append((2.0 * tiles * 128 * bn * k * k * cin * passes, 2.0 * B * ho * wo * cout * cin * k * k))
        h, w = ho, wo
    return out


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        f = [x.strip() for x in out.split(",")]
        return {"name": f[0], "power_limit_w": float(f[1]), "sm_mhz_idle": float(f[2]), "sm_max_mhz": float(f[3])}
    except Exception as e:  # noqa: BLE001  (a report field, not a measurement)
        return {"error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--forwards", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--precision", default="fp16", choices=sorted(PREC))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conv1_bench.py: no CUDA device; the product path has no CPU fallback")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, prec = a.batch, PREC[a.precision]
    ctx = Context(0, max_batch=B)
    ctx.load_weights(synth.make_weights(0))
    g = torch.Generator().manual_seed(7)
    zio = ((torch.rand(B, 3, H, W, generator=g) - 0.5) * 255).to(dev)
    zir = ((torch.rand(B, 3, H, W, generator=g) - 0.5) * 255).to(dev)
    zmo = (torch.rand(B, 1, H, W, generator=g) > 0.5).float().to(dev)
    zmr = (torch.rand(B, 1, H, W, generator=g) > 0.5).float().to(dev)
    info = card()
    ms10 = (ctypes.c_float * 10)()
    capi.check(capi.lib.dim_debug_layer_profile(ctx._h, 1, None))
    for _ in range(a.warmup):
        ctx.net_forward(zio, zir, zmo, zmr, prec)
    torch.cuda.synchronize()
    layers = np.zeros(10)
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.3)
    t0 = time.time()
    for _ in range(a.forwards):
        ctx.net_forward(zio, zir, zmo, zmr, prec)
        capi.check(capi.lib.dim_debug_layer_profile(ctx._h, 1, ms10))  # synchronises, then reads this pass's events
        layers += np.array(ms10[:])
    clocks = sampler.stop(t0, time.time())
    capi.check(capi.lib.dim_debug_layer_profile(ctx._h, 0, None))
    layers /= a.forwards
    n_tile = 80 if a.precision == "bf16x3" else 160
    passes = 3 if a.precision == "bf16x3" else 1  # bf16x3: hi*hi + lo*hi + hi*lo wgmmas per K step
    executed = 2.0 * B * HQ * (WO // n_tile) * 25 * 64 * n_tile * 16 * passes
    useful = 2.0 * B * HO * WO * 64 * 8 * 7 * 7
    c1 = layers[0] * 1e-3
    res = {"metric": "conv tower per-layer device time per forward (dim_net_fwd, layer events)", "unit": "ms",
           "gpu": info, "clocks": clocks, "batch": B, "precision": a.precision, "forwards": a.forwards,
           "weights": "random-init", "layer_ms": {n: round(float(x), 4) for n, x in zip(NAMES, layers)},
           "tower_ms": round(float(layers.sum()), 4),
           "conv1": {"ms": round(float(layers[0]), 4), "executed_gflop": round(executed / 1e9, 2),
                     "useful_gflop": round(useful / 1e9, 2),
                     "executed_tflops": round(executed / c1 / 1e12, 1), "useful_tflops": round(useful / c1 / 1e12, 1)}}
    peak = 132 * 4096 * clocks["sm_mhz"] * 1e6 if clocks and clocks.get("sm_mhz") else None
    if peak:
        res["conv1"]["dense_peak_tflops_at_sampled_clock"] = round(peak / 1e12, 1)
        res["conv1"]["executed_share_of_peak"] = round(executed / c1 / peak, 3)
        res["conv1"]["useful_share_of_peak"] = round(useful / c1 / peak, 3)
    res["igemm"] = {}
    for name, ms, (ex, us) in zip(NAMES[1:], layers[1:], igemm_flops(B, passes)):
        r = {"ms": round(float(ms), 4), "executed_gflop": round(ex / 1e9, 2), "useful_gflop": round(us / 1e9, 2),
             "executed_tflops": round(ex / (ms * 1e-3) / 1e12, 1)}
        if peak:
            r["executed_share_of_peak"] = round(ex / (ms * 1e-3) / peak, 3)
        res["igemm"][name] = r
    ctx.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
