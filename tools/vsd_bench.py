"""VSD cost per batch (dim_pose_error_vsd): the C2 mesh, B = 16 instances, 10 tau values, several batches in flight.

    python tools/vsd_bench.py [--batches 256] [--slots 2] [--oracle-batches 1] [--out vsd_bench.json]

Device: `slots` contexts on their own streams take the batches round-robin, timed by a host clock around work that ends in
a device synchronise -> ms per batch.  The split into the two renders and the VSD pass comes from a separate pass with stage
profiling on (CUDA events around the two parts of each call).  Host: the oracle (oracle/vsd.py, float64 numpy) on the same
batch, one instance per process over every host core.  The GPU's name and power limit are printed beside the numbers."""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "mx-deepim_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from deepim_b200 import synth  # noqa: E402
from icp_bench import gpu_info  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle import vsd as V  # noqa: E402

K = synth.K_LINEMOD
DELTA = 0.015
TAUS = tuple(np.linspace(0.005, 0.05, 10))


def make_batch(mesh, B, seed):
    """observed depth at sampled poses (mm-quantised), estimates 1 cm / 3 deg away"""
    from test_icp_oracle import mm, perturb
    rng = np.random.default_rng(seed)
    gt = synth.sample_pose_pairs(B, seed)[0]
    depth = np.stack([mm(O.render(mesh, gt[b], K, want=("depth",))["depth"]) for b in range(B)])
    return depth, np.stack([perturb(gt[b], rng) for b in range(B)]), gt


_MESH = None


def _oracle_one(args):
    global _MESH
    if _MESH is None:
        _MESH = synth.make_blob()
    est, gt, depth = args
    return V.vsd([_MESH], [0], est[None], gt[None], depth[None], K, DELTA, TAUS)[0][0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--batches", type=int, default=256)
    ap.add_argument("--slots", type=int, default=2)
    ap.add_argument("--oracle-batches", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from deepim_b200.context import Context
    assert torch.cuda.is_available(), "vsd_bench measures the device: it needs a GPU"
    mesh = synth.make_blob()
    B = a.batch
    depth, est, gt = make_batch(mesh, B, 5)
    dev = torch.device("cuda", 0)
    slots = []
    for _ in range(a.slots):
        ctx = Context(0, max_batch=B, max_classes=1, max_verts=len(mesh.verts), max_faces=len(mesh.faces))
        ctx.upload_mesh(0, mesh)
        slots.append((ctx, torch.cuda.Stream(device=dev), torch.from_numpy(depth).to(dev),
                      torch.zeros(B, dtype=torch.int32, device=dev), torch.from_numpy(est).to(dev),
                      torch.from_numpy(gt).to(dev)))

    def enqueue(n):
        for i in range(n):
            ctx, st, d, c, pe, pg = slots[i % len(slots)]
            with torch.cuda.stream(st):
                ctx.pose_error_vsd(d, c, pe, pg, K, DELTA, TAUS)

    enqueue(2 * len(slots))  # warm-up: module load, first launches
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    enqueue(a.batches)
    torch.cuda.synchronize()
    ms_batch = (time.perf_counter() - t0) * 1e3 / a.batches
    # stage split: profiling on, one slot, calls in sequence
    ctx, st, d, c, pe, pg = slots[0]
    ctx.profile_enable(True)
    with torch.cuda.stream(st):
        for _ in range(a.batches):
            r = ctx.pose_error_vsd(d, c, pe, pg, K, DELTA, TAUS)
    stages, n = ctx.profile_read()
    ctx.profile_enable(False)
    ms_render, ms_pass = stages["render"] / n, stages["zoom"] / n
    err = r["err"].cpu().numpy()
    # host: the oracle on the same batch, every core
    t0 = time.perf_counter()
    with ProcessPoolExecutor(os.cpu_count()) as pool:
        for _ in range(a.oracle_batches):
            ref = np.stack(list(pool.map(_oracle_one, [(est[b], gt[b], depth[b]) for b in range(B)])))
    ms_oracle = (time.perf_counter() - t0) * 1e3 / a.oracle_batches
    name, power = gpu_info()
    res = {"tool": "vsd_bench", "gpu": name, "power_limit": power, "workload": "C2 mesh (%d verts), B = %d, %d taus, "
           "%d batches over %d contexts / streams" % (len(mesh.verts), B, len(TAUS), a.batches, a.slots),
           "ms_per_batch": round(ms_batch, 4), "ms_render": round(ms_render, 4), "ms_vsd_pass": round(ms_pass, 4),
           "oracle_ms_per_batch": round(ms_oracle, 1), "host_cores": os.cpu_count(),
           "err_equals_oracle": bool(np.array_equal(err, ref)), "mean_err": [round(float(v), 4) for v in err.mean(0)]}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    for s in slots:
        s[0].close()


if __name__ == "__main__":
    main()
