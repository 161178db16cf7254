"""ICP cost per batch (dim_icp): the C2 mesh, B = 16 instances, 10 iterations, several batches in flight.

    python tools/icp_bench.py [--batches 64] [--slots 2] [--iters 10] [--oracle-batches 1] [--out icp_bench.json]

Device: `slots` contexts on their own streams take the batches round-robin, timed by a host clock around work that ends in
a device synchronise -> ms per batch.  The split into render and association + solve comes from a separate pass with stage
profiling on (CUDA events around the two parts of each call).  Host: the oracle (oracle/icp.py, float64 numpy) on the same
batch, one instance per process over every host core.  The GPU's name and power limit are printed beside the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "mx-deepim_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from deepim_b200 import synth  # noqa: E402
from oracle import icp as I  # noqa: E402
from oracle import oracle as O  # noqa: E402

K = synth.K_LINEMOD


def make_batch(mesh, B, seed):
    """observed depth at sampled poses (mm-quantised), initial poses 1 cm / 3 deg away"""
    from test_icp_oracle import mm, perturb
    rng = np.random.default_rng(seed)
    gt = synth.sample_pose_pairs(B, seed)[0]
    depth = np.stack([mm(O.render(mesh, gt[b], K, want=("depth",))["depth"]) for b in range(B)])
    return depth, np.stack([perturb(gt[b], rng) for b in range(B)])


_MESH = None


def _oracle_one(args):
    global _MESH
    if _MESH is None:
        _MESH = synth.make_blob()
    P0, depth, iters = args
    return I.icp([_MESH], [0], P0[None], depth[None], K, iters)["poses"]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:  # the numbers stay, the label says why it is missing
        import torch
        return torch.cuda.get_device_name(0), "unknown (%s)" % type(e).__name__


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--batches", type=int, default=64)
    ap.add_argument("--slots", type=int, default=2)
    ap.add_argument("--oracle-batches", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from deepim_b200.context import Context
    assert torch.cuda.is_available(), "icp_bench measures the device: it needs a GPU"
    mesh = synth.make_blob()
    B = a.batch
    depth, P0 = make_batch(mesh, B, 5)
    dev = torch.device("cuda", 0)
    slots = []
    for _ in range(a.slots):
        ctx = Context(0, max_batch=B, max_classes=1, max_verts=len(mesh.verts), max_faces=len(mesh.faces))
        ctx.upload_mesh(0, mesh)
        slots.append((ctx, torch.cuda.Stream(device=dev), torch.from_numpy(depth).to(dev),
                      torch.zeros(B, dtype=torch.int32, device=dev), torch.from_numpy(P0).to(dev)))

    def enqueue(n):
        for i in range(n):
            ctx, st, d, c, p = slots[i % len(slots)]
            with torch.cuda.stream(st):
                ctx.icp(d, c, p, K, a.iters)

    enqueue(2 * len(slots))  # warm-up: module load, first launches
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    enqueue(a.batches)
    torch.cuda.synchronize()
    ms_batch = (time.perf_counter() - t0) * 1e3 / a.batches
    # stage split: profiling on, one slot, calls in sequence
    ctx, st, d, c, p = slots[0]
    ctx.profile_enable(True)
    with torch.cuda.stream(st):
        for _ in range(a.batches):
            r = ctx.icp(d, c, p, K, a.iters)
    stages, n = ctx.profile_read()
    ctx.profile_enable(False)
    ms_render, ms_icp = stages["render"] / n, stages["zoom"] / n
    status = r["status"].cpu().numpy()
    # host: the oracle on the same batch, every core
    t0 = time.perf_counter()
    with ProcessPoolExecutor(os.cpu_count()) as pool:
        for _ in range(a.oracle_batches):
            ref = np.stack(list(pool.map(_oracle_one, [(P0[b], depth[b], a.iters) for b in range(B)])))[:, :, 0]
    ms_oracle = (time.perf_counter() - t0) * 1e3 / a.oracle_batches
    ref = np.moveaxis(ref, 0, 1)
    name, power = gpu_info()
    res = {"tool": "icp_bench", "gpu": name, "power_limit": power, "workload": "C2 mesh (%d verts), B = %d, %d iterations, "
           "%d batches over %d contexts / streams" % (len(mesh.verts), B, a.iters, a.batches, a.slots),
           "ms_per_batch": round(ms_batch, 4), "ms_render": round(ms_render, 4), "ms_assoc_solve": round(ms_icp, 4),
           "oracle_ms_per_batch": round(ms_oracle, 1), "host_cores": os.cpu_count(),
           "max_abs_pose_diff_vs_oracle": float(np.abs(r["poses"].cpu().numpy()[-1] - ref[-1]).max()),
           "nonzero_status": int(np.count_nonzero(status))}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    for s in slots:
        s[0].close()


if __name__ == "__main__":
    main()
