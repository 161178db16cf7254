"""Training-step benchmark (BASELINE.json config C4: flow+mask+pose losses on synthetic rendered pairs, per-GPU batch 4,
4 inner iterations per batch, NCCL gradient all-reduce when launched under torchrun).

    python tools/train_bench.py [--batch 4] [--steps 10] [--warmup 3] [--precision bf16|bf16x3]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tools/train_bench.py

One "step" = one data batch of Module.fit = 4 x (zoom front, forward, losses, backward, all-reduce, SGD update, re-render
+ labels).  Prints one JSON line (rank 0): training instances/s over all ranks, ms per inner iteration and its split."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "mx-deepim_b200"))

from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.trainer import Trainer, fit_batch, make_device_batch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    ap.add_argument("--bucket-mb", type=float, default=None, help="gradient bucket size of the overlapped all-reduce (default: Trainer's)")
    ap.add_argument("--no-overlap", action="store_true", help="all-reduce after the backward pass instead of bucket by bucket during it")
    ap.add_argument("--precision", default="bf16", choices=["bf16", "bf16x3"], help="precision of the training step (Trainer)")
    a = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    dist = None
    torch.cuda.set_device(local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
    meshes = synth.make_linemod_like_set(13)
    ctx = Context(local, max_batch=a.batch, max_classes=len(meshes), max_verts=max(len(m.verts) for m in meshes),
                  max_faces=max(len(m.faces) for m in meshes))
    for i, m in enumerate(meshes):
        ctx.upload_mesh(i, m)
    tr = Trainer(ctx, synth.make_train_weights(0), precision=a.precision, **({"bucket_mb": a.bucket_mb} if a.bucket_mb else {}))
    batch, cls, tgt, depth = make_device_batch(ctx, meshes, a.batch, 3 + rank, K, MEANS)
    if a.no_overlap:
        step0 = tr.step
        tr.step = lambda z, dist=None, want_maps=False: step0(z, dist=dist, want_maps=want_maps, overlap=False)
    for _ in range(a.warmup):
        fit_batch(tr, batch, cls, tgt, depth, K, dist=dist)
    torch.cuda.synchronize()
    if dist is not None:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        objs = fit_batch(tr, batch, cls, tgt, depth, K, dist=dist)
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1) / a.steps], device="cuda")
    if dist is not None:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    # split of one inner iteration (rank-local, single extra pass)
    z = tr.zoom_front(batch, K)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    torch.cuda.synchronize()
    import time
    c0 = time.perf_counter()
    ev[0].record(); tr.forward_backward(z, want_maps=False); ev[1].record()
    c1 = time.perf_counter()   # host time to ENQUEUE the step (no sync): if it is close to the device time the step is launch-bound
    tr.allreduce(dist); ev[2].record(); tr.update(); ev[3].record()
    c2 = time.perf_counter()
    torch.cuda.synchronize()
    import ctypes
    from deepim_b200._capi import lib as _lib
    ph = (ctypes.c_float * 7)()
    _lib.dim_train_debug_phases(ctx._h, ph)
    line = {"metric": "training instances/s (4 inner updates per instance)", "value": a.batch * world / (float(ms) / 1e3),
            "unit": "instances/s", "n_gpus": world, "steps": a.steps, "warmup": a.warmup, "ms_per_step": float(ms),
            "ms_per_inner_iteration": float(ms) / 4, "split_ms": {"forward_backward": ev[0].elapsed_time(ev[1]),
                                                                   "allreduce": ev[1].elapsed_time(ev[2]), "sgd_update_repack": ev[2].elapsed_time(ev[3]),
                                                                   "host_enqueue_forward_backward": (c1 - c0) * 1e3, "host_enqueue_update": (c2 - c1) * 1e3},
            "dtype": {"bf16": "bf16 activations/gradients, fp32 master",
                      "bf16x3": "bf16 hi/lo activations/gradients (3 MMA passes), fp32 master"}[a.precision],
            "precision": a.precision, "device": torch.cuda.get_device_name(local), "data": "synthetic", "scaling": "weak",
            "config": {"workload": "C4 training step", "allreduce_overlap": (not a.no_overlap) and world > 1, "per_gpu_batch": a.batch, "inner_iterations": 4, "grad_bytes": tr.n * 4,
                       "buckets_mb": [round((hi - lo) * 4 / 2 ** 20, 1) for lo, hi in tr.buckets]},
            "phases_ms": dict(zip(["encoder_fwd", "decoder_fwd", "losses_heads", "fc_bwd", "decoder_bwd", "encoder_dgrad_chain", "wait_wgrad_stream"], [round(float(x), 4) for x in ph])),
            "objective_last_batch": [float(v) for v in objs.cpu()]}
    if rank == 0:
        print(json.dumps(line))
        if a.out:
            with open(a.out, "w") as f:
                json.dump(line, f)
    if dist is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
