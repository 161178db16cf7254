"""BOP 2019 pose errors per batch: MSSD / MSPD (dim_pose_error_sym) and the VSD in both visibility modes
(dim_pose_error_vsd / dim_pose_error_vsd_ex), with several batches in flight, against the float64 oracle on the host.

    python tools/bop_bench.py [--batches 64] [--slots 2] [--oracle] [--out bop_bench.json]

Device: `slots` contexts on their own streams take the batches round-robin; CUDA events on the launching stream bracket the
whole window (every slot's stream waits for the start event and the end event waits for every slot) -> ms per batch.
Workloads: MSSD / MSPD at M = 16 instances for S in {1, 2, 630} symmetries (identity; a half-turn; a continuous axis
discretised into 315 rotations, combined with the half-turn) and N in {3 000, 30 000} model points; VSD at B = 16 on the C2
mesh with the BOP 2019 taus (10), SIXD 2017 visibility with taus in metres and BOP 2019 visibility with taus relative to the
diameter.  The MSSD / MSPD kernel's float64 rate counts FLOPS_PER_PAIR operations per (point, symmetry) pair (a division
counts as one) over the measured time, against the H100 SXM data sheet's FP64 (non-tensor) peak of 34 TFLOP/s, which counts
a fused multiply-add as two operations (this kernel is compiled with -fmad=false and issues none).
Host (--oracle): oracle/bop.py on the same batch, one instance per process over every host core.
The GPU's name and power limit are printed beside the numbers."""
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

from deepim_b200 import bop, pose_eval, synth  # noqa: E402
from icp_bench import gpu_info  # noqa: E402
from oracle import bop as OB  # noqa: E402
from vsd_bench import make_batch  # noqa: E402

K = synth.K_LINEMOD
M = 16
# per (point, symmetry) pair: T_gs p (9 mul, 9 add), the 3-D difference and its square (3 sub, 3 mul, 2 add), the projection
# (9 mul, 6 add, 2 div), the 2-D difference and its square (2 sub, 2 mul, 1 add)
FLOPS_PER_PAIR = 48
FP64_PEAK = 34e12
DIAM = 0.1


def sym_sets():
    flip = np.diag([-1.0, -1.0, 1.0, 1.0])
    cont = {"axis": [0.0, 0.0, 1.0], "offset": np.zeros(3)}
    return {1: np.eye(3, 4)[None], 2: bop.symmetry_transforms({"symmetries_discrete": [flip]}),
            630: bop.symmetry_transforms({"symmetries_discrete": [flip], "symmetries_continuous": [cont]})}


def _sym_oracle(args):
    est, gt, pts, syms = args
    return OB.mssd_mspd(est[None], gt[None], pts, syms, K)[0][0]


_MESH = None


def _vsd_oracle(args):
    global _MESH
    if _MESH is None:
        _MESH = synth.make_blob()
    est, gt, depth, mode, diam = args
    return OB.vsd([_MESH], [0], est[None], gt[None], depth[None], K, pose_eval.BOP19_VSD_DELTA, pose_eval.BOP19_VSD_TAUS,
                  visib_mode=mode, diameters=None if diam is None else [diam])[0][0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=64)
    ap.add_argument("--slots", type=int, default=2)
    ap.add_argument("--oracle", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from deepim_b200.context import Context
    assert torch.cuda.is_available(), "bop_bench measures the device: it needs a GPU"
    dev = torch.device("cuda", 0)
    mesh = synth.make_blob()
    rng = np.random.default_rng(3)
    depth, est, gt = make_batch(mesh, M, 5)
    from test_icp_oracle import perturb
    est_sym = np.stack([perturb(g, rng, t=0.02, deg=20.0) for g in gt])
    pts = {3000: rng.uniform(-0.05, 0.05, (3000, 3)), 30000: rng.uniform(-0.05, 0.05, (30000, 3))}
    syms = sym_sets()
    slots = []
    for _ in range(a.slots):
        ctx = Context(0, max_batch=M, max_classes=1, max_verts=len(mesh.verts), max_faces=len(mesh.faces))
        ctx.upload_mesh(0, mesh)
        slots.append((ctx, torch.cuda.Stream(device=dev)))
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    d_depth, d_cls, d_est, d_gt, d_est_sym = t(depth), t(np.zeros(M, np.int32)), t(est), t(gt), t(est_sym)
    d_pts, d_syms = {n: t(v) for n, v in pts.items()}, {s: t(v) for s, v in syms.items()}
    d_K = t(np.broadcast_to(K.astype(np.float64), (M, 3, 3)))
    diam = np.full(M, DIAM)

    def timed(fn):
        """ms per batch of fn(ctx) over a.batches calls round-robin over the slots, and the last result"""
        main_st = torch.cuda.current_stream(dev)
        for i in range(2 * len(slots)):  # warm-up
            with torch.cuda.stream(slots[i % len(slots)][1]):
                fn(slots[i % len(slots)][0])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(main_st)
        for _, st in slots:
            st.wait_event(e0)
        r = None
        for i in range(a.batches):
            ctx, st = slots[i % len(slots)]
            with torch.cuda.stream(st):
                r = fn(ctx)
        for _, st in slots:
            main_st.wait_stream(st)
        e1.record(main_st)
        e1.synchronize()
        return e0.elapsed_time(e1) / a.batches, r

    res = {"tool": "bop_bench", "batches": a.batches, "slots": a.slots, "sym": [], "vsd": []}
    pool = ProcessPoolExecutor(os.cpu_count()) if a.oracle else None
    for n in (3000, 30000):
        for S in (1, 2, 630):
            ms, r = timed(lambda ctx: ctx.pose_error_sym(d_est_sym, d_gt, d_pts[n], d_syms[S], d_K))
            row = {"M": M, "N": n, "S": S, "ms_per_batch": round(ms, 4),
                   "fp64_gflops": round(FLOPS_PER_PAIR * M * n * S / (ms * 1e-3) / 1e9, 1),
                   "fp64_peak_share": round(FLOPS_PER_PAIR * M * n * S / (ms * 1e-3) / FP64_PEAK, 4)}
            if pool:
                t0 = time.perf_counter()
                ref = np.stack(list(pool.map(_sym_oracle, [(est_sym[m], gt[m], pts[n], syms[S]) for m in range(M)])))
                row["oracle_ms_per_batch"] = round((time.perf_counter() - t0) * 1e3, 1)
                row["equals_oracle"] = bool(np.array_equal(r["err"].cpu().numpy(), ref))
            res["sym"].append(row)
    for mode, dm in (("sixd17", None), ("bop19", diam)):
        ms, r = timed(lambda ctx: ctx.pose_error_vsd(d_depth, d_cls, d_est, d_gt, K, pose_eval.BOP19_VSD_DELTA,
                                                     pose_eval.BOP19_VSD_TAUS, visib_mode=mode, diameters=dm))
        row = {"B": M, "visib_mode": mode, "relative_taus": dm is not None, "n_tau": len(pose_eval.BOP19_VSD_TAUS),
               "ms_per_batch": round(ms, 4)}
        if pool:
            t0 = time.perf_counter()
            ref = np.stack(list(pool.map(_vsd_oracle, [(est[b], gt[b], depth[b], mode, None if dm is None else DIAM)
                                                       for b in range(M)])))
            row["oracle_ms_per_batch"] = round((time.perf_counter() - t0) * 1e3, 1)
            row["equals_oracle"] = bool(np.array_equal(r["err"].cpu().numpy(), ref))
        res["vsd"].append(row)
    if pool:
        pool.shutdown()
        res["host_cores"] = os.cpu_count()
    res["gpu"], res["power_limit"] = gpu_info()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    for ctx, _ in slots:
        ctx.close()


if __name__ == "__main__":
    main()
