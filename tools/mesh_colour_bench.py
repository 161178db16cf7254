"""Vertex-coloured meshes against textured ones: what the colour source costs in the render and in the refinement loop, and
bench.py's flagship rate on this build against another build of the project.

    python tools/mesh_colour_bench.py [--rounds 3] [--iters 200] [--parent DIR] [--bench-steps 20] [--bench-warmup 3] [--out FILE]

C2 inputs: the 5k-vertex blob textured (its own 256 x 256 texture) and the same blob with vertex colours (seeded, in
[0, 1]), each on its own context, B = 16 random poses, 480 x 640.  `rounds` times, alternating textured / coloured on the
same inputs:
  render   device ms per dim_render of B = 16 (image, depth, mask, bbox; test path), CUDA events around `iters` calls
  refine   refinements/s of the fused loop (dim_refine, 4 iterations, fp16, random-init weights, B = 16), CUDA events
           around `iters` / 10 calls (graph replay)
The best round of each is reported, with the coloured / textured ratios.  With --parent DIR (a built checkout of another
commit), bench.py --gpus 1 is run from DIR and from this tree alternately, `rounds` times each, and each run's JSON line is
reported with the spread.  The card's name and power limit are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "mx-deepim_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from variant_bench import card  # noqa: E402

B, N_ITER = 16, 4
K = synth.K_LINEMOD


def coloured(mesh, seed=7):
    c = np.random.RandomState(seed).uniform(0, 1, (len(mesh.verts), 3)).astype(np.float32)
    return synth.Mesh(mesh.verts, None, mesh.faces, None, mesh.name + "+colours", colours=c)


def timed(fn, n):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(n):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / n


def arms(iters):
    tex = synth.make_blob()
    meshes = {"textured": tex, "coloured": coloured(tex)}
    w = synth.make_weights(0)
    obs, ini = synth.sample_pose_pairs(B, 3)
    img = torch.from_numpy(np.stack([synth.transform_image(synth.composite_observed(
        np.zeros((480, 640, 3), np.float32), np.zeros((480, 640), np.float32), b)) for b in range(B)])).cuda()
    cls = torch.zeros(B, dtype=torch.int32, device="cuda")
    pose = torch.from_numpy(obs.astype(np.float32)).cuda()
    ini_d = torch.from_numpy(ini).cuda()
    out = {}
    for name, m in meshes.items():
        ctx = Context(0, max_batch=B, max_classes=1, max_verts=6000, max_faces=11000)
        ctx.upload_mesh(0, m)
        ctx.load_weights(w)
        state = {"r": None, "o": None}

        def render(ctx=ctx, state=state):
            state["r"] = ctx.render(cls, pose, K, pixel_means_rgb=synth.PIXEL_MEANS_RGB, want=("image", "depth", "mask"))

        def refine(ctx=ctx, state=state):
            state["o"] = ctx.refine(img, cls, ini_d, K, N_ITER, pixel_means_rgb=synth.PIXEL_MEANS_RGB, out=state["o"])

        for _ in range(3):
            render()
            refine()
        torch.cuda.synchronize()
        out[name] = (ctx, render, refine)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--parent", default=None, help="a built checkout of another commit to run bench.py from")
    ap.add_argument("--bench-steps", type=int, default=20)
    ap.add_argument("--bench-warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "mesh_colour_bench needs a GPU"
    res = {"card": card(), "B": B, "n_iter": N_ITER, "render_ms": {}, "refine_per_s": {}}
    a = arms(args.iters)
    for _ in range(args.rounds):
        for name, (ctx, render, refine) in a.items():
            res["render_ms"].setdefault(name, []).append(timed(render, args.iters))
            res["refine_per_s"].setdefault(name, []).append(B * 1000.0 / timed(refine, max(args.iters // 10, 5)))
    for name, (ctx, _, _) in a.items():
        ctx.close()
    best = {"render_ms": {k: min(v) for k, v in res["render_ms"].items()},
            "refine_per_s": {k: max(v) for k, v in res["refine_per_s"].items()}}
    res["best"] = best
    res["ratio_coloured_over_textured"] = {"render_ms": best["render_ms"]["coloured"] / best["render_ms"]["textured"],
                                           "refine_per_s": best["refine_per_s"]["coloured"] / best["refine_per_s"]["textured"]}
    if args.parent:
        runs = {"parent": [], "this": []}
        for _ in range(args.rounds):
            for name, tree in (("parent", os.path.abspath(args.parent)), ("this", ROOT)):
                p = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps",
                                    str(args.bench_steps), "--warmup", str(args.bench_warmup)], cwd=tree, capture_output=True,
                                   text=True, check=True)
                runs[name].append(json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("{")][-1]))
        res["bench"] = runs
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
