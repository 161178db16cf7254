"""End-to-end parity report on a larger sample (config C3-like: 13 meshes, 64 instances, 4 iterations).

    GPU:     python tools/parity_report.py gpu      -> parity_gpu.npz in the current directory (all three precision modes)
    CPU:     python tools/parity_report.py compare  (reads parity_gpu.npz; the oracle runs on the CPU) -> parity_report.json
"""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "mx-deepim_b200"))
import numpy as np
from deepim_b200 import synth

N, N_ITER, SEED = 64, 4, 2
K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB


def inputs():
    meshes = synth.make_linemod_like_set(13, seed=SEED)
    obs, ini = synth.sample_pose_pairs(N, 1234)
    cls = (np.arange(N) % 13).astype(np.int32)
    return meshes, obs, ini, cls


def gpu():
    import torch
    from deepim_b200.refiner import PoseRefiner
    from deepim_b200.context import Context
    meshes, obs, ini, cls = inputs()
    w = synth.make_weights(0)
    dev = torch.device("cuda", 0)
    out = {}
    for prec in ("fp16", "bf16x3", "bf16"):
        r = PoseRefiner(meshes, w, K, device=0, max_batch=16, n_iter=N_ITER, precision=prec, n_slots=2)
        # observed images: GPU render of the observed pose composited over seeded noise (bit-exact vs oracle render)
        u8 = np.zeros((N, 480, 640, 3), np.uint8)
        for a in range(0, N, 16):
            o = r.ctx.render(torch.from_numpy(cls[a:a + 16]).to(dev), torch.from_numpy(obs[a:a + 16].astype(np.float32)).to(dev),
                             K, want=("bgr", "mask"))
            bgr, m = o["bgr"].cpu().numpy(), o["mask"].cpu().numpy()[:, 0]
            for b in range(bgr.shape[0]):
                u8[a + b] = synth.composite_observed(bgr[b], m[b], a + b)
        out["poses_" + prec] = r.refine(u8, cls, ini)
        out["u8_sum"] = np.array([int(u8.astype(np.int64).sum())])
        r.close()
    np.savez_compressed("parity_gpu.npz", **out)
    print("saved", {k: v.shape for k, v in out.items()})


def compare():
    from oracle import oracle as O
    meshes, obs, ini, cls = inputs()
    w = synth.make_weights(0)
    g = np.load("parity_gpu.npz")
    imgs, tot = [], 0
    for b in range(N):
        r = O.render(meshes[cls[b]], obs[b], K)
        u8 = synth.composite_observed(r["bgr"], r["mask"], b)
        tot += int(u8.astype(np.int64).sum())
        imgs.append(synth.transform_image(u8))
    assert tot == int(g["u8_sum"][0]), "observed images differ between GPU render and oracle render"
    ref = np.zeros((N_ITER, N, 3, 4))
    for a in range(0, N, 8):
        res = O.refine(w, meshes, cls[a:a + 8], np.stack(imgs[a:a + 8]), ini[a:a + 8], K, N_ITER, MEANS.astype(np.float32))
        ref[:, a:a + 8] = res["poses"]
        print("oracle", a, flush=True)
    report = {"config": "13 synthetic LINEMOD-scale meshes, %d instances, %d iterations, random-init FlowNetS" % (N, N_ITER),
              "note": "FREE-RUNNING comparison: the CUDA path and the oracle each follow their own pose trajectory, so a difference "
                      "of iteration k moves the integer bbox / zoom of iteration k+1 and compounds (a random-init network is not "
                      "contractive); the north-star tolerance (1e-4 rot / 1e-3 trans on the regressed se3) is per iteration on the "
                      "same inputs and is asserted in tests/test_gpu_headline_b16.py and tests/test_gpu_parity.py"}
    for prec in ("fp16", "bf16x3", "bf16"):
        p = g["poses_" + prec]
        add_g, add_o, acc_g, acc_o = [], [], [], []
        for b in range(N):
            m = meshes[cls[b]]
            pts = m.verts.astype(np.float64)[::4]
            eg = O.add_metric(p[-1, b, :, :3], p[-1, b, :, 3], obs[b, :, :3], obs[b, :, 3], pts)
            eo = O.add_metric(ref[-1, b, :, :3], ref[-1, b, :, 3], obs[b, :, :3], obs[b, :, 3], pts)
            add_g.append(eg / m.diameter); add_o.append(eo / m.diameter)
            acc_g.append(eg < 0.1 * m.diameter); acc_o.append(eo < 0.1 * m.diameter)
        d = np.abs(p - ref)
        report[prec] = {
            "pose_max_abs_diff_per_iter": [float(d[i].max()) for i in range(N_ITER)],
            "pose_median_abs_diff_last_iter": float(np.median(d[-1].reshape(N, -1).max(1))),
            "ADD_over_diameter_mean_gpu": float(np.mean(add_g)), "ADD_over_diameter_mean_oracle": float(np.mean(add_o)),
            "ADD_abs_diff_over_diameter_max": float(np.max(np.abs(np.array(add_g) - np.array(add_o)))),
            "ADD_0.1d_accuracy_pct_gpu": 100.0 * float(np.mean(acc_g)), "ADD_0.1d_accuracy_pct_oracle": 100.0 * float(np.mean(acc_o)),
        }
    json.dump(report, open("parity_report.json", "w"), indent=1)
    print(json.dumps(report, indent=1))


if __name__ == "__main__":
    {"gpu": gpu, "compare": compare}[sys.argv[1]]()
