"""GPU diagnostic: the device training step (forward, losses, gradients, SGD) against the CPU training oracle,
tensor by tensor.  Writes the report as JSON.
Usage: python tools/gpu_train_check.py [B [OUT.json]] [--precision bf16|bf16x3]  (defaults 2, train_check.json, bf16)"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "mx-deepim_b200"))

from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.trainer import Trainer  # noqa: E402
from oracle import oracle as O, train_oracle as T  # noqa: E402

K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB


def make_batch(meshes, B, seed):
    obs, ini = synth.sample_pose_pairs(B, seed)
    cls = (np.arange(B) % len(meshes)).astype(np.int32)
    src32, tgt32 = ini.astype(np.float32), obs.astype(np.float32)
    r_obs = [O.render(meshes[cls[b]], obs[b], K, trunc_u8=False) for b in range(B)]
    depth_gt = np.stack([r["depth"] for r in r_obs])[:, None]
    mask_gt = np.stack([r["mask"] for r in r_obs])[:, None]
    upd = O.train_update(meshes, cls, src32, np.tile(np.array([1, 0, 0, 0], np.float32), (B, 1)), np.zeros((B, 3), np.float32),
                         tgt32, depth_gt, K, MEANS)
    img_obs = np.stack([synth.transform_image(synth.composite_observed(r_obs[b]["bgr"], r_obs[b]["mask"], b)) for b in range(B)])
    rng = np.random.default_rng(seed)
    pts, pw = np.zeros((B, 3, 3000), np.float32), np.zeros((B, 3, 3000), np.float32)
    for b in range(B):  # get_point_cloud_model (lib/utils/image.py:452-478): up to 3000 shuffled model points, weight 1
        v = meshes[cls[b]].verts
        keep = rng.permutation(len(v))[:3000]
        pts[b, :, :len(keep)] = v[keep].T
        pw[b, :, :len(keep)] = 1
    pobs = np.stack([tgt32[b, :, :3] @ pts[b] + tgt32[b, :, 3:4] for b in range(B)]).astype(np.float32)
    box = np.stack([O.box_mask(O.mask_bbox(mask_gt[b, 0], 0.0), 480, 640) for b in range(B)])[:, None]
    return dict(image_observed=img_obs, image_rendered=upd["image_rendered"], mask_observed=box, mask_gt_observed=mask_gt,
                mask_rendered=upd["mask_rendered"], src_pose=upd["src_pose"], rot=upd["rot"], trans=upd["trans"], flow=upd["flow"],
                flow_weights=upd["flow_weights"], point_cloud_model=pts, point_cloud_weights=pw, point_cloud_observed=pobs)


def cmp(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    den = max(np.abs(b).max(), 1e-30)
    cos = float(a @ b / max(np.linalg.norm(a) * np.linalg.norm(b), 1e-30))
    return {"max_abs_err": float(np.abs(a - b).max()), "ref_max": float(den), "rel": float(np.abs(a - b).max() / den), "cos": cos}


def main():
    argv = list(sys.argv[1:])
    precision = "bf16"
    if "--precision" in argv:
        i = argv.index("--precision")
        precision = argv[i + 1]
        del argv[i:i + 2]
    B = int(argv[0]) if argv and argv[0].isdigit() else 2
    meshes = [synth.make_cube(), synth.make_blob()]
    w = synth.make_train_weights(0)
    batch = make_batch(meshes, B, 11)
    t0 = time.time()
    out, g, zin, lab = T.forward_backward(w, batch, K, MEANS)
    t_cpu = time.time() - t0
    ctx = Context(0, max_batch=B, max_classes=2, max_verts=6000, max_faces=11000)
    tr = Trainer(ctx, w, precision=precision)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    z = {"zoom_image_observed": dev(zin["zoom_image_observed"]), "zoom_image_rendered": dev(zin["zoom_image_rendered"]),
         "zoom_mask_observed": dev(zin["zoom_mask_observed"]), "zoom_mask_rendered": dev(zin["zoom_mask_rendered"]),
         "zoom_factor": dev(lab["zoom_factor"]), "zoom_flow": dev(lab["zoom_flow"]), "zoom_flow_weights": dev(lab["zoom_flow_weights"]),
         "zoom_mask_gt_observed": dev(lab["zoom_mask_gt_observed"]), "src_pose": dev(lab["src_pose"]),
         "point_cloud_model": dev(lab["point_cloud_model"]), "point_cloud_weights": dev(lab["point_cloud_weights"]),
         "point_cloud_observed": dev(lab["point_cloud_observed"])}
    rep = {"B": B, "precision": precision, "cpu_oracle_s": t_cpu}
    res = tr.forward_backward(z)
    torch.cuda.synchronize()
    losses = res["losses"].cpu().numpy()
    rep["losses"] = {"gpu": losses.tolist(), "oracle": [float(out["flow_loss"].sum()), float(out["point_matching_loss"].sum()),
                                                        None, out["objective"]]}
    fwd = {}
    nhwc = lambda a: np.transpose(a, (0, 2, 3, 1))
    for tid, name in ((0, "flow6"), (1, "flow5"), (2, "flow4"), (3, "mask4")):
        fwd[name] = cmp(tr.debug_tensor(tid), nhwc(out[name]))
    for tid, name, C in ((10, "concat2", 1026), (11, "concat3", 770)):
        buf, (py, px, H, W) = tr.debug_tensor(tid)
        got = buf[:, py:py + H, px:px + W, :]
        ref = nhwc(out[name])
        c_mid = 512
        fwd[name + "_skip"] = cmp(got[..., :c_mid], ref[..., :c_mid])
        fwd[name + "_deconv"] = cmp(got[..., c_mid:C - 2], ref[..., c_mid:C - 2])
        fwd[name + "_flowup"] = cmp(got[..., C - 2:C], ref[..., C - 2:])
        fwd[name + "_pad_absmax"] = float(np.abs(got[..., C:]).max())
    fwd["rot_est_norm"] = cmp(res["rot_est_norm"].cpu().numpy(), out["rot_est_norm"])
    fwd["trans_est"] = cmp(res["trans_est"].cpu().numpy(), out["trans_est"])
    fwd["flow_est"] = cmp(res["flow_est"].cpu().numpy(), out["flow_est"])
    fwd["mask_prob"] = cmp(res["mask_prob"].cpu().numpy(), out["mask_prob"])
    rep["forward"] = fwd
    gd = tr.grads_dict()
    rep["grads"] = {k: cmp(gd[k], g[k]) for k in sorted(gd)}
    dz = {}
    for i, (name, _, _) in enumerate(T.ENC):
        buf, (py, px, H, W) = tr.debug_tensor(20 + i)
        dz[name] = cmp(buf[:, py:py + H, px:px + W, :], nhwc(g["dz_" + name]))
        dz[name]["border_absmax"] = float(max(np.abs(buf[:, 0]).max(), np.abs(buf[:, -1]).max(), np.abs(buf[:, :, 0]).max(),
                                              np.abs(buf[:, :, -1]).max()))
    rep["dz"] = dz
    # one SGD update
    mom = {k: np.zeros_like(v) for k, v in w.items()}
    w2 = {k: v.copy() for k, v in w.items()}
    T.sgd_update(w2, mom, g)
    tr.update()
    torch.cuda.synchronize()
    p2 = tr.get_params()
    rep["sgd"] = {k: cmp(p2[k] - w[k], w2[k] - w[k]) for k in ("conv3_1_weight", "fc6_weight", "deconv5_weight", "rot_bias", "flow_conv1_weight")}
    # timing of forward_backward + update
    for _ in range(2):
        tr.step(z)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        tr.step(z)
    e1.record()
    torch.cuda.synchronize()
    rep["ms_per_step"] = e0.elapsed_time(e1) / 5
    rep["device"] = torch.cuda.get_device_name(0)
    with open(argv[1] if len(argv) > 1 else "train_check.json", "w") as f:
        json.dump(rep, f, indent=1)
    bad = [k for k, v in rep["grads"].items() if v["cos"] < 0.99 and v["ref_max"] > 0]
    print(json.dumps({"losses": rep["losses"], "ms_per_step": rep["ms_per_step"], "bad_grads": bad}, indent=1))
    for sec in ("forward", "dz", "grads", "sgd"):
        print("==", sec)
        for k, v in rep[sec].items():
            print("  %-28s %s" % (k, json.dumps(v) if isinstance(v, dict) else v))


if __name__ == "__main__":
    main()
