"""First-light diagnostics on a real GPU: runs every kernel family once against the oracle and prints
per-stage error summaries (also written to first_light.log in the current directory).  Not a test; see tests/."""
import os, sys, time, traceback
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "mx-deepim_b200"))
import numpy as np
import torch
from oracle import oracle as O
from deepim_b200 import synth
from deepim_b200.context import Context, launch_count
from deepim_b200 import _capi as capi

LOG = open("first_light.log", "w")
def log(*a):
    s = " ".join(str(x) for x in a)
    print(s, flush=True); LOG.write(s + "\n"); LOG.flush()

def stage(name):
    def deco(fn):
        def run(*a, **k):
            log("=== " + name)
            try:
                t = time.time(); r = fn(*a, **k); torch.cuda.synchronize(); log("    ok %.2fs" % (time.time() - t)); return r
            except Exception:
                log("    FAILED\n" + traceback.format_exc()); return None
        return run
    return deco

K = synth.K_LINEMOD
MEANS = synth.PIXEL_MEANS_RGB
dev = torch.device("cuda", 0)
log(torch.cuda.get_device_name(0), torch.version.cuda)
B = int(os.environ.get("FL_B", "2"))
ctx = Context(0, max_batch=max(B, 4))
meshes = [synth.make_cube(), synth.make_blob()]
for i, m in enumerate(meshes): ctx.upload_mesh(i, m)
obs, ini = synth.sample_pose_pairs(B, 0)
cls = np.array([i % 2 for i in range(B)], np.int32)
cls_t = torch.from_numpy(cls).to(dev)

@stage("render")
def t_render():
    pose = torch.from_numpy(ini.astype(np.float32)).to(dev)
    out = ctx.render(cls_t, pose, K, pixel_means_rgb=MEANS, want=("image", "depth", "mask", "bgr"))
    for b in range(B):
        r = O.render(meshes[cls[b]], ini[b], K, means_rgb=MEANS)
        for k in ("image", "depth", "mask", "bgr"):
            g = out[k][b].cpu().numpy().reshape(r[k].shape)
            log("   b%d %-6s mismatches %d maxabs %.3g" % (b, k, int((g != r[k]).sum()), float(np.abs(g - r[k]).max())))
        log("   b%d bbox gpu %s oracle %s" % (b, out["bbox"][b].cpu().numpy(), r["bbox"]))
    return out

@stage("zoom ops")
def t_zoom(rout):
    mr = rout["mask"]; bbox = rout["bbox"]
    mo = ctx.update_mask_box(bbox)
    pose32 = torch.from_numpy(ini.astype(np.float32)).to(dev)
    zo, zg, zr, zf, bb, st = ctx.zoom_mask(mo, mo, mr, pose32, K)
    mo_n, mr_n = mo.cpu().numpy(), mr.cpu().numpy()
    ozo, ozg, ozr, ozf, obb = O.zoom_mask(mo_n, mo_n, mr_n, ini.astype(np.float32), K)
    log("   box mask mismatches", int((mo_n[:, 0] != np.stack([O.box_mask(bbox[b].cpu().numpy(), 480, 640) for b in range(B)])).sum()))
    log("   bbox8 equal", np.array_equal(bb.cpu().numpy(), obb), bb.cpu().numpy().tolist())
    log("   zoom_factor gpu", zf.cpu().numpy().tolist(), "oracle", ozf.tolist(), "bit-equal", np.array_equal(zf.cpu().numpy(), ozf))
    log("   zoomed masks mismatches", int((zo.cpu().numpy() != ozo).sum()), int((zr.cpu().numpy() != ozr).sum()))
    img_o = torch.from_numpy(np.stack([synth.transform_image(synth.composite_observed(
        O.render(meshes[cls[b]], obs[b], K)["bgr"], O.render(meshes[cls[b]], obs[b], K)["mask"], b)) for b in range(B)])).to(dev)
    zio, zir = ctx.zoom_image_with_factor(zf, img_o, rout["image"], MEANS.astype(np.float32))
    ozio, ozir = O.zoom_image_with_factor(ozf, img_o.cpu().numpy(), rout["image"].cpu().numpy(), MEANS.astype(np.float32))
    log("   zoom image mismatches", int((zio.cpu().numpy() != ozio).sum()), int((zir.cpu().numpy() != ozir).sum()),
        "maxabs", float(np.abs(zio.cpu().numpy() - ozio).max()))
    return dict(img_o=img_o, zio=zio, zir=zir, zo=zo, zr=zr, zf=zf)

@stage("se3 / flow")
def t_geom():
    g = np.load(os.path.join(ROOT, "tests/golden/ref_se3.npz"))
    ps = torch.from_numpy(g["pose_src"][:4]).to(dev)
    se3 = torch.from_numpy(np.concatenate([g["quat"][:4], g["trans"][:4]], 1).astype(np.float32)).to(dev)
    c2 = Context.__new__(Context)  # reuse ctx
    out = ctx.se3_compose(ps, se3, (0, 0, 0), (1, 1, 1), "camera").cpu().numpy()
    ref = np.stack([O.rt_transform(g["pose_src"][k], se3[k, :4].cpu().numpy(), se3[k, 4:].cpu().numpy()) for k in range(4)])
    log("   se3 compose maxabs vs oracle %.3g" % np.abs(out - ref).max())

@stage("net (bf16x3) layer by layer")
def t_net(z, precision, tag):
    w = synth.make_weights(0)
    if not getattr(t_net, "loaded", False):
        ctx.load_weights(w); t_net.loaded = True
    rot, trans = ctx.net_forward(z["zio"], z["zir"], z["zo"], z["zr"], precision)
    torch.cuda.synchronize()
    orot, otrans, feats = O.net_forward(w, z["zio"].cpu().numpy(), z["zir"].cpu().numpy(), z["zo"].cpu().numpy(),
                                        z["zr"].cpu().numpy(), return_features=True)
    names = ["flow_conv1", "conv2", "conv3", "conv3_1", "conv4", "conv4_1", "conv5", "conv5_1", "conv6", "conv6_1"]
    for i, n in enumerate(names):
        act, g = ctx.debug_activation(i + 1, B, lo=False)
        if precision == capi.PREC_BF16X3:
            act = act + ctx.debug_activation(i + 1, B, lo=True)[0]
        rows, cols, C_, py, px = g[0], g[1], g[2], g[3], g[4]
        f = feats[n]  # [B,C,H,W]
        Ho, Wo = f.shape[2], f.shape[3]
        inner = act[:, py:py + Ho, px:px + Wo, :].transpose(0, 3, 1, 2)
        err = np.abs(inner - f)
        border = act.copy(); border[:, py:py + Ho, px:px + Wo, :] = 0
        log("   %-10s %s maxabs %.3g  rel %.3g  ref_rms %.3g  border_nonzero %d nan %d" % (
            n, tag, err.max(), err.max() / (np.abs(f).max() + 1e-9), np.sqrt((f ** 2).mean()), int((border != 0).sum()), int(np.isnan(act).sum())))
    log("   rot gpu", rot.cpu().numpy().tolist()); log("   rot ora", orot.tolist())
    log("   trans gpu", trans.cpu().numpy().tolist()); log("   trans ora", otrans.tolist())
    log("   |rot diff| %.3g |trans diff| %.3g" % (np.abs(rot.cpu().numpy() - orot).max(), np.abs(trans.cpu().numpy() - otrans).max()))

@stage("refine loop")
def t_refine(z, precision, tag):
    w = synth.make_weights(0)
    pose0 = torch.from_numpy(ini).to(dev)
    launch_count(True)
    t = time.time()
    res = ctx.refine(z["img_o"], cls_t, pose0, K, 4, pixel_means_rgb=MEANS, precision=precision)
    torch.cuda.synchronize()
    log("   refine %s took %.1f ms, launches %d" % (tag, (time.time() - t) * 1e3, launch_count()))
    ref = O.refine(w, meshes, cls, z["img_o"].cpu().numpy(), ini, K, 4, MEANS.astype(np.float32))
    for it in range(4):
        log("   it%d se3 diff rot %.3g trans %.3g  pose diff %.3g  bbox equal %s zf diff %.3g" % (
            it, np.abs(res["se3"][it].cpu().numpy()[:, :4] - ref["se3"][it][:, :4]).max(),
            np.abs(res["se3"][it].cpu().numpy()[:, 4:] - ref["se3"][it][:, 4:]).max(),
            np.abs(res["poses"][it].cpu().numpy() - ref["poses"][it]).max(),
            np.array_equal(res["bbox"][it].cpu().numpy(), ref["bbox"][it]),
            np.abs(res["zoom_factor"][it].cpu().numpy() - ref["zoom_factor"][it]).max()))

r = t_render()
z = t_zoom(r) if r is not None else None
t_geom()
if z is not None:
    t_net(z, capi.PREC_BF16X3, "x3")
    t_net(z, capi.PREC_BF16, "bf16")
    t_refine(z, capi.PREC_BF16X3, "x3")
    t_refine(z, capi.PREC_BF16, "bf16")
log("done")
