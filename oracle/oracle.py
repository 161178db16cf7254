"""CPU ORACLE (TEST INFRASTRUCTURE ONLY).

Python face of the oracle: ctypes bindings of oracle/liboracle.so (the C restatement in
deepim_oracle.c), the FlowNetS forward in torch-CPU fp32 and the test-time iteration glue.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may
import this module.  The product package never does (tests/test_no_oracle_in_product.py).

The network variants are arguments, as on the device: the lit render of the ModelNet branch (`lighting`), the RGB-D
network (the depths) and the image-only network (no masks).  The light and depth helpers restate the reference
independently of the product's deepim_b200.lighting; tests/test_lighting.py compares the two.

Reference anchors:
  net            deepim/symbols/deepIM_flownet.py:32-118 (get_convs), 715-726 (heads)
  iteration glue deepim/core/tester.py:340-485, lib/pair_matching/data_pair.py:66-129,
                 lib/utils/image.py:583-594
  lit render     deepim/core/tester.py:146-188, lib/pair_matching/batch_updater_py_multi.py:187-235
  ADD / ADI      lib/utils/pose_error.py:72-108
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")


def build(force: bool = False) -> str:
    so = os.path.join(_HERE, "liboracle.so")
    src = os.path.join(_HERE, "deepim_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        vp = C.c_void_p
        L.orc_render.argtypes = [f32p, f32p, C.c_int32, i32p, C.c_int32, u8p, C.c_int32, C.c_int32, f32p, f32p,
                                 C.c_float, C.c_float, C.c_int32, C.c_int32, f64p, C.c_int32, vp, vp, vp, vp, vp]
        L.orc_render.restype = None
        L.orc_render_lit.argtypes = [f32p, f32p, f32p, C.c_int32, i32p, C.c_int32, u8p, C.c_int32, C.c_int32, f32p, f32p,
                                     C.c_float, C.c_float, C.c_int32, C.c_int32, f64p, f32p, f32p, C.c_float, C.c_float,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_render_lit.restype = None
        L.orc_mask_bbox.argtypes = [f32p, C.c_int32, C.c_int32, C.c_float, i32p]
        L.orc_zoom_factor.argtypes = [i32p, i32p, f32p, f32p, C.c_int32, C.c_int32, f32p]
        L.orc_zoom_factor.restype = C.c_int32
        L.orc_zoom_plane.argtypes = [f32p, f32p, C.c_int32, C.c_int32, f32p, C.c_int32, C.c_float]
        L.orc_inv_zoom_affine.argtypes = [f32p, C.c_int32, C.c_int32, f32p]
        L.orc_box_mask.argtypes = [i32p, C.c_int32, C.c_int32, f32p]
        L.orc_zoom_trans.argtypes = [f32p, f32p, C.c_int32, C.c_int32, f32p]
        L.orc_rt_transform.argtypes = [f64p, f64p, f64p, f64p, f64p, C.c_int32, f64p]
        L.orc_rt_delta.argtypes = [f64p, f64p, f64p, f64p, C.c_int32, f64p, f64p]
        L.orc_flow.argtypes = [f32p, f32p, f32p, f32p, C.c_int32, C.c_int32, C.c_int32, f32p, f32p]
        _LIB = L
    return _LIB


ROT_COORD = {"model": 0, "camera": 1, "camera_new": 2}
# FlowNetS encoder (deepIM_flownet.py:32-105): name, stride, padding
ENC = [("flow_conv1", 2, 3), ("conv2", 2, 2), ("conv3", 2, 2), ("conv3_1", 1, 1), ("conv4", 2, 1),
       ("conv4_1", 1, 1), ("conv5", 2, 1), ("conv5_1", 1, 1), ("conv6", 2, 1), ("conv6_1", 1, 1)]
# the ModelNet branch's light: offset of light index 2 and Render_Py_Light_ModelNet_Multi's brightness ratio
OFFSET = (0.0, 0.5, 0.5)
BRIGHTNESS_RATIO = 0.7


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def k4(K):
    K = np.asarray(K, dtype=np.float32)
    return np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], dtype=np.float32)


# ------------------------------------------------------------------------------------------ render
def render(mesh, pose, K, zn=0.25, zf=6.0, H=480, W=640, means_rgb=None, trunc_u8=True,
           want=("bgr", "depth", "image", "mask")):
    """One instance.  Returns dict with bgr [H,W,3], depth [H,W], image [3,H,W], mask [H,W], bbox[4]."""
    pose32 = np.ascontiguousarray(pose, dtype=np.float32)
    means = np.zeros(3, np.float64) if means_rgb is None else np.ascontiguousarray(means_rgb, dtype=np.float64)
    out = {
        "bgr": np.empty((H, W, 3), np.float32) if "bgr" in want else None,
        "depth": np.empty((H, W), np.float32) if "depth" in want else None,
        "image": np.empty((3, H, W), np.float32) if "image" in want else None,
        "mask": np.empty((H, W), np.float32) if "mask" in want else None,
    }
    bbox = np.zeros(4, np.int32)
    lib().orc_render(mesh.verts, mesh.uvs, len(mesh.verts), mesh.faces, len(mesh.faces), mesh.tex,
                     mesh.tex.shape[0], mesh.tex.shape[1], pose32, k4(K), zn, zf, H, W, means, int(trunc_u8),
                     _ptr(out["bgr"]), _ptr(out["depth"]), _ptr(out["image"]), _ptr(out["mask"]), _ptr(bbox))
    out["bbox"] = bbox
    return out


def render_lit(mesh, normals, pose, K, light_position, light_intensity, brightness_ratio=0.7, zn=0.25, zf=6.0, H=480, W=640,
               means_rgb=None, want=("bgr", "depth", "image", "mask")):
    """Render_Py_Light_ModelNet_Multi.render (lib/render_glumpy/render_py_light_modelnet_multi.py:131-175): Lambert-lit
    textured render; light position in the GL camera frame, bgr holds the 8-bit quantised colours as floats."""
    pose32 = np.ascontiguousarray(pose, dtype=np.float32)
    means = np.zeros(3, np.float64) if means_rgb is None else np.ascontiguousarray(means_rgb, dtype=np.float64)
    out = {
        "bgr": np.empty((H, W, 3), np.float32) if "bgr" in want else None,
        "depth": np.empty((H, W), np.float32) if "depth" in want else None,
        "image": np.empty((3, H, W), np.float32) if "image" in want else None,
        "mask": np.empty((H, W), np.float32) if "mask" in want else None,
    }
    bbox = np.zeros(4, np.int32)
    lib().orc_render_lit(mesh.verts, mesh.uvs, np.ascontiguousarray(normals, np.float32), len(mesh.verts), mesh.faces,
                         len(mesh.faces), mesh.tex, mesh.tex.shape[0], mesh.tex.shape[1], pose32, k4(K), zn, zf, H, W, means,
                         np.ascontiguousarray(light_position, np.float32), np.ascontiguousarray(light_intensity, np.float32),
                         float(np.float32(1.0 - float(np.float32(brightness_ratio)))), float(np.float32(brightness_ratio)),
                         _ptr(out["bgr"]), _ptr(out["depth"]), _ptr(out["image"]), _ptr(out["mask"]), _ptr(bbox))
    out["bbox"] = bbox
    return out


def light_position(pose, offset=OFFSET):
    """The light of the ModelNet branch's renders (tester.py:146-160) on the float64 pose being rendered, cast to float32
    at the end like the glumpy uniform:
        light_position = np.array([0, 1, 1]) * 0.5
        light_position[0] += pose[0, 3]; light_position[1] -= pose[1, 3]; light_position[2] -= pose[2, 3]"""
    light = np.array(offset, dtype=np.float64)
    pose = np.asarray(pose, dtype=np.float64)
    light[0] += pose[0, 3]
    light[1] -= pose[1, 3]
    light[2] -= pose[2, 3]
    return light.astype(np.float32)


def _render_lit(mesh, pose, K, intensity, lighting, zn, zf, H, W, means_rgb, want):
    """render_lit at the light of `pose`; lighting = {"offset", "brightness_ratio"} (defaults OFFSET, BRIGHTNESS_RATIO),
    the mesh carries `normals`."""
    return render_lit(mesh, mesh.normals, pose, K, light_position(pose, lighting.get("offset", OFFSET)), intensity,
                      lighting.get("brightness_ratio", BRIGHTNESS_RATIO), zn, zf, H, W, means_rgb, want)


def depth_from_u16(u16, depth_factor=1000.0):
    """lib/utils/image.py:203,218: a float32 array divided by a Python float stays float32 (float32-rounded factor)."""
    return np.asarray(u16).astype(np.float32) / depth_factor


# -------------------------------------------------------------------------------------------- zoom
def mask_bbox(mask, thresh):
    m = np.ascontiguousarray(mask, dtype=np.float32).reshape(mask.shape[-2], mask.shape[-1])
    bbox = np.zeros(4, np.int32)
    lib().orc_mask_bbox(m, m.shape[0], m.shape[1], thresh, bbox)
    return bbox


def zoom_plane(src, affine, mode, param=0.0):
    src = np.ascontiguousarray(src, dtype=np.float32)
    dst = np.empty_like(src)
    lib().orc_zoom_plane(src, dst, src.shape[0], src.shape[1], np.ascontiguousarray(affine, dtype=np.float32),
                         mode, param)
    return dst


def zoom_mask(mask_observed, mask_gt_observed, mask_rendered, src_pose, K):
    """ZoomMask forward (deepim/operator_py/zoom_mask.py:29-112) on (B,1,H,W) float32 arrays.
    Returns zoom_mask_observed, zoom_mask_gt_observed, zoom_mask_rendered, zoom_factor(B,4), bbox(B,8)
    where bbox = real x0,x1,y0,y1, rendered x0,x1,y0,y1 (-1 if empty)."""
    B, _, H, W = mask_observed.shape
    K9 = np.ascontiguousarray(K, dtype=np.float32).reshape(9)
    outs = [np.empty_like(mask_observed, dtype=np.float32) for _ in range(3)]
    zf = np.zeros((B, 4), np.float32)
    bboxes = np.zeros((B, 8), np.int32)
    for b in range(B):
        bb_real = mask_bbox(mask_gt_observed[b].sum(axis=0), 0.3)
        ren_bin = (mask_rendered[b] > 0.2).astype(np.float32)
        bb_ren = mask_bbox(ren_bin.sum(axis=0), 0.3)
        sp = np.ascontiguousarray(src_pose[b], dtype=np.float32)
        z = np.zeros(4, np.float32)
        rc = lib().orc_zoom_factor(bb_real, bb_ren, sp, K9, H, W, z)
        if rc != 0:
            raise ValueError("zoom_mask: observed mask empty (the reference raises here as well)")
        zf[b] = z
        bboxes[b, :4], bboxes[b, 4:] = bb_real, bb_ren
        outs[0][b, 0] = zoom_plane(mask_observed[b, 0], z, 1)
        outs[1][b, 0] = zoom_plane(mask_gt_observed[b, 0], z, 1)
        outs[2][b, 0] = zoom_plane(ren_bin[0], z, 1)
    return outs[0], outs[1], outs[2], zf, bboxes


def zoom_image(image_observed, image_rendered, src_pose, K, means_rgb):
    """ZoomImage forward (deepim/operator_py/zoom_image.py:26-107): boxes from sum_c(image + mean) > 0.01 (float32 adds
    in channel order, as np.sum over 3 non-contiguous elements), then the ZoomMask centre/crop rule and the
    ZoomImageWithFactor sampling.  Returns zoom_image_observed, zoom_image_rendered, zoom_factor, bbox(B,8)."""
    B, _, H, W = image_observed.shape
    K9 = np.ascontiguousarray(K, dtype=np.float32).reshape(9)
    m = np.asarray(means_rgb, np.float32)
    zf = np.zeros((B, 4), np.float32)
    bboxes = np.zeros((B, 8), np.int32)
    for b in range(B):
        so = ((image_observed[b, 0] + m[0]) + (image_observed[b, 1] + m[1])) + (image_observed[b, 2] + m[2])
        sr = ((image_rendered[b, 0] + m[0]) + (image_rendered[b, 1] + m[1])) + (image_rendered[b, 2] + m[2])
        bb_real, bb_ren = mask_bbox(so.astype(np.float32), 0.01), mask_bbox(sr.astype(np.float32), 0.01)
        z = np.zeros(4, np.float32)
        if lib().orc_zoom_factor(bb_real, bb_ren, np.ascontiguousarray(src_pose[b], dtype=np.float32), K9, H, W, z) != 0:
            raise ValueError("zoom_image: observed image empty (the reference raises here as well)")
        zf[b] = z
        bboxes[b, :4], bboxes[b, 4:] = bb_real, bb_ren
    o, r = zoom_image_with_factor(zf, image_observed, image_rendered, m)
    return o, r, zf, bboxes


def zoom_image_with_factor(zoom_factor, image_observed, image_rendered, means_rgb):
    """ZoomImageWithFactor forward (zoom_image_with_factor.py:31-65); means_rgb = reversed pixel_means."""
    B = image_observed.shape[0]
    o = np.empty_like(image_observed, dtype=np.float32)
    r = np.empty_like(image_rendered, dtype=np.float32)
    for b in range(B):
        for c in range(3):
            o[b, c] = zoom_plane(image_observed[b, c], zoom_factor[b], 3, float(means_rgb[c]))
            r[b, c] = zoom_plane(image_rendered[b, c], zoom_factor[b], 3, float(means_rgb[c]))
    return o, r


def inv_zoom_affine(zf, H, W):
    a = np.zeros(4, np.float32)
    lib().orc_inv_zoom_affine(np.ascontiguousarray(zf, dtype=np.float32), H, W, a)
    return a


def zoom_mask_with_factor(zoom_factor, mask, b_inv_zoom):
    """ZoomMaskWithFactor (zoom_mask_with_factor.py:29-64)."""
    B, _, H, W = mask.shape
    out = np.empty_like(mask, dtype=np.float32)
    for b in range(B):
        aff = inv_zoom_affine(zoom_factor[b], H, W) if b_inv_zoom else zoom_factor[b]
        out[b, 0] = zoom_plane(mask[b, 0], aff, 2)
    return out


def zoom_flow(zoom_factor, flow, flow_weights=None, b_inv_zoom=False):
    """ZoomFlow (zoom_flow.py:28-71)."""
    B, _, H, W = flow.shape
    out = np.empty_like(flow, dtype=np.float32)
    outw = None if (b_inv_zoom or flow_weights is None) else np.empty_like(flow_weights, dtype=np.float32)
    for b in range(B):
        aff = inv_zoom_affine(zoom_factor[b], H, W) if b_inv_zoom else zoom_factor[b]
        wx = np.float32(zoom_factor[b, 0])
        for c in range(2):
            s = zoom_plane(flow[b, c], aff, 0)
            out[b, c] = s * wx if b_inv_zoom else s / wx
        if outw is not None:
            for c in range(flow_weights.shape[1]):  # 1 channel, or 2 when tiled (batch_updater_py_multi.py:293-296)
                outw[b, c] = zoom_plane(flow_weights[b, c], aff, 5)
    return out, outw


def zoom_depth(zoom_factor, depth):
    out = np.empty_like(depth, dtype=np.float32)
    for b in range(depth.shape[0]):
        out[b, 0] = zoom_plane(depth[b, 0], zoom_factor[b], 0)
    return out


def box_mask(bbox4, H, W):
    m = np.empty((H, W), np.float32)
    lib().orc_box_mask(np.ascontiguousarray(bbox4, dtype=np.int32), H, W, m)
    return m


def zoom_trans(zoom_factor, trans, b_inv_zoom):
    B = trans.shape[0]
    out = np.empty((B, 3), np.float32)
    lib().orc_zoom_trans(np.ascontiguousarray(zoom_factor, dtype=np.float32),
                         np.ascontiguousarray(trans, dtype=np.float32), B, int(b_inv_zoom), out)
    return out


# --------------------------------------------------------------------------------------------- se3
def rt_transform(pose_src, r, t, T_means=(0, 0, 0), T_stds=(1, 1, 1), rot_coord="camera"):
    out = np.zeros((3, 4), np.float64)
    lib().orc_rt_transform(np.ascontiguousarray(pose_src, dtype=np.float64),
                           np.ascontiguousarray(np.squeeze(r), dtype=np.float64),
                           np.ascontiguousarray(np.squeeze(t), dtype=np.float64),
                           np.ascontiguousarray(T_means, dtype=np.float64),
                           np.ascontiguousarray(T_stds, dtype=np.float64), ROT_COORD[rot_coord.lower()], out)
    return out


def rt_delta(pose_src, pose_tgt, T_means=(0, 0, 0), T_stds=(1, 1, 1), rot_coord="camera"):
    R = np.zeros((3, 3), np.float64)
    T = np.zeros(3, np.float64)
    lib().orc_rt_delta(np.ascontiguousarray(pose_src, dtype=np.float64),
                       np.ascontiguousarray(pose_tgt, dtype=np.float64),
                       np.ascontiguousarray(T_means, dtype=np.float64),
                       np.ascontiguousarray(T_stds, dtype=np.float64), ROT_COORD[rot_coord.lower()], R, T)
    return R, T


def flow(depth_src, depth_tgt, KT, Kinv):
    """gpu_flow (lib/flow_c/gpu_flow.pyx:24-41): (B,1,H,W),(B,1,H,W),(B,3,4),(3,3) -> flow(B,2,H,W), valid(B,1,H,W)"""
    B, _, H, W = depth_src.shape
    fl = np.empty((B, 2, H, W), np.float32)
    va = np.empty((B, 1, H, W), np.float32)
    lib().orc_flow(np.ascontiguousarray(depth_src, dtype=np.float32), np.ascontiguousarray(depth_tgt, dtype=np.float32),
                   np.ascontiguousarray(KT, dtype=np.float32).reshape(B, 12),
                   np.ascontiguousarray(Kinv, dtype=np.float32).reshape(9), B, H, W, fl, va)
    return fl, va


# --------------------------------------------------------------------------------------------- net
def conv1_input(zio, zir, zdo=None, zdr=None, zmo=None, zmr=None):
    """conv1's input (B,C,H,W) float32 numpy in the symbol's channel order (deepIM_flownet.py:33-62): the zoomed images
    / 255, the zoomed depths / 255 (INPUT_DEPTH), the zoomed masks (INPUT_MASK); a blob the network does not take is None.
    The divisions are the graph's correctly rounded float32 ones, done by torch's multithreaded CPU kernel (numpy's
    single-threaded division would add ~1 ms to each batch-1 forward of bench.py's reference leg)."""
    import torch

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    scaled = [t(a) / 255.0 for a in (zio, zir, zdo, zdr) if a is not None]
    return torch.cat(scaled + [t(a) for a in (zmo, zmr) if a is not None], dim=1).numpy()


def net_forward(weights, zio, zir, zmo=None, zmr=None, num_threads=None, return_features=False, emulate_bf16=False,
                emulate_fp16=False, *, zdo=None, zdr=None):
    """FlowNetS encoder + fc + heads, torch-CPU fp32 (deepIM_flownet.py:53-116, 716-717) on the zoomed blobs:
    without masks the image-only network, with depths the RGB-D network (flow_conv1_weight must have conv1_input's
    channels).  Returns rot (B,4) raw quaternion, trans (B,3) zoomed translation.
    emulate_bf16=True rounds what the device's throughput mode (DIM_PREC_BF16) stores in bf16 -- the conv / fc6 operand
    weights and every conv activation -- keeping fp32 accumulation: calibrates that mode's tolerance (tests).
    emulate_fp16=True does the same for DIM_PREC_FP16 (IEEE half storage, 11 significant bits)."""
    import torch
    import torch.nn.functional as F

    if num_threads:
        torch.set_num_threads(num_threads)
    from_np = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    with torch.no_grad():
        rb = (lambda t: t.bfloat16().float()) if emulate_bf16 else ((lambda t: t.half().float()) if emulate_fp16 else (lambda t: t))
        x = rb(torch.from_numpy(conv1_input(zio, zir, zdo, zdr, zmo, zmr)))
        feats = {}
        for name, s, p in ENC:
            x = F.conv2d(x, rb(from_np(weights[name + "_weight"])), from_np(weights[name + "_bias"]), stride=s, padding=p)
            x = rb(F.leaky_relu(x, 0.1))
            if return_features:
                feats[name] = x.numpy().copy()
        x = x.flatten(1)  # NCHW flatten: c*80 + h*10 + w (deepIM_flownet.py:110)
        x = F.leaky_relu(F.linear(x, rb(from_np(weights["fc6_weight"])), from_np(weights["fc6_bias"])), 0.1)
        if return_features:
            feats["fc6"] = x.numpy().copy()
        x = F.leaky_relu(F.linear(x, from_np(weights["fc7_weight"]), from_np(weights["fc7_bias"])), 0.1)
        if return_features:
            feats["fc7"] = x.numpy().copy()
        rot = F.linear(x, from_np(weights["rot_weight"]), from_np(weights["rot_bias"]))
        trans = F.linear(x, from_np(weights["trans_weight"]), from_np(weights["trans_bias"]))
    if return_features:
        return rot.numpy(), trans.numpy(), feats
    return rot.numpy(), trans.numpy()


# ------------------------------------------------------------------------------------------- chain
def test_forward(weights, image_observed, image_rendered, mask_observed, mask_rendered, src_pose, K, means_rgb,
                 depth_observed=None, depth_rendered=None, return_inputs=False):
    """One pass of the FAST_TEST graph (get_test_symbol_share, deepIM_flownet.py:548-735): returns se3 (B,7),
    zoom_factor (B,4), bbox (B,8) and, with return_inputs, the zoomed blobs: dict zio, zir, zoom_factor, bbox, plus
    zdo, zdr and zmo, zmr where the network takes them.
    With masks the zoom is ZoomMask + ZoomImageWithFactor; without (image-only network, masks None) it is ZoomImage
    (symbol:562-601).  Depths (RGB-D network) are zoomed with ZoomDepth (zoom_depth.py:24-44) by the same factor."""
    z = {}
    if mask_observed is None:
        z["zio"], z["zir"], zf, bbox = zoom_image(image_observed, image_rendered, src_pose, K, means_rgb)
    else:
        z["zmo"], _, z["zmr"], zf, bbox = zoom_mask(mask_observed, mask_observed, mask_rendered, src_pose, K)
        z["zio"], z["zir"] = zoom_image_with_factor(zf, image_observed, image_rendered, means_rgb)
    if depth_observed is not None:
        z["zdo"], z["zdr"] = zoom_depth(zf, depth_observed), zoom_depth(zf, depth_rendered)
    rot, trans_z = net_forward(weights, z["zio"], z["zir"], z.get("zmo"), z.get("zmr"), zdo=z.get("zdo"), zdr=z.get("zdr"))
    se3 = np.concatenate([rot, zoom_trans(zf, trans_z, True)], axis=1).astype(np.float32)
    if return_inputs:
        return se3, zf, bbox, dict(z, zoom_factor=zf, bbox=bbox)
    return se3, zf, bbox


def refine(weights, meshes, cls_idx, image_observed, pose_init, K, n_iter=4, means_rgb=None, zn=0.25, zf=6.0,
           poses_override=None, *, lighting=None, depth_observed=None, input_mask=True, return_inputs=False):
    """Test-time refinement loop restated from deepim/core/tester.py:340-485 (SURVEY Appendix A).
    image_observed (B,3,H,W) float32 RGB-mean; pose_init (B,3,4).  The initial rendered blobs are the
    render at pose_init (the reference loads the same thing pre-rendered from disk).
    poses_override[it] (B,3,4), if given, replaces the pose fed to iteration `it` (teacher forcing for
    per-iteration parity tests).
    lighting = {"intensity": float32 [n_iter,B,3], "offset", "brightness_ratio"}: the ModelNet branch's lit render, instance b
    of iteration `it` with intensity[it, b] and the light of its float64 pose (every mesh carries `normals`).
    depth_observed (B,1,H,W) float32 metres: the RGB-D network, fed the render's depth at the pose being refined
    (tester.py:427,437-438; the depth of the lit render is the unlit one).
    input_mask=False: the image-only network, zoomed with ZoomImage; the loop carries no masks (tester.py:439).
    Returns dict poses (n_iter,B,3,4) f64, se3 (n_iter,B,7) f32, zoom_factor (n_iter,B,4), bbox (n_iter,B,8) and, with
    return_inputs, "inputs": test_forward's zoomed blobs of each iteration."""
    B, _, H, W = image_observed.shape
    if means_rgb is None:
        means_rgb = np.array([103.939, 116.779, 123.68], np.float32)
    want = ("image",) + (("depth",) if depth_observed is not None else ()) + (("mask",) if input_mask else ())
    inten = None if lighting is None else np.asarray(lighting["intensity"], np.float32)
    pose = np.array(pose_init, dtype=np.float64)
    res = {"poses": np.zeros((n_iter, B, 3, 4)), "se3": np.zeros((n_iter, B, 7), np.float32),
           "zoom_factor": np.zeros((n_iter, B, 4), np.float32), "bbox": np.zeros((n_iter, B, 8), np.int32)}
    if return_inputs:
        res["inputs"] = []
    for it in range(n_iter):
        if poses_override is not None and poses_override[it] is not None:
            pose = np.array(poses_override[it], dtype=np.float64)
        img_r = np.empty((B, 3, H, W), np.float32)
        d_r = np.empty((B, 1, H, W), np.float32) if depth_observed is not None else None
        m_r, m_o = (np.empty((B, 1, H, W), np.float32), np.empty((B, 1, H, W), np.float32)) if input_mask else (None, None)
        for b in range(B):
            mesh = meshes[int(cls_idx[b])]
            if lighting is None:
                r = render(mesh, pose[b], K, zn, zf, H, W, means_rgb, True, want=want)
            else:
                r = _render_lit(mesh, pose[b], K, inten[it, b], lighting, zn, zf, H, W, means_rgb, want)
            img_r[b] = r["image"]
            if d_r is not None:
                d_r[b, 0] = r["depth"]
            if input_mask:
                m_r[b, 0] = r["mask"]
                m_o[b, 0] = box_mask(r["bbox"], H, W)  # data_pair.py:93-105 (end-exclusive rectangle)
        out = test_forward(weights, image_observed, img_r, m_o, m_r, pose.astype(np.float32), K, means_rgb, depth_observed, d_r,
                           return_inputs)
        se3, zfac, bbox = out[:3]
        new_pose = np.zeros_like(pose)
        for b in range(B):
            new_pose[b] = rt_transform(pose[b], se3[b, :4], se3[b, 4:], (0, 0, 0), (1, 1, 1), "camera")
        res["poses"][it], res["se3"][it], res["zoom_factor"][it], res["bbox"][it] = new_pose, se3, zfac, bbox
        if return_inputs:
            res["inputs"].append(out[3])
        pose = new_pose
    return res


# ---------------------------------------------------------------------------------------- ADD / ADI
def rt_dist(pose_est, pose_gt):
    """calc_rt_dist_m (lib/pair_matching/RT_transform.py:162-173): (rotation distance in degrees, translation distance).
    The reference takes |logm(R_est^T R_gt)|_F / sqrt(2); for rotation matrices that is the geodesic angle, evaluated here
    as atan2(|axis part|, (trace - 1) / 2)."""
    M = pose_est[:, :3].T @ pose_gt[:, :3]
    s = 0.5 * np.linalg.norm([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]])
    return float(np.degrees(np.arctan2(s, 0.5 * (np.trace(M) - 1.0)))), float(np.linalg.norm(pose_gt[:, 3] - pose_est[:, 3]))


def arp_2d(pose_est, pose_gt, pts, K):
    """lib/utils/pose_error.py:27-69: mean 2D distance between the projections of the model points under the two poses"""
    def proj(P):
        c = (np.asarray(K, np.float64) @ (P[:, :3] @ pts.T + P[:, 3:4])).T
        return c[:, :2] / c[:, 2:3]
    return float(np.linalg.norm(proj(pose_est) - proj(pose_gt), axis=1).mean())


def add_metric(R_est, t_est, R_gt, t_gt, pts):
    """lib/utils/pose_error.py:72-87"""
    pe = pts @ np.asarray(R_est).T + np.asarray(t_est).reshape(1, 3)
    pg = pts @ np.asarray(R_gt).T + np.asarray(t_gt).reshape(1, 3)
    return float(np.linalg.norm(pe - pg, axis=1).mean())


def adi_metric(R_est, t_est, R_gt, t_gt, pts):
    """lib/utils/pose_error.py:90-108 (nearest neighbour from gt points into est points)"""
    from scipy import spatial

    pe = pts @ np.asarray(R_est).T + np.asarray(t_est).reshape(1, 3)
    pg = pts @ np.asarray(R_gt).T + np.asarray(t_gt).reshape(1, 3)
    d, _ = spatial.cKDTree(pe).query(pg, k=1)
    return float(d.mean())


# ------------------------------------------------------------------------------------ Transform3D
def _quat2mat_t3d(q):
    """quat2mat_forward (deepim/operator_py/transform3d.py:185-212): identity unless |Nq-1| < 1e-2."""
    w, x, y, z = [np.float32(v) for v in q]
    Nq = np.float32(w * w + x * x + y * y + z * z)
    if not (-1e-2 < float(Nq) - 1 < 1e-2):
        return np.eye(3, dtype=np.float32)
    s = 2.0 / float(Nq)
    X, Y, Z = float(x) * s, float(y) * s, float(z) * s
    wX, wY, wZ = float(w) * X, float(w) * Y, float(w) * Z
    xX, xY, xZ = float(x) * X, float(x) * Y, float(x) * Z
    yY, yZ, zZ = float(y) * Y, float(y) * Z, float(z) * Z
    return np.array([[1.0 - (yY + zZ), xY - wZ, xZ + wY], [xY + wZ, 1.0 - (xX + zZ), yZ - wX],
                     [xZ - wY, yZ + wX, 1.0 - (xX + yY)]], dtype=np.float32)


def transform3d_forward(point_cloud, rotation, translation, pose_src, T_means, T_stds, rot_coord="model"):
    """Transform3D forward (transform3d.py:34-97), numpy float32.  point_cloud (B,3,N)."""
    B = point_cloud.shape[0]
    out = np.empty_like(point_cloud, dtype=np.float32)
    Tm, Ts = np.asarray(T_means, np.float32), np.asarray(T_stds, np.float32)
    for b in range(B):
        Rd = _quat2mat_t3d(rotation[b])
        Rs = pose_src[b, :, :3].astype(np.float32)
        Rt = (Rs @ Rd) if rot_coord.lower() == "model" else (Rd @ Rs)
        d = translation[b].astype(np.float32) * Ts + Tm
        src = pose_src[b, :, 3].astype(np.float32)
        z2 = src[2] / np.exp(d[2])
        if rot_coord.lower() == "camera_new":
            Tt = np.array([src[2] * d[0] + src[0], src[2] * d[1] + src[1], z2], np.float32)
        else:
            Tt = np.array([z2 * (d[0] + src[0] / src[2]), z2 * (d[1] + src[1] / src[2]), z2], np.float32)
        out[b] = Rt @ point_cloud[b].astype(np.float32) + Tt[:, None]
    return out


def transform3d_backward(out_grad, point_cloud, rotation, translation, pose_src, T_means, T_stds, rot_coord="model"):
    """Transform3D backward (transform3d.py:99-281): returns rot_grad (B,4), trans_grad (B,3)."""
    B = point_cloud.shape[0]
    Tm, Ts = np.asarray(T_means, np.float64), np.asarray(T_stds, np.float64)
    rg, tg = np.zeros((B, 4), np.float32), np.zeros((B, 3), np.float32)
    for b in range(B):
        D = out_grad[b].astype(np.float64).sum(axis=1)
        d = translation[b].astype(np.float64) * Ts + Tm
        src = pose_src[b, :, 3].astype(np.float64)
        z2 = src[2] / np.exp(d[2])
        if rot_coord.lower() == "camera_new":
            tg[b] = [D[0] * Ts[0] * src[2], D[1] * Ts[1] * src[2], D[2] * (-Ts[2] * z2)]
        else:
            share = -Ts[2] * z2
            tg[b] = [D[0] * Ts[0] * z2, D[1] * Ts[1] * z2,
                     D[0] * share * (d[0] + src[0] / src[2]) + D[1] * share * (d[1] + src[1] / src[2]) + D[2] * share]
        RtD = out_grad[b].astype(np.float64) @ point_cloud[b].astype(np.float64).T
        Rs = pose_src[b, :, :3].astype(np.float64)
        Dm = (Rs.T @ RtD) if rot_coord.lower() == "model" else (RtD @ Rs.T)
        w, x, y, z = [float(v) for v in rotation[b]]
        Nq = w * w + x * x + y * y + z * z
        if not (-1e-4 < Nq - 1 < 1e-4):
            continue
        Ns = np.sqrt(Nq)
        w_, x_, y_, z_ = w / Ns, x / Ns, y / Ns, z / Ns
        wd = 2 * (-z_ * Dm[0, 1] + y_ * Dm[0, 2] + z_ * Dm[1, 0] - x_ * Dm[1, 2] - y_ * Dm[2, 0] + x_ * Dm[2, 1])
        xd = 2 * (y_ * Dm[0, 1] + z_ * Dm[0, 2] + y_ * Dm[1, 0] - 2 * x_ * Dm[1, 1] - w_ * Dm[1, 2] + z_ * Dm[2, 0]
                  + w_ * Dm[2, 1] - 2 * x_ * Dm[2, 2])
        yd = 2 * (-2 * y_ * Dm[0, 0] + x_ * Dm[0, 1] + w_ * Dm[0, 2] + x_ * Dm[1, 0] + z_ * Dm[1, 2] - w_ * Dm[2, 0]
                  + z_ * Dm[2, 1] - 2 * y_ * Dm[2, 2])
        zd = 2 * (-2 * z_ * Dm[0, 0] - w_ * Dm[0, 1] + x_ * Dm[0, 2] + w_ * Dm[1, 0] - 2 * z_ * Dm[1, 1]
                  + y_ * Dm[1, 2] + x_ * Dm[2, 0] + y_ * Dm[2, 1])
        share = Ns ** 3 * (w * wd + x * xd + y * yd + z * zd)
        rg[b] = [Ns * wd - w * share, Ns * xd - x * share, Ns * yd - y * share, Ns * zd - z * share]
    return rg, tg


# ----------------------------------------------------------------------- train-time batch update
def mat2quat(M):
    """RT_transform.py:432-509 (Bar-Itzhack): eigenvector of the largest eigenvalue of a symmetric 4x4."""
    Qxx, Qyx, Qzx, Qxy, Qyy, Qzy, Qxz, Qyz, Qzz = np.asarray(M, np.float64).flat
    Kq = np.array([[Qxx - Qyy - Qzz, 0, 0, 0], [Qyx + Qxy, Qyy - Qxx - Qzz, 0, 0],
                   [Qzx + Qxz, Qzy + Qyz, Qzz - Qxx - Qyy, 0],
                   [Qyz - Qzy, Qzx - Qxz, Qxy - Qyx, Qxx + Qyy + Qzz]]) / 3.0
    vals, vecs = np.linalg.eigh(Kq)
    q = vecs[[3, 0, 1, 2], np.argmax(vals)]
    if q[0] < 0:
        q = -q
    return q


def rt_delta_f32tgt(pose_src, pose_tgt32, T_means, T_stds, rot_coord):
    """calc_RT_delta as the train loop calls it: pose_src float64 (refined pose), pose_tgt a float32 array
    (it comes out of an NDArray), so T_tgt[0]/T_tgt[2] is a float32 division (RT_transform.py:120-121)."""
    tgt32 = np.asarray(pose_tgt32, np.float32)
    Rd, Td = rt_delta(pose_src, tgt32.astype(np.float64), T_means, T_stds, rot_coord)
    if rot_coord.lower() != "camera_new":
        src = np.asarray(pose_src, np.float64)
        d0 = np.float64(tgt32[0, 3] / tgt32[2, 3]) - src[0, 3] / src[2, 3]
        d1 = np.float64(tgt32[1, 3] / tgt32[2, 3]) - src[1, 3] / src[2, 3]
        Td = Td.copy()
        Td[0] = (d0 - T_means[0]) / T_stds[0]
        Td[1] = (d1 - T_means[1]) / T_stds[1]
    return Rd, Td


def calc_se3_f32(pose_src, pose_tgt):
    """calc_se3 (RT_transform.py:176-187) over lib/utils/projection.py se3_inverse / se3_mul, which store
    their results in float32 arrays.  pose_src float64 (refined pose), pose_tgt float32."""
    R, T = np.asarray(pose_src)[:, :3], np.asarray(pose_src)[:, 3].reshape(3, 1)
    inv = np.zeros((3, 4), np.float32)
    inv[:, :3] = R.T
    inv[:, 3] = (-1 * (R.T @ T)).reshape(3)
    R1, T1 = np.asarray(pose_tgt, np.float32)[:, :3], np.asarray(pose_tgt, np.float32)[:, 3].reshape(3, 1)
    out = np.zeros((3, 4), np.float32)
    out[:, :3] = R1 @ inv[:, :3]
    out[:, 3] = (R1 @ inv[:, 3].reshape(3, 1) + T1).reshape(3)
    return out


def train_update(meshes, cls_idx, src_pose, rot_est, trans_est, tgt_pose, depth_gt_observed, K, means_rgb,
                 T_means=(0, 0, 0), T_stds=(1, 1, 1), rot_coord="camera", zn=0.25, zf=6.0, lighting=None):
    """batchUpdaterPyMulti.forward (lib/pair_matching/batch_updater_py_multi.py:91-328) for one context.
    src_pose / tgt_pose / rot_est / trans_est are float32 (they come out of NDArrays).
    lighting = {"intensity": float32 [B,3], "offset", "brightness_ratio"}: the ModelNet branch, whose re-render is lit at the
    float64 refined pose (l.187-229) and whose image is refined_image[:, :, [2,1,0]].transpose([2,0,1]).astype(np.float32)
    - pixel_means in float32 (l.234-235); the unlit image is the render's, its means subtracted in float64."""
    B = len(cls_idx)
    H, W = depth_gt_observed.shape[-2:]
    out = {"image_rendered": np.zeros((B, 3, H, W), np.float32), "depth_rendered": np.zeros((B, 1, H, W), np.float32),
           "mask_rendered": np.zeros((B, 1, H, W), np.float32), "src_pose": np.zeros((B, 3, 4), np.float32),
           "rot": np.zeros((B, 4), np.float32), "trans": np.zeros((B, 3), np.float32)}
    KT = np.zeros((B, 3, 4), np.float32)
    if lighting is not None:
        inten, m32 = np.asarray(lighting["intensity"], np.float32), np.asarray(means_rgb, np.float32)
    for b in range(B):
        refined = rt_transform(src_pose[b].astype(np.float64), rot_est[b], trans_est[b], T_means, T_stds, rot_coord)
        mesh = meshes[int(cls_idx[b])]
        if lighting is None:
            r = render(mesh, refined, K, zn, zf, H, W, means_rgb, trunc_u8=False, want=("image", "depth", "mask"))
            out["image_rendered"][b] = r["image"]
        else:
            r = _render_lit(mesh, refined, K, inten[b], lighting, zn, zf, H, W, means_rgb, ("bgr", "depth", "mask"))
            out["image_rendered"][b] = r["bgr"][:, :, [2, 1, 0]].transpose([2, 0, 1]).astype(np.float32) - m32[:, None, None]
        out["depth_rendered"][b, 0], out["mask_rendered"][b, 0] = r["depth"], r["mask"]
        Rd, Td = rt_delta_f32tgt(refined, tgt_pose[b], T_means, T_stds, rot_coord)
        out["rot"][b], out["trans"][b] = mat2quat(Rd), Td
        out["src_pose"][b] = refined
        KT[b] = (np.asarray(K, np.float64) @ calc_se3_f32(refined, tgt_pose[b]).astype(np.float64)).astype(np.float32)
    Kinv = np.linalg.inv(np.asarray(K, np.float64)).astype(np.float32)
    fl, va = flow(out["depth_rendered"], depth_gt_observed, KT, Kinv)
    out["flow"], out["flow_weights"], out["KT"] = fl, np.tile(va, [1, 2, 1, 1]), KT
    return out
