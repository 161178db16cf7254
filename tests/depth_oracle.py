"""CPU checker of the RGB-D network (config.network.INPUT_DEPTH with INPUT_MASK), built from the oracle's pieces
(oracle.render's depth, oracle.zoom_depth, the zoom / RT_transform chain of oracle.test_forward) and a torch-CPU tower with
a 10-channel flow_conv1.  Test infrastructure only, like the oracle.

The reference (deepim/symbols/deepIM_flownet.py:35-43) feeds conv1 with

    concat(image_observed/255, image_rendered/255, depth_observed/255, depth_rendered/255, mask_observed, mask_rendered)

where the depths are zoomed by ZoomDepth (zoom_depth.py:24-44) with the iteration's zoom factor, depth_observed is the
loader's float32(u16) / DEPTH_FACTOR (lib/utils/image.py:203,218) and depth_rendered is the render's depth at the pose
being refined (tester.py:427,437-438), 0 on the background.
"""
import numpy as np

from oracle import oracle as O

CONV_SPECS = [("flow_conv1", 2, 3), ("conv2", 2, 2), ("conv3", 2, 2), ("conv3_1", 1, 1), ("conv4", 2, 1),
              ("conv4_1", 1, 1), ("conv5", 2, 1), ("conv5_1", 1, 1), ("conv6", 2, 1), ("conv6_1", 1, 1)]


def depth_from_u16(u16, depth_factor=1000.0):
    """lib/utils/image.py:203,218: a float32 array divided by a Python float stays float32 (float32-rounded factor)."""
    return np.asarray(u16).astype(np.float32) / depth_factor


def conv1_input(zio, zir, zdo, zdr, zmo, zmr):
    """The RGB-D network's conv1 input (B,10,H,W) float32, the graph's float32 divisions included."""
    f = lambda a: np.asarray(a, np.float32)
    return np.concatenate([f(zio) / np.float32(255), f(zir) / np.float32(255), f(zdo) / np.float32(255),
                           f(zdr) / np.float32(255), f(zmo), f(zmr)], axis=1)


def net_forward(weights, zio, zir, zdo, zdr, zmo, zmr):
    """oracle.net_forward with the 10-channel input: FlowNetS tower + fc + heads in torch-CPU fp32.
    Returns rot (B,4) raw quaternion, trans (B,3) zoomed translation."""
    import torch
    import torch.nn.functional as F

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    with torch.no_grad():
        x = t(conv1_input(zio, zir, zdo, zdr, zmo, zmr))
        for name, s, p in CONV_SPECS:
            x = F.leaky_relu(F.conv2d(x, t(weights[name + "_weight"]), t(weights[name + "_bias"]), stride=s, padding=p), 0.1)
        x = x.flatten(1)
        x = F.leaky_relu(F.linear(x, t(weights["fc6_weight"]), t(weights["fc6_bias"])), 0.1)
        x = F.leaky_relu(F.linear(x, t(weights["fc7_weight"]), t(weights["fc7_bias"])), 0.1)
        rot = F.linear(x, t(weights["rot_weight"]), t(weights["rot_bias"]))
        trans = F.linear(x, t(weights["trans_weight"]), t(weights["trans_bias"]))
    return rot.numpy(), trans.numpy()


def zoom_inputs(image_observed, image_rendered, depth_observed, depth_rendered, mask_observed, mask_rendered, src_pose, K,
                means_rgb):
    """The zoomed blobs of one pass: dict zio, zir, zdo, zdr, zmo, zmr, zoom_factor, bbox."""
    zmo, _, zmr, zf, bbox = O.zoom_mask(mask_observed, mask_observed, mask_rendered, src_pose, K)
    zio, zir = O.zoom_image_with_factor(zf, image_observed, image_rendered, means_rgb)
    zdo, zdr = O.zoom_depth(zf, depth_observed), O.zoom_depth(zf, depth_rendered)
    return dict(zio=zio, zir=zir, zdo=zdo, zdr=zdr, zmo=zmo, zmr=zmr, zoom_factor=zf, bbox=bbox)


def test_forward(weights, image_observed, image_rendered, depth_observed, depth_rendered, mask_observed, mask_rendered,
                 src_pose, K, means_rgb):
    """oracle.test_forward of the RGB-D graph: se3 (B,7), zoom_factor (B,4), bbox (B,8), the zoomed blobs."""
    z = zoom_inputs(image_observed, image_rendered, depth_observed, depth_rendered, mask_observed, mask_rendered, src_pose, K,
                    means_rgb)
    rot, trans_z = net_forward(weights, z["zio"], z["zir"], z["zdo"], z["zdr"], z["zmo"], z["zmr"])
    trans = O.zoom_trans(z["zoom_factor"], trans_z, True)
    return np.concatenate([rot, trans], axis=1).astype(np.float32), z["zoom_factor"], z["bbox"], z


def refine(weights, meshes, cls_idx, image_observed, depth_observed, pose_init, K, n_iter=4, means_rgb=None, zn=0.25,
           zf=6.0, poses_override=None, lighting=None):
    """oracle.refine of the RGB-D network: each iteration renders image, mask and depth at the current pose and feeds both
    zoomed depths to the tower.  depth_observed (B,1,H,W) float32 metres.  lighting: None = unlit; else as lit_oracle.refine
    (the render's depth is the unlit one).  Returns oracle.refine's dict plus "inputs": the zoomed blobs of each iteration."""
    B, _, H, W = image_observed.shape
    if means_rgb is None:
        means_rgb = np.array([103.939, 116.779, 123.68], np.float32)
    if lighting is not None:
        import lit_oracle
        inten = np.asarray(lighting["intensity"], np.float32)
    pose = np.array(pose_init, dtype=np.float64)
    res = {"poses": np.zeros((n_iter, B, 3, 4)), "se3": np.zeros((n_iter, B, 7), np.float32),
           "zoom_factor": np.zeros((n_iter, B, 4), np.float32), "bbox": np.zeros((n_iter, B, 8), np.int32), "inputs": []}
    for it in range(n_iter):
        if poses_override is not None and poses_override[it] is not None:
            pose = np.array(poses_override[it], dtype=np.float64)
        img_r = np.empty((B, 3, H, W), np.float32)
        d_r = np.empty((B, 1, H, W), np.float32)
        m_r = np.empty((B, 1, H, W), np.float32)
        m_o = np.empty((B, 1, H, W), np.float32)
        for b in range(B):
            mesh = meshes[int(cls_idx[b])]
            if lighting is None:
                r = O.render(mesh, pose[b], K, zn, zf, H, W, means_rgb, True, want=("image", "depth", "mask"))
            else:
                r = lit_oracle._render(mesh, pose[b], K, inten[it, b], lighting, zn, zf, H, W, means_rgb,
                                       ("image", "depth", "mask"))
            img_r[b], d_r[b, 0], m_r[b, 0] = r["image"], r["depth"], r["mask"]
            m_o[b, 0] = O.box_mask(r["bbox"], H, W)
        se3, zfac, bbox, z = test_forward(weights, image_observed, img_r, depth_observed, d_r, m_o, m_r,
                                          pose.astype(np.float32), K, means_rgb)
        new_pose = np.zeros_like(pose)
        for b in range(B):
            new_pose[b] = O.rt_transform(pose[b], se3[b, :4], se3[b, 4:], (0, 0, 0), (1, 1, 1), "camera")
        res["poses"][it], res["se3"][it], res["zoom_factor"][it], res["bbox"][it] = new_pose, se3, zfac, bbox
        res["inputs"].append(z)
        pose = new_pose
    return res


def train_forward_backward(weights, batch, K, means_rgb, requires_grad=True):
    """The RGB-D train graph (symbol:461-475 with INPUT_DEPTH) on the oracle's zoom front: batch = train_oracle's batch plus
    depth_observed and depth_rendered (B,1,H,W) metres, zoomed with the pair's zoom factor (ZoomDepth).  train_oracle.graph
    builds conv1's input as cat(observed/255, rendered/255, masks): handing it the two image blobs as one 6-channel
    "observed" image and the two depths as a 2-channel "rendered" one gives exactly the 10-channel order of the symbol.
    Returns (outputs, grads, zin with the zoomed depths, labels) like train_oracle.forward_backward."""
    from oracle import train_oracle as T
    zin, labels = T.zoom_inputs(batch, K, means_rgb)
    zf = labels["zoom_factor"]
    zin["zoom_depth_observed"] = O.zoom_depth(zf, batch["depth_observed"])
    zin["zoom_depth_rendered"] = O.zoom_depth(zf, batch["depth_rendered"])
    cat = {"zoom_image_observed": np.concatenate([zin["zoom_image_observed"], zin["zoom_image_rendered"]], axis=1),
           "zoom_image_rendered": np.concatenate([zin["zoom_depth_observed"], zin["zoom_depth_rendered"]], axis=1),
           "zoom_mask_observed": zin["zoom_mask_observed"], "zoom_mask_rendered": zin["zoom_mask_rendered"]}
    out, grads = T.graph(weights, cat, labels, requires_grad)
    return out, grads, zin, labels
