"""CPU checker of the image-only network (config.network.INPUT_MASK: False), built from the oracle's pieces (oracle.zoom_image,
the render / RT_transform chain of oracle.refine, train_oracle.graph) and a torch-CPU tower with a 6-channel flow_conv1.  Test
infrastructure only, like the oracle.

The reference (deepim/symbols/deepIM_flownet.py:53-62) feeds conv1 with

    concat(image_observed/255, image_rendered/255)

and its test graph zooms both images with ZoomImage (zoom_image.py:26-107; symbol:562-601): the boxes are the pixels with
sum_c(image + mean) > 0.01, and an empty rendered box centres the zoom on the observed one.  The loop carries no masks
(tester.py:439).
"""
import numpy as np

from oracle import oracle as O

CONV_SPECS = [("flow_conv1", 2, 3), ("conv2", 2, 2), ("conv3", 2, 2), ("conv3_1", 1, 1), ("conv4", 2, 1),
              ("conv4_1", 1, 1), ("conv5", 2, 1), ("conv5_1", 1, 1), ("conv6", 2, 1), ("conv6_1", 1, 1)]


def conv1_input(zio, zir):
    """The image-only network's conv1 input (B,6,H,W) float32, the graph's float32 divisions included."""
    f = lambda a: np.asarray(a, np.float32)
    return np.concatenate([f(zio) / np.float32(255), f(zir) / np.float32(255)], axis=1)


def net_forward(weights, zio, zir):
    """oracle.net_forward with the mask columns removed: FlowNetS tower + fc + heads in torch-CPU fp32 on the 6-channel input.
    Returns rot (B,4) raw quaternion, trans (B,3) zoomed translation."""
    import torch
    import torch.nn.functional as F

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    with torch.no_grad():
        x = t(conv1_input(zio, zir))
        for name, s, p in CONV_SPECS:
            x = F.leaky_relu(F.conv2d(x, t(weights[name + "_weight"]), t(weights[name + "_bias"]), stride=s, padding=p), 0.1)
        x = x.flatten(1)
        x = F.leaky_relu(F.linear(x, t(weights["fc6_weight"]), t(weights["fc6_bias"])), 0.1)
        x = F.leaky_relu(F.linear(x, t(weights["fc7_weight"]), t(weights["fc7_bias"])), 0.1)
        rot = F.linear(x, t(weights["rot_weight"]), t(weights["rot_bias"]))
        trans = F.linear(x, t(weights["trans_weight"]), t(weights["trans_bias"]))
    return rot.numpy(), trans.numpy()


def zoom_inputs(image_observed, image_rendered, src_pose, K, means_rgb):
    """ZoomImage of one pass: dict zio, zir, zoom_factor, bbox (8 ints: observed x0,x1,y0,y1, rendered x0,x1,y0,y1)."""
    zio, zir, zf, bbox = O.zoom_image(image_observed, image_rendered, src_pose, K, means_rgb)
    return dict(zio=zio, zir=zir, zoom_factor=zf, bbox=bbox)


def test_forward(weights, image_observed, image_rendered, src_pose, K, means_rgb):
    """One pass of the image-only FAST_TEST graph: se3 (B,7), zoom_factor (B,4), bbox (B,8), the zoomed blobs."""
    z = zoom_inputs(image_observed, image_rendered, src_pose, K, means_rgb)
    rot, trans_z = net_forward(weights, z["zio"], z["zir"])
    trans = O.zoom_trans(z["zoom_factor"], trans_z, True)
    return np.concatenate([rot, trans], axis=1).astype(np.float32), z["zoom_factor"], z["bbox"], z


def refine(weights, meshes, cls_idx, image_observed, pose_init, K, n_iter=4, means_rgb=None, zn=0.25, zf=6.0,
           poses_override=None, lighting=None):
    """oracle.refine of the image-only network: each iteration renders the image at the current pose and zooms with
    ZoomImage.  lighting: None = unlit; else as lit_oracle.refine.  Returns oracle.refine's dict plus "inputs": the zoomed
    blobs of each iteration."""
    B, _, H, W = image_observed.shape
    if means_rgb is None:
        means_rgb = np.array([103.939, 116.779, 123.68], np.float32)
    if lighting is not None:
        import lit_oracle
        inten = np.asarray(lighting["intensity"], np.float32)
    means32 = np.asarray(means_rgb, np.float32)
    pose = np.array(pose_init, dtype=np.float64)
    res = {"poses": np.zeros((n_iter, B, 3, 4)), "se3": np.zeros((n_iter, B, 7), np.float32),
           "zoom_factor": np.zeros((n_iter, B, 4), np.float32), "bbox": np.zeros((n_iter, B, 8), np.int32), "inputs": []}
    for it in range(n_iter):
        if poses_override is not None and poses_override[it] is not None:
            pose = np.array(poses_override[it], dtype=np.float64)
        img_r = np.empty((B, 3, H, W), np.float32)
        for b in range(B):
            mesh = meshes[int(cls_idx[b])]
            if lighting is None:
                r = O.render(mesh, pose[b], K, zn, zf, H, W, means_rgb, True, want=("image",))
            else:
                r = lit_oracle._render(mesh, pose[b], K, inten[it, b], lighting, zn, zf, H, W, means_rgb, ("image",))
            img_r[b] = r["image"]
        se3, zfac, bbox, z = test_forward(weights, image_observed, img_r, pose.astype(np.float32), K, means32)
        new_pose = np.zeros_like(pose)
        for b in range(B):
            new_pose[b] = O.rt_transform(pose[b], se3[b, :4], se3[b, 4:], (0, 0, 0), (1, 1, 1), "camera")
        res["poses"][it], res["se3"][it], res["zoom_factor"][it], res["bbox"][it] = new_pose, se3, zfac, bbox
        res["inputs"].append(z)
        pose = new_pose
    return res


def train_forward_backward(weights, batch, K, means_rgb, requires_grad=True):
    """The train graph of the image-only network with PRED_MASK (ZoomMask front and mask labels unchanged,
    deepIM_flownet.py:391) on the oracle's zoom front.  train_oracle.graph builds conv1's input as
    cat(observed/255, rendered/255, masks): zero-channel mask blobs make it exactly the 6-channel input.
    Returns (outputs, grads, zin, labels) like train_oracle.forward_backward."""
    from oracle import train_oracle as T
    zin, labels = T.zoom_inputs(batch, K, means_rgb)
    B, _, H, W = zin["zoom_image_observed"].shape
    none = np.zeros((B, 0, H, W), np.float32)
    out, grads = T.graph(weights, dict(zin, zoom_mask_observed=none, zoom_mask_rendered=none), labels, requires_grad)
    return out, grads, zin, labels
