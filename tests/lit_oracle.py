"""CPU checker of the ModelNet (unseen-object) branch of the test and train loops, built from the oracle's pieces
(oracle.render_lit, the zoom / net / RT_transform chain of oracle.test_forward, the label and flow helpers of
oracle.train_update).  Test infrastructure only, like the oracle.

The reference (deepim/core/tester.py:146-188, lib/pair_matching/batch_updater_py_multi.py:187-235) renders every pose of
those loops with Render_Py_Light_ModelNet_Multi; per render, with `pose` the float64 pose being rendered:

    light_position = np.array([0, 1, 1]) * 0.5
    light_position[0] += pose[0, 3]; light_position[1] -= pose[1, 3]; light_position[2] -= pose[2, 3]

cast to float32 by the glumpy uniform.  `lighting` = {"intensity": float32 [n_iter,B,3] (refine) / [B,3] (train_update),
"offset": (0, 0.5, 0.5), "brightness_ratio": 0.7}; every mesh carries `normals`.
"""
import numpy as np

from oracle import oracle as O

OFFSET = (0.0, 0.5, 0.5)
BRIGHTNESS_RATIO = 0.7


def light_position(pose, offset=OFFSET):
    """The reference's statements on the float64 pose, cast to float32 at the end."""
    light = np.array(offset, dtype=np.float64)
    pose = np.asarray(pose, dtype=np.float64)
    light[0] += pose[0, 3]
    light[1] -= pose[1, 3]
    light[2] -= pose[2, 3]
    return light.astype(np.float32)


def _render(mesh, pose, K, intensity, lighting, zn, zf, H, W, means_rgb, want):
    return O.render_lit(mesh, mesh.normals, pose, K, light_position(pose, lighting.get("offset", OFFSET)), intensity,
                        lighting.get("brightness_ratio", BRIGHTNESS_RATIO), zn, zf, H, W, means_rgb, want)


def refine(weights, meshes, cls_idx, image_observed, pose_init, K, lighting, n_iter=4, means_rgb=None, zn=0.25, zf=6.0,
           poses_override=None):
    """oracle.refine with the lit render: iteration `it` renders instance b with intensity[it, b] and the light of its
    float64 pose; everything after the render is the unlit loop's."""
    B, _, H, W = image_observed.shape
    if means_rgb is None:
        means_rgb = np.array([103.939, 116.779, 123.68], np.float32)
    inten = np.asarray(lighting["intensity"], np.float32)
    pose = np.array(pose_init, dtype=np.float64)
    res = {"poses": np.zeros((n_iter, B, 3, 4)), "se3": np.zeros((n_iter, B, 7), np.float32),
           "zoom_factor": np.zeros((n_iter, B, 4), np.float32), "bbox": np.zeros((n_iter, B, 8), np.int32)}
    for it in range(n_iter):
        if poses_override is not None and poses_override[it] is not None:
            pose = np.array(poses_override[it], dtype=np.float64)
        img_r = np.empty((B, 3, H, W), np.float32)
        m_r = np.empty((B, 1, H, W), np.float32)
        m_o = np.empty((B, 1, H, W), np.float32)
        for b in range(B):
            r = _render(meshes[int(cls_idx[b])], pose[b], K, inten[it, b], lighting, zn, zf, H, W, means_rgb,
                        ("image", "mask"))
            img_r[b], m_r[b, 0] = r["image"], r["mask"]
            m_o[b, 0] = O.box_mask(r["bbox"], H, W)
        se3, zfac, bbox = O.test_forward(weights, image_observed, img_r, m_o, m_r, pose.astype(np.float32), K, means_rgb)
        new_pose = np.zeros_like(pose)
        for b in range(B):
            new_pose[b] = O.rt_transform(pose[b], se3[b, :4], se3[b, 4:], (0, 0, 0), (1, 1, 1), "camera")
        res["poses"][it], res["se3"][it], res["zoom_factor"][it], res["bbox"][it] = new_pose, se3, zfac, bbox
        pose = new_pose
    return res


def train_update(meshes, cls_idx, src_pose, rot_est, trans_est, tgt_pose, depth_gt_observed, K, means_rgb, lighting,
                 T_means=(0, 0, 0), T_stds=(1, 1, 1), rot_coord="camera", zn=0.25, zf=6.0):
    """oracle.train_update with the lit render at the float64 refined pose (l.187-229), then
    refined_image[:, :, [2,1,0]].transpose([2,0,1]).astype(np.float32) - pixel_means in float32 (l.234-235)."""
    B = len(cls_idx)
    H, W = depth_gt_observed.shape[-2:]
    inten = np.asarray(lighting["intensity"], np.float32)
    m32 = np.asarray(means_rgb, np.float32)
    out = {"image_rendered": np.zeros((B, 3, H, W), np.float32), "depth_rendered": np.zeros((B, 1, H, W), np.float32),
           "mask_rendered": np.zeros((B, 1, H, W), np.float32), "src_pose": np.zeros((B, 3, 4), np.float32),
           "rot": np.zeros((B, 4), np.float32), "trans": np.zeros((B, 3), np.float32)}
    KT = np.zeros((B, 3, 4), np.float32)
    for b in range(B):
        refined = O.rt_transform(src_pose[b].astype(np.float64), rot_est[b], trans_est[b], T_means, T_stds, rot_coord)
        r = _render(meshes[int(cls_idx[b])], refined, K, inten[b], lighting, zn, zf, H, W, means_rgb, ("bgr", "depth", "mask"))
        out["image_rendered"][b] = r["bgr"][:, :, [2, 1, 0]].transpose([2, 0, 1]).astype(np.float32) - m32[:, None, None]
        out["depth_rendered"][b, 0], out["mask_rendered"][b, 0] = r["depth"], r["mask"]
        Rd, Td = O.rt_delta_f32tgt(refined, tgt_pose[b], T_means, T_stds, rot_coord)
        out["rot"][b], out["trans"][b] = O.mat2quat(Rd), Td
        out["src_pose"][b] = refined
        KT[b] = (np.asarray(K, np.float64) @ O.calc_se3_f32(refined, tgt_pose[b]).astype(np.float64)).astype(np.float32)
    Kinv = np.linalg.inv(np.asarray(K, np.float64)).astype(np.float32)
    fl, va = O.flow(out["depth_rendered"], depth_gt_observed, KT, Kinv)
    out["flow"], out["flow_weights"], out["KT"] = fl, np.tile(va, [1, 2, 1, 1]), KT
    return out
