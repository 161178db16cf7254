"""Context: Python owner of a dim_ctx (one per CUDA device) and thin tensor-level wrappers.

PyTorch is used only for device memory and streams (torch.Tensor.data_ptr, torch.cuda.current_stream);
all compute goes through libdeepim_b200.so.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _capi as capi
from . import lighting as _lighting
from ._capi import check, farr, lib

WEIGHT_ORDER = ["flow_conv1", "conv2", "conv3", "conv3_1", "conv4", "conv4_1", "conv5", "conv5_1", "conv6",
                "conv6_1", "fc6", "fc7", "rot", "trans"]




VISIB_MODES = {"sixd17": 0, "bop19": 1}  # pose_error_vsd's visib_mode -> dim_pose_error_vsd_ex's


def _p(t):
    if t is None:
        return None
    if not t.is_cuda or not t.is_contiguous():
        raise ValueError("expected a contiguous CUDA tensor")
    return C.c_void_p(t.data_ptr())


def _chk(t, dtype, shape=None, name="tensor"):
    if t.dtype != dtype:
        raise TypeError("%s: expected dtype %s, got %s" % (name, dtype, t.dtype))
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError("%s: expected shape %s, got %s" % (name, tuple(shape), tuple(t.shape)))
    return t


def hptr(a):
    """host pointer of a numpy array or a CPU torch tensor"""
    return C.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else C.c_void_p(a.ctypes.data)


def _host(a, dtype, tdtype, name):
    """a as a contiguous host array of dtype (a CPU torch tensor must already have it)"""
    if isinstance(a, torch.Tensor):
        if a.is_cuda or a.dtype != tdtype:
            raise ValueError("%s must be a host %s array" % (name, np.dtype(dtype).name))
        return a.contiguous()
    return np.ascontiguousarray(a, dtype)


def _lighting_arg(lighting, shape, on_device):
    """dim_lighting for a lighting dict (see deepim_b200.lighting): intensity float32 `shape`, a contiguous CUDA tensor when
    on_device, else a host array (numpy or CPU torch tensor).  Returns (struct, host array to keep alive)."""
    if "intensity" not in lighting:
        raise ValueError("lighting needs 'intensity' (float32 %s)" % (tuple(shape),))
    offset, ratio = _lighting.params(lighting)
    inten, keep = lighting["intensity"], None
    if on_device:
        _chk(inten, torch.float32, shape, "lighting['intensity']")
        ptr = _p(inten)
    else:
        if isinstance(inten, torch.Tensor):
            if inten.is_cuda:
                raise ValueError("lighting['intensity'] must be a host array for the host entry point")
            keep = inten.contiguous()
            _chk(keep, torch.float32, shape, "lighting['intensity']")
            ptr = C.c_void_p(keep.data_ptr())
        else:
            keep = np.ascontiguousarray(inten, np.float32)
            if keep.shape != tuple(shape):
                raise ValueError("lighting['intensity']: expected shape %s, got %s" % (tuple(shape), keep.shape))
            ptr = C.c_void_p(keep.ctypes.data)
    return capi.Lighting(ptr, (C.c_double * 3)(*offset), float(np.float32(ratio))), keep


def _per_frame_k(K, F):
    """True when K holds one camera per frame ([F,3,3]), False for one camera ([3,3], or anything of 9 values as before);
    raises on an [n,3,3] whose n is not F"""
    shape = tuple(K.shape) if isinstance(K, torch.Tensor) else np.shape(K)
    if len(shape) != 3:
        return False
    if shape != (F, 3, 3):
        raise ValueError("K: expected [3,3] (one camera) or [F,3,3] = %s (one camera per frame), got %s" % ((F, 3, 3), shape))
    return True


class Context:
    def __init__(self, device=0, max_batch=16, height=480, width=640, max_classes=16, max_verts=60000,
                 max_faces=120000, input_depth=False, input_mask=True):
        """input_depth=True: the RGB-D network (config.network.INPUT_DEPTH, deepIM_flownet.py:33-51).  Its input gains
        depth_observed/255 and depth_rendered/255 as channels 6 and 7, so flow_conv1_weight is (64, 10, 7, 7); refine /
        refine_host then need the observed depth and net_forward the zoomed depths.
        input_mask=False: the image-only network (config.network.INPUT_MASK: False, deepIM_flownet.py:53-62): conv1 sees the
        two images only, so flow_conv1_weight is (64, 6, 7, 7); refine / refine_host zoom with ZoomImage (boxes from the
        images' colours) and net_forward takes no masks.  Not combinable with input_depth."""
        if not torch.cuda.is_available():
            raise capi.DeepIMError("deepim_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        torch.cuda.set_device(self.device)
        self.H, self.W, self.max_batch = height, width, max_batch
        h = C.c_void_p()
        check(lib.dim_ctx_create(device, max_batch, height, width, max_classes, max_verts, max_faces, C.byref(h)))
        self._h = h
        self.num_classes = 0
        self.input_depth = bool(input_depth)
        self.input_mask = bool(input_mask)
        if self.input_depth:
            check(lib.dim_ctx_set_input_depth(h, 1))
        if not self.input_mask:
            check(lib.dim_ctx_set_input_mask(h, 0))

    def _stream(self):
        """torch's current stream OF THIS CONTEXT'S DEVICE (a process may hold contexts on several GPUs)"""
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def close(self):
        if getattr(self, "_h", None):
            lib.dim_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------------------ setup
    def upload_mesh(self, cls_idx, mesh):
        """a textured mesh (uvs + tex) or a vertex-coloured one (colours), with its normals when it has them"""
        v = np.ascontiguousarray(mesh.verts, np.float32)
        f = np.ascontiguousarray(mesh.faces, np.int32)
        colours = getattr(mesh, "colours", None)
        if colours is not None:
            c = np.ascontiguousarray(colours, np.float32)
            check(lib.dim_mesh_upload_colours(self._h, cls_idx, v.ctypes.data, c.ctypes.data, len(v), f.ctypes.data, len(f)))
        else:
            uv = np.ascontiguousarray(mesh.uvs, np.float32)
            tex = np.ascontiguousarray(mesh.tex, np.uint8)
            check(lib.dim_mesh_upload(self._h, cls_idx, v.ctypes.data, uv.ctypes.data, len(v), f.ctypes.data, len(f),
                                      tex.ctypes.data, tex.shape[0], tex.shape[1]))
        self.num_classes = max(self.num_classes, cls_idx + 1)
        if getattr(mesh, "normals", None) is not None:
            self.upload_normals(cls_idx, mesh.normals)

    def upload_normals(self, cls_idx, normals):
        n = np.ascontiguousarray(normals, np.float32)
        check(lib.dim_mesh_upload_normals(self._h, cls_idx, n.ctypes.data, len(n)))

    def load_weights(self, weights: dict):
        """weights: name_weight / name_bias float32 arrays with MXNet layouts
        (deepim/symbols/deepIM_flownet.py:63-116,716-717)."""
        shape = tuple(np.shape(weights["flow_conv1_weight"]))
        want = (64, 10 if self.input_depth else (8 if self.input_mask else 6), 7, 7)
        if shape != want:
            raise ValueError("flow_conv1_weight has shape %s: this context's network takes %s (Context(input_depth=%s, "
                             "input_mask=%s)); (64, 8, 7, 7) belongs to Context(), (64, 10, 7, 7) to Context(input_depth=True), "
                             "(64, 6, 7, 7) to Context(input_mask=False)" % (shape, want, self.input_depth, self.input_mask))
        keep = []
        W = (C.c_void_p * 14)()
        Bv = (C.c_void_p * 14)()
        for i, n in enumerate(WEIGHT_ORDER):
            w = np.ascontiguousarray(weights[n + "_weight"], np.float32)
            b = np.ascontiguousarray(weights[n + "_bias"], np.float32)
            keep += [w, b]
            W[i], Bv[i] = w.ctypes.data, b.ctypes.data
        check(lib.dim_net_load(self._h, W, Bv))

    def _new(self, shape, dtype=torch.float32):
        return torch.empty(shape, dtype=dtype, device=self.device)

    # ------------------------------------------------------------------------------ render
    def render(self, cls_idx, pose, K, znear=0.25, zfar=6.0, pixel_means_rgb=(0, 0, 0), trunc_u8=True,
               want=("image", "depth", "mask")):
        """cls_idx int32[B], pose float32[B,3,4] (CUDA). Returns dict of CUDA tensors + bbox int32[B,4]."""
        B = pose.shape[0]
        _chk(pose, torch.float32, (B, 3, 4), "pose")
        _chk(cls_idx, torch.int32, (B,), "cls_idx")
        out = {
            "image": self._new((B, 3, self.H, self.W)) if "image" in want else None,
            "depth": self._new((B, 1, self.H, self.W)) if "depth" in want else None,
            "mask": self._new((B, 1, self.H, self.W)) if "mask" in want else None,
            "bgr": self._new((B, self.H, self.W, 3)) if "bgr" in want else None,
            "bbox": self._new((B, 4), torch.int32),
        }
        K9 = farr(np.asarray(K, np.float32).reshape(9), 9)
        means = farr(pixel_means_rgb, 3, C.c_double)
        check(lib.dim_render(self._h, _p(cls_idx), _p(pose), B, K9, znear, zfar, means, int(trunc_u8), _p(out["image"]),
                             _p(out["depth"]), _p(out["mask"]), _p(out["bgr"]), _p(out["bbox"]), self._stream()))
        return out

    def render_lit(self, cls_idx, pose, K, light_position, light_intensity, brightness_ratio=0.7, znear=0.25, zfar=6.0,
                   pixel_means_rgb=(0, 0, 0), want=("bgr", "depth")):
        """Lambert-lit render (render_py_light_modelnet_multi.py:131-175).  light_position / light_intensity float32[B,3]
        CUDA tensors (position in the GL camera frame)."""
        B = pose.shape[0]
        _chk(pose, torch.float32, (B, 3, 4), "pose")
        _chk(cls_idx, torch.int32, (B,), "cls_idx")
        _chk(light_position, torch.float32, (B, 3), "light_position")
        _chk(light_intensity, torch.float32, (B, 3), "light_intensity")
        out = {
            "image": self._new((B, 3, self.H, self.W)) if "image" in want else None,
            "depth": self._new((B, 1, self.H, self.W)) if "depth" in want else None,
            "mask": self._new((B, 1, self.H, self.W)) if "mask" in want else None,
            "bgr": self._new((B, self.H, self.W, 3)) if "bgr" in want else None,
            "bbox": self._new((B, 4), torch.int32),
        }
        check(lib.dim_render_lit(self._h, _p(cls_idx), _p(pose), B, farr(np.asarray(K, np.float32).reshape(9), 9), znear, zfar,
                                 farr(pixel_means_rgb, 3, C.c_double), _p(light_position), _p(light_intensity),
                                 float(np.float32(brightness_ratio)), _p(out["image"]), _p(out["depth"]), _p(out["mask"]),
                                 _p(out["bgr"]), _p(out["bbox"]), self._stream()))
        return out

    def render_dataset(self, cls_idx, pose, K, znear=0.25, zfar=6.0, depth_factor=1000.0, light_position=None,
                       light_intensity=None, brightness_ratio=None, want=("bgr", "depth", "label")):
        """dim_render_dataset: the dataset files' images from one rasterisation (toolkit/LM6d_ds_1, ds_2, ds_4, LM6d_0).
        want names the outputs: "lit_bgr" uint8 [B,H,W,3] (Render_Py_Light colour; needs light_position / light_intensity
        float32 [B,3] (GL camera frame) and brightness_ratio float32 [B], CUDA tensors), "bgr" uint8 [B,H,W,3] (unlit
        Render_Py colour), "depth" uint16 [B,H,W] (depth * depth_factor, truncated), "label" uint8 [B,H,W] (depth != 0)."""
        B = pose.shape[0]
        _chk(pose, torch.float32, (B, 3, 4), "pose")
        _chk(cls_idx, torch.int32, (B,), "cls_idx")
        lit = "lit_bgr" in want
        if lit:
            _chk(light_position, torch.float32, (B, 3), "light_position")
            _chk(light_intensity, torch.float32, (B, 3), "light_intensity")
            _chk(brightness_ratio, torch.float32, (B,), "brightness_ratio")
        elif light_position is not None or light_intensity is not None or brightness_ratio is not None:
            raise ValueError("render_dataset: the light arguments are used only for 'lit_bgr', which `want` does not name")
        out = {
            "lit_bgr": self._new((B, self.H, self.W, 3), torch.uint8) if lit else None,
            "bgr": self._new((B, self.H, self.W, 3), torch.uint8) if "bgr" in want else None,
            "depth": self._new((B, self.H, self.W), torch.uint16) if "depth" in want else None,
            "label": self._new((B, self.H, self.W), torch.uint8) if "label" in want else None,
        }
        check(lib.dim_render_dataset(self._h, _p(cls_idx), _p(pose), B, farr(np.asarray(K, np.float32).reshape(9), 9), znear,
                                     zfar, float(depth_factor), _p(light_position), _p(light_intensity), _p(brightness_ratio),
                                     _p(out["lit_bgr"]), _p(out["bgr"]), _p(out["depth"]), _p(out["label"]), self._stream()))
        return {k: v for k, v in out.items() if v is not None}

    # -------------------------------------------------------------------------------- zoom
    def zoom_mask(self, mask_observed, mask_gt_observed, mask_rendered, src_pose, K):
        B = mask_observed.shape[0]
        shp = (B, 1, self.H, self.W)
        for n, t in (("mask_observed", mask_observed), ("mask_gt_observed", mask_gt_observed),
                     ("mask_rendered", mask_rendered)):
            _chk(t, torch.float32, shp, n)
        _chk(src_pose, torch.float32, (B, 3, 4), "src_pose")
        zo, zg, zr = self._new(shp), self._new(shp), self._new(shp)
        zf = self._new((B, 4))
        bbox = self._new((B, 8), torch.int32)
        status = self._new((B,), torch.int32)
        K9 = farr(np.asarray(K, np.float32).reshape(9), 9)
        check(lib.dim_zoom_mask_fwd(self._h, _p(mask_observed), _p(mask_gt_observed), _p(mask_rendered), _p(src_pose), B,
                                    K9, _p(zo), _p(zg), _p(zr), _p(zf), _p(bbox), _p(status), self._stream()))
        return zo, zg, zr, zf, bbox, status

    def zoom_image_with_factor(self, zoom_factor, image_observed, image_rendered, pixel_means_rgb):
        B = image_observed.shape[0]
        shp = (B, 3, self.H, self.W)
        _chk(image_observed, torch.float32, shp, "image_observed")
        _chk(image_rendered, torch.float32, shp, "image_rendered")
        _chk(zoom_factor, torch.float32, (B, 4), "zoom_factor")
        zo, zr = self._new(shp), self._new(shp)
        check(lib.dim_zoom_image_with_factor_fwd(self._h, _p(zoom_factor), _p(image_observed), _p(image_rendered), B,
                                                 farr(pixel_means_rgb, 3), _p(zo), _p(zr), self._stream()))
        return zo, zr

    def zoom_image(self, image_observed, image_rendered, src_pose, K, pixel_means_rgb):
        """ZoomImage (zoom_image.py:26-107): boxes from sum_c(image + mean) > 0.01."""
        B = image_observed.shape[0]
        shp = (B, 3, self.H, self.W)
        _chk(image_observed, torch.float32, shp, "image_observed")
        _chk(image_rendered, torch.float32, shp, "image_rendered")
        _chk(src_pose, torch.float32, (B, 3, 4), "src_pose")
        zo, zr, zf = self._new(shp), self._new(shp), self._new((B, 4))
        bbox, status = self._new((B, 8), torch.int32), self._new((B,), torch.int32)
        check(lib.dim_zoom_image_fwd(self._h, _p(image_observed), _p(image_rendered), _p(src_pose), B,
                                     farr(np.asarray(K, np.float32).reshape(9), 9), farr(pixel_means_rgb, 3), _p(zo), _p(zr),
                                     _p(zf), _p(bbox), _p(status), self._stream()))
        return zo, zr, zf, bbox, status

    def group_picker(self, data, group_idx, group_num, backward=False, channels=None):
        """GroupPicker (group_picker.py:22-56).  forward: data [B,C,...] -> [B,C/group_num,...];
        backward: data = out_grad [B,C/group_num,...] -> [B,channels,...] (zero outside the picked group)."""
        B = data.shape[0]
        Ctot = channels if backward else data.shape[1]
        n = int(np.prod(data.shape[2:])) if data.dim() > 2 else 1
        gi = group_idx.reshape(-1).to(torch.float32).contiguous()
        _chk(data, torch.float32, tuple(data.shape), "data")
        out = self._new((B, Ctot if backward else Ctot // group_num) + tuple(data.shape[2:]))
        check(lib.dim_group_picker(self._h, _p(data), _p(gi), B, Ctot, group_num, n, int(backward), _p(out), self._stream()))
        return out

    def zoom_mask_with_factor(self, zoom_factor, mask, b_inv_zoom):
        B = mask.shape[0]
        _chk(mask, torch.float32, (B, 1, self.H, self.W), "mask")
        out = self._new(mask.shape)
        check(lib.dim_zoom_mask_with_factor_fwd(self._h, _p(zoom_factor), _p(mask), B, int(b_inv_zoom), _p(out),
                                                self._stream()))
        return out

    def zoom_flow(self, zoom_factor, flow, flow_weights=None, b_inv_zoom=False):
        B = flow.shape[0]
        _chk(flow, torch.float32, (B, 2, self.H, self.W), "flow")
        out = self._new(flow.shape)
        outw = None
        fwc = 1
        if not b_inv_zoom and flow_weights is not None:
            fwc = flow_weights.shape[1]  # 1, or 2 when tiled like batch_updater_py_multi.py:293-296
            _chk(flow_weights, torch.float32, (B, fwc, self.H, self.W), "flow_weights")
            outw = self._new(flow_weights.shape)
        check(lib.dim_zoom_flow_fwd(self._h, _p(zoom_factor), _p(flow), _p(flow_weights), fwc, B, int(b_inv_zoom), _p(out),
                                    _p(outw), self._stream()))
        return out, outw

    def zoom_depth(self, zoom_factor, depth_observed, depth_rendered):
        B = depth_observed.shape[0]
        zo, zr = self._new(depth_observed.shape), self._new(depth_rendered.shape)
        check(lib.dim_zoom_depth_fwd(self._h, _p(zoom_factor), _p(depth_observed), _p(depth_rendered), B, _p(zo), _p(zr),
                                     self._stream()))
        return zo, zr

    def zoom_trans(self, zoom_factor, trans, b_inv_zoom):
        B = trans.shape[0]
        _chk(trans, torch.float32, (B, 3), "trans_delta")
        out = self._new((B, 3))
        check(lib.dim_zoom_trans_fwd(self._h, _p(zoom_factor), _p(trans), B, int(b_inv_zoom), _p(out), self._stream()))
        return out

    def zoom_trans_backward(self, zoom_factor, out_grad, b_inv_zoom, b_zoom_grad):
        B = out_grad.shape[0]
        out = self._new((B, 3))
        check(lib.dim_zoom_trans_bwd(self._h, _p(zoom_factor), _p(out_grad), B, int(b_inv_zoom), int(b_zoom_grad),
                                     _p(out), self._stream()))
        return out

    def update_mask_box(self, bbox4):
        B = bbox4.shape[0]
        _chk(bbox4, torch.int32, (B, 4), "bbox")
        out = self._new((B, 1, self.H, self.W))
        check(lib.dim_update_mask_box(self._h, _p(bbox4), B, _p(out), self._stream()))
        return out

    # ---------------------------------------------------------------------------- geometry
    def se3_compose(self, pose_src, se3, T_means=(0, 0, 0), T_stds=(1, 1, 1), rot_coord="camera"):
        B = pose_src.shape[0]
        _chk(pose_src, torch.float64, (B, 3, 4), "pose_src")
        _chk(se3, torch.float32, (B, 7), "se3")
        out = self._new((B, 3, 4), torch.float64)
        check(lib.dim_se3_compose(self._h, _p(pose_src), _p(se3), B, farr(T_means, 3, C.c_double),
                                  farr(T_stds, 3, C.c_double), capi.ROT_COORD[rot_coord.lower()], _p(out), self._stream()))
        return out

    def flow(self, depth_src, depth_tgt, KT, Kinv):
        B = depth_src.shape[0]
        shp = (B, 1, self.H, self.W)
        _chk(depth_src, torch.float32, shp, "depth_src")
        _chk(depth_tgt, torch.float32, shp, "depth_tgt")
        _chk(KT, torch.float32, (B, 3, 4), "KT")
        fl, va = self._new((B, 2, self.H, self.W)), self._new(shp)
        check(lib.dim_flow_fwd(self._h, _p(depth_src), _p(depth_tgt), _p(KT), farr(np.asarray(Kinv, np.float32).reshape(9), 9),
                               B, _p(fl), _p(va), self._stream()))
        return fl, va

    def transform3d(self, point_cloud, rotation, translation, pose_src, T_means, T_stds, rot_coord="model"):
        B, _, N = point_cloud.shape
        out = self._new(point_cloud.shape)
        check(lib.dim_transform3d_fwd(self._h, _p(point_cloud), _p(rotation), _p(translation), _p(pose_src), B, N,
                                      farr(T_means, 3), farr(T_stds, 3), capi.ROT_COORD[rot_coord.lower()], _p(out),
                                      self._stream()))
        return out

    def transform3d_backward(self, out_grad, point_cloud, rotation, translation, pose_src, T_means, T_stds,
                             rot_coord="model"):
        B, _, N = point_cloud.shape
        rg, tg = self._new((B, 4)), self._new((B, 3))
        check(lib.dim_transform3d_bwd(self._h, _p(out_grad), _p(point_cloud), _p(rotation), _p(translation),
                                      _p(pose_src), B, N, farr(T_means, 3), farr(T_stds, 3),
                                      capi.ROT_COORD[rot_coord.lower()], _p(rg), _p(tg), self._stream()))
        return rg, tg

    def train_update(self, cls_idx, src_pose, rot_est, trans_est, tgt_pose, depth_gt_observed, K,
                     pixel_means_rgb=(103.939, 116.779, 123.68), T_means=(0, 0, 0), T_stds=(1, 1, 1),
                     rot_coord="camera", znear=0.25, zfar=6.0, want_flow=True, lighting=None):
        """batchUpdaterPyMulti.forward on the device (lib/pair_matching/batch_updater_py_multi.py:91-328).
        T_means / T_stds / rot_coord: the pose parameterisation of rot_est / trans_est and of the labels.  The defaults are
        the standalone operator's; inside a training loop pass the context's (get_config()), which the training step's
        Transform3D and refine() use, as the reference composes with network.ROT_COORD and dataset.trans_means / trans_stds
        (l.23-27, 179-180).  trainer.fit_batch does.
        lighting: None = the unlit re-render (LINEMOD); a dict {intensity float32 [B,3] CUDA, offset, brightness_ratio}
        = the ModelNet branch's lit re-render (l.187-229; see deepim_b200.lighting), every other output unchanged."""
        B = src_pose.shape[0]
        for n, t, shp in (("src_pose", src_pose, (B, 3, 4)), ("tgt_pose", tgt_pose, (B, 3, 4)), ("rot_est", rot_est, (B, 4)),
                          ("trans_est", trans_est, (B, 3))):
            _chk(t, torch.float32, shp, n)
        _chk(cls_idx, torch.int32, (B,), "cls_idx")
        out = {
            "image_rendered": self._new((B, 3, self.H, self.W)), "depth_rendered": self._new((B, 1, self.H, self.W)),
            "mask_rendered": self._new((B, 1, self.H, self.W)), "src_pose": self._new((B, 3, 4)),
            "rot": self._new((B, 4)), "trans": self._new((B, 3)),
            "flow": self._new((B, 2, self.H, self.W)) if want_flow else None,
            "flow_weights": self._new((B, 2, self.H, self.W)) if want_flow else None,
        }
        if want_flow:
            _chk(depth_gt_observed, torch.float32, (B, 1, self.H, self.W), "depth_gt_observed")
        lit = None if lighting is None else C.byref(_lighting_arg(lighting, (B, 3), True)[0])
        check(lib.dim_train_update(self._h, _p(cls_idx), _p(src_pose), _p(rot_est), _p(trans_est), _p(tgt_pose),
                                   _p(depth_gt_observed) if want_flow else None, B,
                                   farr(np.asarray(K, np.float64).reshape(9), 9, C.c_double), znear, zfar,
                                   farr(pixel_means_rgb, 3, C.c_double), farr(T_means, 3, C.c_double),
                                   farr(T_stds, 3, C.c_double), capi.ROT_COORD[rot_coord.lower()],
                                   _p(out["image_rendered"]), _p(out["depth_rendered"]), _p(out["mask_rendered"]),
                                   _p(out["src_pose"]), _p(out["rot"]), _p(out["trans"]), _p(out["flow"]),
                                   _p(out["flow_weights"]), lit, self._stream()))
        return out

    def transform_image_u8(self, bgr_u8, pixel_means_rgb):
        B = bgr_u8.shape[0]
        _chk(bgr_u8, torch.uint8, (B, self.H, self.W, 3), "bgr_u8")
        out = self._new((B, 3, self.H, self.W))
        check(lib.dim_transform_image_u8(self._h, _p(bgr_u8), B, farr(pixel_means_rgb, 3, C.c_double), _p(out), self._stream()))
        return out

    # -------------------------------------------------------------------------- augmentation
    def replace_background(self, observed_bgr, mask, bg_index, pixel_means_rgb, want_composite=False):
        """dim_replace_background (image.py:96-157): observed_bgr float32 [B,H,W,3] BGR in [0,255] (render's "bgr"),
        mask float32 [B,1,H,W] (!= 0 keeps the observed pixel), bg_index host int32 [B] photo of the context's background
        bank (deepim_b200.augment.BackgroundBank) or -1 = keep.  Returns image_observed float32 [B,3,H,W] (RGB - means),
        and with want_composite also the uint8 BGR composite [B,H,W,3]."""
        B = observed_bgr.shape[0]
        _chk(observed_bgr, torch.float32, (B, self.H, self.W, 3), "observed_bgr")
        _chk(mask, torch.float32, (B, 1, self.H, self.W), "mask")
        idx = np.ascontiguousarray(bg_index, np.int32)
        if idx.shape != (B,):
            raise ValueError("bg_index: expected shape (%d,), got %s" % (B, idx.shape))
        out = self._new((B, 3, self.H, self.W))
        comp = self._new((B, self.H, self.W, 3), torch.uint8) if want_composite else None
        check(lib.dim_replace_background(self._h, _p(observed_bgr), _p(mask), idx.ctypes.data, B,
                                         farr(pixel_means_rgb, 3, C.c_double), _p(out), _p(comp), self._stream()))
        return (out, comp) if want_composite else out

    def mask_dilate(self, mask, draws):
        """dim_mask_dilate (mask_dilate.py:19-47): mask float32 [B,1,H,W]; draws int32 [B,5] (host or CUDA; see
        deepim_b200.augment.mask_dilate_draws).  Returns the dilated mask (a new tensor)."""
        B = mask.shape[0]
        _chk(mask, torch.float32, (B, 1, self.H, self.W), "mask")
        d = torch.as_tensor(np.asarray(draws, np.int32) if not isinstance(draws, torch.Tensor) else draws)
        d = d.to(self.device).contiguous()
        _chk(d, torch.int32, (B, 5), "draws")
        out = self._new(mask.shape)
        check(lib.dim_mask_dilate(self._h, _p(mask), _p(d), B, _p(out), self._stream()))
        return out

    # --------------------------------------------------------------------------------- net
    def net_forward(self, zoom_image_observed, zoom_image_rendered, zoom_mask_observed=None, zoom_mask_rendered=None,
                    precision=capi.PREC_BF16X3, zoom_depth_observed=None, zoom_depth_rendered=None):
        """The network on already-zoomed blobs; an RGB-D context (input_depth=True) also takes the zoomed depths
        f32 [B,1,H,W] (metres); an image-only context (input_mask=False) takes no masks (None)."""
        B = zoom_image_observed.shape[0]
        for n, t in (("zoom_depth_observed", zoom_depth_observed), ("zoom_depth_rendered", zoom_depth_rendered)):
            if t is not None:
                _chk(t, torch.float32, (B, 1, self.H, self.W), n)
        rot, trans = self._new((B, 4)), self._new((B, 3))
        check(lib.dim_net_fwd(self._h, _p(zoom_image_observed), _p(zoom_image_rendered), _p(zoom_depth_observed),
                              _p(zoom_depth_rendered), _p(zoom_mask_observed), _p(zoom_mask_rendered), B, precision,
                              _p(rot), _p(trans), self._stream()))
        return rot, trans

    def debug_activation(self, idx, B, lo=False, fp16=False):
        """16-bit NHWC activation buffer feeding conv layer idx (10 = fc6 input) as float32 numpy
        [B, rows, cols, C] including the zero border (fp16=True: the last pass ran in DIM_PREC_FP16)."""
        g = (C.c_int32 * 8)()
        check(lib.dim_debug_layer_geometry(self._h, idx, g))
        rows, cols, ch = g[0], g[1], g[2]
        n = B * rows * cols * ch
        buf = np.empty(n, np.uint16)
        torch.cuda.synchronize()
        check(lib.dim_debug_activation(self._h, idx, int(lo), buf.ctypes.data, n * 2))
        f = buf.view(np.float16).astype(np.float32) if fp16 else (buf.astype(np.uint32) << 16).view(np.float32)
        return f.reshape(B, rows, cols, ch), tuple(g)

    def debug_train_update(self, B):
        """What the last train_update of B instances computed besides its outputs (dim_debug_train_update): float32 numpy
        KT [B,3,4] = K . calc_se3(refined, tgt), the matrix of its flow labels, and the light position [B,3] of its lit
        re-render (meaningful after a call with lighting)"""
        kt, light = np.empty((B, 3, 4), np.float32), np.empty((B, 3), np.float32)
        check(lib.dim_debug_train_update(self._h, B, kt.ctypes.data_as(capi.pf32), light.ctypes.data_as(capi.pf32)))
        return kt, light

    # ------------------------------------------------------------------------------ refine
    def get_config(self) -> dict:
        """dim_train_get_config: loss weights / normalisers / pose parameterisation in effect on this context"""
        cfg = capi.TrainConfig()
        check(lib.dim_train_get_config(self._h, C.byref(cfg)))
        return {"lw_flow": cfg.lw_flow, "lw_mask": cfg.lw_mask, "lw_pm": cfg.lw_pm, "num_3d_sample": cfg.num_3d_sample,
                "normalize_3d_point": cfg.normalize_3d_point, "normalize_flow": cfg.normalize_flow,
                "trans_means": list(cfg.trans_means), "trans_stds": list(cfg.trans_stds),
                "rot_coord": "CAMERA" if cfg.rot_coord == 1 else "MODEL"}

    def set_config(self, **fields):
        """dim_train_set_config: override some of the yaml-level constants (see get_config for the names).  trans_means /
        trans_stds / rot_coord also drive refine(); the rest applies to the training step."""
        cfg = capi.TrainConfig()
        check(lib.dim_train_get_config(self._h, C.byref(cfg)))
        for k, v in fields.items():
            if k in ("trans_means", "trans_stds"):
                setattr(cfg, k, (C.c_float * 3)(*[float(x) for x in v]))
            elif k == "rot_coord":
                cfg.rot_coord = capi.ROT_COORD[v.lower()] if isinstance(v, str) else int(v)
            elif hasattr(cfg, k):
                setattr(cfg, k, float(v))
            else:
                raise ValueError("unknown config field %r" % k)
        check(lib.dim_train_set_config(self._h, C.byref(cfg)))

    def refine(self, image_observed, cls_idx, pose_init, K, n_iter=4, znear=0.25, zfar=6.0,
               pixel_means_rgb=(103.939, 116.779, 123.68), precision=capi.PREC_FP16, pose_override=None, out=None,
               lighting=None, depth_observed=None):
        """Device-resident fused loop.  image_observed f32[B,3,H,W], cls_idx i32[B], pose_init f64[B,3,4].
        out = the dict returned by an earlier call with the same shapes: results are written into those tensors again
        (same device addresses -> the library replays its CUDA graph of the chain instead of re-enqueuing ~90 launches).
        lighting: None = the unlit loop (LINEMOD); a dict {intensity float32 [n_iter,B,3] CUDA, offset, brightness_ratio}
        = the ModelNet branch's lit loop (see deepim_b200.lighting).  Reusing the same intensity tensor lets the lit chain
        replay its graph as well.
        depth_observed: f32 [B,1,H,W] CUDA, metres -- required on an RGB-D context (input_depth=True), refused otherwise."""
        return self._refine(image_observed, None, cls_idx, pose_init, np.asarray(K, np.float32).reshape(3, 3), n_iter, znear,
                            zfar, pixel_means_rgb, precision, pose_override, out, lighting, depth_observed,
                            ("image_observed", "depth_observed"))

    def refine_host(self, image_observed_u8, cls_idx, pose_init, K, n_iter=4, znear=0.25, zfar=6.0,
                    pixel_means_rgb=(103.939, 116.779, 123.68), precision=capi.PREC_FP16, poses_out=None,
                    se3_out=None, sync=True, lighting=None, depth_observed_u16=None, depth_factor=1000.0):
        """Host-buffer entry (what a tester loop calls): uint8 BGR HWC images (pinned torch tensors or
        numpy), host poses in / out.  sync=False only enqueues on the current torch stream (outputs must
        then be pinned and are valid after the stream is synchronised).
        lighting: as refine() but with a HOST intensity array float32 [n_iter,B,3] (copied before the call returns,
        unless it is pinned: then it must stay untouched until the stream is synchronised).
        depth_observed_u16: RGB-D context only, host uint16 [B,H,W] depth file values (the *-depth.png of the observed
        frame); the device converts them as the reference's loader does, float32(u16) / float32(depth_factor).  With
        sync=False a pinned depth array is copied asynchronously too: keep it untouched until the stream is synchronised."""
        return self._refine_host(image_observed_u8, None, cls_idx, pose_init, np.asarray(K, np.float32).reshape(3, 3), n_iter,
                                 znear, zfar, pixel_means_rgb, precision, poses_out, se3_out, sync, lighting,
                                 depth_observed_u16, depth_factor, ("image_observed_u8", "depth_observed_u16"))

    def refine_frames(self, frames, frame_idx, cls_idx, pose_init, K, n_iter=4, znear=0.25, zfar=6.0,
                      pixel_means_rgb=(103.939, 116.779, 123.68), precision=capi.PREC_FP16, pose_override=None, out=None,
                      lighting=None, depth_frames=None):
        """refine() against F shared observed frames: frames f32[F,3,H,W] (RGB - mean), frame_idx i32[B] CUDA (instance b
        observes frames[frame_idx[b]]), 1 <= F <= max_batch.  Instance b's results equal refine(frames[frame_idx], ...)'s, bit
        for bit; each frame is packed once.  An index outside [0, F) is not an error here: that instance observes frame 0
        and refine_status() reports bit 3.  Writing new indices into the same frame_idx tensor replays the captured graph.
        depth_frames: f32 [F,1,H,W] CUDA, metres -- required on an RGB-D context, refused otherwise.
        K: [3,3], one camera for every instance, or [F,3,3], one camera per frame: instance b is rendered and zoomed with
        K[frame_idx[b]], and its results equal refine_frames(..., K=K[frame_idx[b]]) bit for bit.  A float32 CUDA tensor
        [F,3,3] is read in place, also at graph replay: new intrinsics written into it need no re-capture; any other [F,3,3]
        array is copied to the device first.  Every other argument as refine()."""
        return self._refine(frames, frame_idx, cls_idx, pose_init, K, n_iter, znear, zfar, pixel_means_rgb, precision,
                            pose_override, out, lighting, depth_frames, ("frames", "depth_frames"))

    def refine_frames_host(self, frames_u8, frame_idx, cls_idx, pose_init, K, n_iter=4, znear=0.25, zfar=6.0,
                           pixel_means_rgb=(103.939, 116.779, 123.68), precision=capi.PREC_FP16, poses_out=None,
                           se3_out=None, sync=True, lighting=None, depth_frames_u16=None, depth_factor=1000.0):
        """refine_host() against F shared observed frames: frames_u8 uint8 [F,H,W,3] BGR, frame_idx int32 [B] (host; every
        index is checked: one outside [0, F) raises before anything is enqueued), depth_frames_u16 uint16 [F,H,W] on an
        RGB-D context.  Each frame is uploaded once.
        K: [3,3], or [F,3,3] host float32, one camera per frame (see refine_frames): every row must be a finite pinhole
        matrix [[fx,0,cx],[0,fy,cy],[0,0,1]] with fx, fy > 0, else the call raises naming the frame before anything is
        enqueued.  With sync=False a pinned K is copied asynchronously: keep it untouched until the stream is synchronised.
        Every other argument as refine_host()."""
        return self._refine_host(frames_u8, frame_idx, cls_idx, pose_init, K, n_iter, znear, zfar, pixel_means_rgb,
                                 precision, poses_out, se3_out, sync, lighting, depth_frames_u16, depth_factor,
                                 ("frames_u8", "depth_frames_u16"))

    def _refine(self, frames, frame_idx, cls_idx, pose_init, K, n_iter, znear, zfar, pixel_means_rgb, precision,
                pose_override, out, lighting, depth, names):
        """refine / refine_frames: one dim_refine call.  frame_idx None = instance b observes frames[b]; K [3,3] or [F,3,3]
        (_per_frame_k); names = the caller's names of the frames and depth arguments, for the messages."""
        F, B, K9, K_frames = self._frame_batch(frames, frame_idx, cls_idx, K)
        _chk(frames, torch.float32, (F, 3, self.H, self.W), names[0])
        _chk(pose_init, torch.float64, (B, 3, 4), "pose_init")
        if out is not None:
            poses, se3, zf, bbox = out["poses"], out["se3"], out["zoom_factor"], out["bbox"]
            _chk(poses, torch.float64, (n_iter, B, 3, 4), "out['poses']")
            _chk(se3, torch.float32, (n_iter, B, 7), "out['se3']")
            _chk(zf, torch.float32, (n_iter, B, 4), "out['zoom_factor']")
            _chk(bbox, torch.int32, (n_iter, B, 8), "out['bbox']")
        else:
            poses = self._new((n_iter, B, 3, 4), torch.float64)
            se3 = self._new((n_iter, B, 7))
            zf = self._new((n_iter, B, 4))
            bbox = self._new((n_iter, B, 8), torch.int32)
        if pose_override is not None:
            _chk(pose_override, torch.float64, (n_iter, B, 3, 4), "pose_override")
        if depth is not None:
            _chk(depth, torch.float32, (F, 1, self.H, self.W), names[1])
        lit = None if lighting is None else C.byref(_lighting_arg(lighting, (n_iter, B, 3), True)[0])
        check(lib.dim_refine(self._h, _p(frames), F, _p(frame_idx), K9, _p(K_frames), _p(cls_idx), _p(pose_init), B, n_iter,
                             znear, zfar, farr(pixel_means_rgb, 3, C.c_double), precision, _p(pose_override), _p(poses),
                             _p(se3), _p(zf), _p(bbox), _p(depth), lit, self._stream()))
        return {"poses": poses, "se3": se3, "zoom_factor": zf, "bbox": bbox}

    def _refine_host(self, frames_u8, frame_idx, cls_idx, pose_init, K, n_iter, znear, zfar, pixel_means_rgb, precision,
                     poses_out, se3_out, sync, lighting, depth_u16, depth_factor, names):
        """refine_host / refine_frames_host / PoseRefiner: one dim_refine_host_async call, then (sync) a synchronise of the
        stream.  frame_idx None = instance b observes frames_u8[b]; K [3,3] or [F,3,3] (_per_frame_k); names = the caller's
        names of the frames and depth arguments, for the messages."""
        fidx = None if frame_idx is None else _host(frame_idx, np.int32, torch.int32, "frame_idx")
        cls = _host(cls_idx, np.int32, torch.int32, "cls_idx")
        pose = _host(pose_init, np.float64, torch.float64, "pose_init")
        F, B, K9, K_frames = self._frame_batch(frames_u8, fidx, cls, K, host=True)
        if tuple(frames_u8.shape) != (F, self.H, self.W, 3):
            raise ValueError("%s: expected shape %s, got %s" % (names[0], (F, self.H, self.W, 3), tuple(frames_u8.shape)))
        if poses_out is None:
            poses_out = np.empty((n_iter, B, 3, 4), np.float64)
        if se3_out is None:
            se3_out = np.empty((n_iter, B, 7), np.float32)
        dkeep = None
        if depth_u16 is not None:
            dkeep = _host(depth_u16, np.uint16, torch.uint16, names[1])
            if tuple(dkeep.shape) != (F, self.H, self.W):
                raise ValueError("%s: expected shape %s, got %s" % (names[1], (F, self.H, self.W), tuple(dkeep.shape)))
        frames = frames_u8 if isinstance(frames_u8, torch.Tensor) else np.ascontiguousarray(frames_u8, np.uint8)
        lit, _keep = (None, None) if lighting is None else _lighting_arg(lighting, (n_iter, B, 3), False)
        check(lib.dim_refine_host_async(self._h, hptr(frames), F, None if fidx is None else hptr(fidx), K9,
                                        None if K_frames is None else hptr(K_frames), hptr(cls), hptr(pose), B, n_iter, znear,
                                        zfar, farr(pixel_means_rgb, 3, C.c_double), precision, hptr(poses_out),
                                        hptr(se3_out), None if dkeep is None else hptr(dkeep), float(np.float32(depth_factor)),
                                        None if lit is None else C.byref(lit), self._stream()))
        if sync:
            torch.cuda.current_stream(self.device).synchronize()
        return poses_out, se3_out


    # ------------------------------------------------------------------------------ ICP
    def icp(self, depth_frames, cls_idx, poses, K, n_iter=10, max_dist=0.02, min_points=64, frame_idx=None, znear=0.25,
            zfar=6.0):
        """Projective point-to-plane ICP of poses against observed depth (dim_icp; the contract is oracle/icp.py): the model
        surface is rendered once at float32(poses), then n_iter Gauss-Newton steps, all in float64.
        depth_frames f32 [F,H,W] (or [F,1,H,W]) CUDA, metres, 0 = hole; cls_idx i32 [B] CUDA; poses f64 [B,3,4] CUDA.
        frame_idx None = instance b observes frame b (F == B), else i32 [B] CUDA (an index outside [0, F) means frame 0 and
        status bit 3).  K: [3,3] (one camera) or [F,3,3] (one per frame), as refine_frames.
        max_dist (metres) bounds the inlier depth residual and the depth step between neighbouring model pixels;
        min_points is the fewest inliers an update needs.  The defaults (10 iterations, 2 cm, 64 points) are starting
        values and have not been tuned.
        Returns CUDA tensors: poses f64 [n_iter,B,3,4] (after each iteration), inliers i32 [n_iter,B], rms f32 [n_iter,B]
        (both before that iteration's update), status i32 [n_iter,B] (bit 0 no model pixel, bit 1 bad class, bit 3 frame
        index out of range, bit 4 too few inliers or a singular system; with bit 0 or 4 the pose is unchanged)."""
        F, B, K9, K_frames = self._frame_batch(depth_frames, frame_idx, cls_idx, K)
        _chk(depth_frames, torch.float32, (F, 1, self.H, self.W) if depth_frames.dim() == 4 else (F, self.H, self.W),
             "depth_frames")
        _chk(poses, torch.float64, (B, 3, 4), "poses")
        out = {"poses": self._new((n_iter, B, 3, 4), torch.float64), "inliers": self._new((n_iter, B), torch.int32),
               "rms": self._new((n_iter, B)), "status": self._new((n_iter, B), torch.int32)}
        check(lib.dim_icp(self._h, _p(depth_frames), F, _p(frame_idx), K9, _p(K_frames), _p(cls_idx), _p(poses), B, n_iter,
                          znear, zfar, float(max_dist), int(min_points), _p(out["poses"]), _p(out["inliers"]), _p(out["rms"]),
                          _p(out["status"]), self._stream()))
        return out

    def pose_error_vsd(self, depth_frames, cls_idx, poses_est, poses_gt, K, delta=0.015, taus=(0.02,), frame_idx=None,
                       znear=0.25, zfar=6.0, visib_mode="sixd17", diameters=None):
        """Visible Surface Discrepancy of poses_est against poses_gt (dim_pose_error_vsd; Hodan et al., ECCVW 2016; the
        contract is oracle/vsd.py): both poses are rendered at float32, and the visible surfaces are compared against the
        observed depth with tolerance delta (metres) and the step cost at each tau (metres, at most 16 of them).
        depth_frames f32 [F,H,W] (or [F,1,H,W]) CUDA, metres, 0 = hole; cls_idx i32 [B] CUDA; poses_est / poses_gt f64
        [B,3,4] CUDA; frame_idx and K as icp.
        visib_mode "sixd17" (default) is the SIXD 2017 visibility; "bop19" is BOP 2019's, where sensor holes count as
        visible.  diameters: None (taus in metres) or [B] host values in metres, each finite and > 0, making the taus
        fractions of each instance's diameter, as BOP 2019 does (dim_pose_error_vsd_ex; the contract is oracle/bop.py's vsd()).
        Returns CUDA tensors: err f64 [B,n_tau] (1 = worst; 1 when neither pose leaves a visible pixel) and status i32 [B]
        (bit 0 empty union, bit 1 bad class, bit 3 frame index out of range)."""
        if visib_mode not in VISIB_MODES:
            raise ValueError("visib_mode must be one of %s, got %r" % (tuple(VISIB_MODES), visib_mode))
        F, B, K9, K_frames = self._frame_batch(depth_frames, frame_idx, cls_idx, K)
        _chk(depth_frames, torch.float32, (F, 1, self.H, self.W) if depth_frames.dim() == 4 else (F, self.H, self.W),
             "depth_frames")
        _chk(poses_est, torch.float64, (B, 3, 4), "poses_est")
        _chk(poses_gt, torch.float64, (B, 3, 4), "poses_gt")
        taus = np.ascontiguousarray(np.asarray(taus, np.float64).reshape(-1))
        diam = None
        if diameters is not None:
            diam = np.ascontiguousarray(np.asarray(diameters, np.float64).reshape(-1))
            if diam.shape != (B,):
                raise ValueError("diameters: expected shape %s, got %s" % ((B,), diam.shape))
        out = {"err": self._new((B, len(taus)), torch.float64), "status": self._new((B,), torch.int32)}
        args = (self._h, _p(depth_frames), F, _p(frame_idx), K9, _p(K_frames), _p(cls_idx), _p(poses_est), _p(poses_gt), B,
                znear, zfar, float(delta), farr(taus, ctype=C.c_double), len(taus))
        tail = (_p(out["err"]), _p(out["status"]), self._stream())
        if visib_mode == "sixd17" and diam is None:
            check(lib.dim_pose_error_vsd(*args, *tail))
        else:
            check(lib.dim_pose_error_vsd_ex(*args, VISIB_MODES[visib_mode], None if diam is None else diam.ctypes.data_as(C.POINTER(C.c_double)), *tail))
        return out

    def pose_error_sym(self, poses_est, poses_gt, points, syms, K):
        """BOP 2019's MSSD (metres) and MSPD (pixels) of poses_est against poses_gt over one class's symmetry set
        (dim_pose_error_sym; the contract is oracle/bop.py): the max over the model points, then the min over the symmetries.
        poses_est / poses_gt f64 [M,3,4] CUDA (any M: called in slices of max_batch); points [N,3] and syms [S,3,4] (e.g.
        bop.symmetry_transforms, S <= 4096), float64 CUDA tensors or host arrays; K [3,3] (one camera, broadcast) or [M,3,3].
        A point with Z <= 0 under either pose makes that symmetry's MSPD inf.
        Returns CUDA tensors: err f64 [M,2] (MSSD, MSPD) and sym_idx i32 [M,2] (the minimising symmetry of each, the lowest
        index on ties)."""
        M = poses_est.shape[0]
        _chk(poses_est, torch.float64, (M, 3, 4), "poses_est")
        _chk(poses_gt, torch.float64, (M, 3, 4), "poses_gt")
        dev = lambda a: torch.as_tensor(a, dtype=torch.float64).to(self.device).contiguous()
        pts = dev(points).reshape(-1, 3).contiguous()
        sy = dev(syms).reshape(-1, 3, 4).contiguous()
        Kd = dev(K)
        if Kd.numel() == 9:
            Kd = Kd.reshape(1, 9).expand(M, 9).contiguous()
        elif tuple(Kd.shape) != (M, 3, 3):
            raise ValueError("K: expected shape (3, 3) or %s, got %s" % ((M, 3, 3), tuple(Kd.shape)))
        Kd = Kd.reshape(M, 9)
        out = {"err": self._new((M, 2), torch.float64), "sym_idx": self._new((M, 2), torch.int32)}
        for a in range(0, M, self.max_batch):
            b = min(M, a + self.max_batch)
            check(lib.dim_pose_error_sym(self._h, _p(poses_est[a:b]), _p(poses_gt[a:b]), b - a, _p(pts), pts.shape[0],
                                         _p(sy), sy.shape[0], _p(Kd[a:b]), _p(out["err"][a:b]), _p(out["sym_idx"][a:b]),
                                         self._stream()))
        return out

    def _frame_batch(self, frames, frame_idx, cls_idx, K, host=False):
        """The frame batch of refine*, icp and pose_error_vsd: F = frames.shape[0] frames, instance b observing frame
        frame_idx[b] (None: frame b, so B = F) through K, [3,3] for every instance or [F,3,3] one per frame (_per_frame_k).
        Checks frame_idx and cls_idx, int32 CUDA tensors; host: the refine*_host entries' host arrays (_host), whose K is
        host too.  -> (F, B, K9 host array or None, K_frames or None: a float32 CUDA tensor, K itself when it is one
        already; host: a host array)"""
        F = frames.shape[0]
        B = F if frame_idx is None else cls_idx.shape[0]
        if host:
            if frame_idx is not None and tuple(frame_idx.shape) != (B,):
                raise ValueError("frame_idx: expected shape %s, got %s" % ((B,), tuple(frame_idx.shape)))
        else:
            if frame_idx is not None:
                _chk(frame_idx, torch.int32, (B,), "frame_idx")
            _chk(cls_idx, torch.int32, (B,), "cls_idx")
        if not _per_frame_k(K, F):
            if isinstance(K, torch.Tensor) and not host:
                K = K.cpu()
            return F, B, farr(np.asarray(K, np.float32).reshape(9), 9), None
        if host:
            return F, B, None, _host(K, np.float32, torch.float32, "K")
        if not (isinstance(K, torch.Tensor) and K.device == self.device and K.dtype == torch.float32 and K.is_contiguous()):
            K = torch.as_tensor(np.ascontiguousarray(K.cpu() if isinstance(K, torch.Tensor) else K, np.float32),
                                device=self.device)
        return F, B, None, K

    def depth_from_u16(self, depth_u16, depth_factor=1000.0):
        """uint16 depth file values [F,H,W] CUDA -> metres f32 [F,H,W], float32(u16) / float32(depth_factor) (the
        reference's loader, lib/utils/image.py:203,218)."""
        F = depth_u16.shape[0]
        _chk(depth_u16, torch.uint16, (F, self.H, self.W), "depth_u16")
        out = self._new((F, self.H, self.W))
        check(lib.dim_depth_from_u16(self._h, _p(depth_u16), F, float(np.float32(depth_factor)), _p(out), self._stream()))
        return out


def _refine_status(self, B, n_iter, out=None, sync=True):
    """Per-iteration status of the last refine / refine_host / refine_frames(_host) call: int32 [min(n_iter,8), B]; 0 = ok,
    bit 0 = empty rendered mask in that iteration (pose meaningless; the reference crashes there), bit 1 = bad class index,
    bit 3 = refine_frames: frame index out of range (frame 0 observed).  `out`: pinned int32 tensor for an asynchronous copy
    on the current stream (sync=False)."""
    n = min(int(n_iter), 8)
    if out is None:
        out = torch.empty((n, B), dtype=torch.int32).pin_memory()
    check(lib.dim_refine_status(self._h, B, n_iter, C.c_void_p(out.data_ptr()), self._stream()))
    if sync:
        torch.cuda.current_stream(self.device).synchronize()
    return out


Context.refine_status = _refine_status


def _profile_enable(self, on=True):
    check(lib.dim_profile_enable(self._h, int(on)))


def _profile_read(self):
    """-> (dict stage -> ms accumulated since last read, iterations)"""
    ms = (C.c_float * 4)()
    n = C.c_int32()
    check(lib.dim_profile_read(self._h, ms, C.byref(n)))
    return {"render": ms[0], "zoom": ms[1], "conv": ms[2], "head": ms[3]}, n.value


Context.profile_enable = _profile_enable
Context.profile_read = _profile_read


def launch_count(reset=False):
    return int(lib.dim_launch_count(int(reset)))
