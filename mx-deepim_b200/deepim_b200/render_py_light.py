"""Call-compatible stand-ins for the reference's two lit glumpy renderers, backed by the CUDA rasteriser.

Render_Py_Light_ModelNet_Multi -- lib/render_glumpy/render_py_light_modelnet_multi.py (Lambert-lit renderer of the ModelNet /
unseen-object branch) on dim_render_lit:

    rm = Render_Py_Light_ModelNet_Multi(meshes, K, brightness_ratios=[0.7])
    bgr_u8, depth = rm.render(model_idx, r, t, light_position, light_intensity, brightness_k=0, r_type="mat")

Render_Py_Light -- lib/render_glumpy/render_py_light.py (the renderer of the LM6d_refine_syn observed images,
toolkit/LM6d_ds_1_gen_observed.py), where the light colour scales only the diffuse term, on dim_render_dataset:

    rm = Render_Py_Light(mesh, K, brightness_ratios=[0.2, 0.25, 0.3, 0.35, 0.4])
    bgr_u8, depth = rm.render(r, t, light_position, light_intensity, brightness_k=0, r_type="quat")

As in render_py_multi.py the meshes are deepim_b200.synth.Mesh objects carrying `normals` [V,3] (the reference reads
OBJ files with glumpy); both return (480,640,3) uint8 BGR and (480,640) float32 metres."""
import numpy as np
import torch

from .context import Context
from .render_py_multi import Render_Py
from .toolkit import quat2mat


class Render_Py_Light(Render_Py):
    def __init__(self, mesh, K, width=640, height=480, zNear=0.25, zFar=6.0, brightness_ratios=(0.4, 0.3, 0.2), device=0,
                 ctx=None, mesh_slot=0):
        """mesh: the one model of the reference's model_folder (with normals); ctx / mesh_slot: render mesh `mesh_slot` of an
        existing context instead of a private one"""
        if getattr(mesh, "normals", None) is None:
            raise ValueError("the mesh has no per-vertex normals (synth.vertex_normals / dim_mesh_upload_normals)")
        super().__init__([mesh], ["model"], K, width, height, zNear, zFar, device, ctx)
        self.brightness_ratios = list(brightness_ratios)
        self.mesh_slot = 0 if ctx is None else mesh_slot

    def render(self, r, t, light_position, light_intensity, brightness_k=0, r_type="quat", K=None):
        if r_type == "quat":
            R = quat2mat(r)
        elif r_type == "mat":
            R = np.asarray(r)
        else:
            raise ValueError("unknown r_type %r" % (r_type,))
        dev = self.ctx.device
        pose = torch.from_numpy(np.hstack([R, np.asarray(t).reshape(3, 1)]).astype(np.float32)[None]).to(dev)
        cls = torch.tensor([self.mesh_slot], dtype=torch.int32, device=dev)
        K = self.K if K is None else np.asarray(K, np.float32)
        out = self.ctx.render_dataset(
            cls, pose, K, self.zNear, self.zFar,
            light_position=torch.from_numpy(np.asarray(light_position, np.float32).reshape(1, 3)).to(dev),
            light_intensity=torch.from_numpy(np.asarray(light_intensity, np.float32).reshape(1, 3)).to(dev),
            brightness_ratio=torch.tensor([self.brightness_ratios[brightness_k]], dtype=torch.float32, device=dev),
            want=("lit_bgr",))
        depth = self.ctx.render(cls, pose, K, self.zNear, self.zFar, trunc_u8=False, want=("depth",))["depth"]
        return out["lit_bgr"][0].cpu().numpy(), depth[0, 0].cpu().numpy()


class Render_Py_Light_ModelNet_Multi(Render_Py):
    def __init__(self, meshes, K, width=640, height=480, zNear=0.25, zFar=6.0, brightness_ratios=(0.7,), device=0, ctx=None):
        super().__init__(meshes, ["model_%d" % i for i in range(len(meshes))], K, width, height, zNear, zFar, device, ctx)
        self.brightness_ratios = list(brightness_ratios)
        for i, m in enumerate(meshes):
            if getattr(m, "normals", None) is None:
                raise ValueError("mesh %d has no per-vertex normals" % i)
            if ctx is not None:
                self.ctx.upload_normals(i, m.normals)

    def render(self, model_idx, r, t, light_position, light_intensity, brightness_k=0, r_type="quat"):
        if r_type == "quat":
            w, x, y, z = [float(v) for v in r]
            s = 2.0 / (w * w + x * x + y * y + z * z)
            R = np.array([[1 - s * (y * y + z * z), s * (x * y - z * w), s * (x * z + y * w)],
                          [s * (x * y + z * w), 1 - s * (x * x + z * z), s * (y * z - x * w)],
                          [s * (x * z - y * w), s * (y * z + x * w), 1 - s * (x * x + y * y)]])
        elif r_type == "mat":
            R = np.asarray(r)
        else:
            raise ValueError("unknown r_type %r" % (r_type,))
        dev = self.ctx.device
        pose = torch.from_numpy(np.hstack([R, np.asarray(t).reshape(3, 1)]).astype(np.float32)[None]).to(dev)
        lp = torch.from_numpy(np.asarray(light_position, np.float32).reshape(1, 3)).to(dev)
        li = torch.from_numpy(np.asarray(light_intensity, np.float32).reshape(1, 3)).to(dev)
        out = self.ctx.render_lit(torch.tensor([model_idx], dtype=torch.int32, device=dev), pose, self.K, lp, li,
                                  self.brightness_ratios[brightness_k], self.zNear, self.zFar, want=("bgr", "depth"))
        return out["bgr"][0].cpu().numpy().astype(np.uint8), out["depth"][0, 0].cpu().numpy()
