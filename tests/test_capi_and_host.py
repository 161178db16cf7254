"""CPU: the C-ABI library loads and exports every symbol include/deepim_b200.h declares (no compute
calls without a GPU), the product package never touches the oracle, the op mirror has the
reference's surface, and the product fails loudly without a GPU."""
import ctypes
import os
import re

import numpy as np
import pytest


def declared_symbols(root):
    txt = open(os.path.join(root, "include", "deepim_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"DIM_API\s+[\w\s\*]+?\b(dim_\w+)\s*\(", txt)))


def test_library_exports_every_declared_symbol_at_abi_4(root):
    so = os.path.join(root, "mx-deepim_b200", "libdeepim_b200.so")
    assert os.path.exists(so), "run python __graft_entry__.py (build) first"
    lib = ctypes.CDLL(so)
    syms = declared_symbols(root)
    assert len(syms) >= 25
    for s in syms:
        assert hasattr(lib, s), "symbol %s declared in the header but not exported" % s
    lib.dim_abi_version.restype = ctypes.c_int32
    assert lib.dim_abi_version() == 4


def test_library_exports_no_undeclared_symbol(root):
    """Every dim_ symbol the library exports is declared in the header: an entry point removed from the header but left
    in the library would otherwise go unnoticed."""
    import shutil
    import subprocess
    if shutil.which("nm") is None:
        pytest.skip("nm not on PATH")
    so = os.path.join(root, "mx-deepim_b200", "libdeepim_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True, check=True).stdout
    exported = sorted({line.split()[-1] for line in out.splitlines() if line.split() and line.split()[-1].startswith("dim_")})
    assert exported == declared_symbols(root)


def test_library_is_sm90a_native_wgmma_and_tma(root):
    """The hot kernels of the shipped library are Hopper-native: the conv tower issues wgmma (SASS HGMMA) on operands staged
    by TMA (UTMALDG), and the only architecture in the fatbin is sm_90a."""
    import shutil
    import subprocess
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    so = os.path.join(root, "mx-deepim_b200", "libdeepim_b200.so")
    elf = subprocess.run(["cuobjdump", "-lelf", so], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\w+)\.cubin", elf))
    assert archs == {"90a"}, archs
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    per_kernel, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            per_kernel[cur] = {"HGMMA": 0, "UTMALDG": 0}
        elif cur:
            for k in per_kernel[cur]:
                if re.search(r"\b%s\b" % k, line):
                    per_kernel[cur][k] += 1
    def of(name):
        return [v for k, v in per_kernel.items() if name in k]
    for name in ("conv_igemm_persistent_kernel", "conv1_kernel", "conv_wgrad_kernel", "conv1_wgrad_kernel"):
        ks = [v for v in of(name) if v["HGMMA"]]     # (cuobjdump also lists empty stubs under the same name)
        assert ks, name
        for v in ks:
            assert v["HGMMA"] >= 4 and v["UTMALDG"] >= 1, (name, v)


def test_train_config_struct_layout_matches_the_header(root, tmp_path):
    """dim_train_config crosses the C ABI by pointer: the ctypes mirror must have the C compiler's layout of the header's struct."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("gcc not on PATH")
    from deepim_b200 import _capi
    src = tmp_path / "layout.c"
    fields = [f for f, _ in _capi.TrainConfig._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "deepim_b200.h"\nint main(void) {\n  printf("%zu", sizeof(dim_train_config));\n'
                   + "".join('  printf(" %%zu", offsetof(dim_train_config, %s));\n' % f for f in fields) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)])
    nums = [int(x) for x in subprocess.check_output([str(exe)]).decode().split()]
    assert nums[0] == ctypes.sizeof(_capi.TrainConfig)
    assert nums[1:] == [getattr(_capi.TrainConfig, f).offset for f in fields]


def test_ctypes_binding_covers_the_header(root):
    from deepim_b200 import _capi
    assert sorted(_capi.SIGNATURES) == declared_symbols(root)


def header_prototypes(root):
    """{name: (return type, [parameter declarations])} of every function the header declares"""
    txt = open(os.path.join(root, "include", "deepim_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return {m.group(2): (" ".join(m.group(1).split()), [" ".join(p.split()) for p in m.group(3).split(",")])
            for m in re.finditer(r"DIM_API\s+([\w\s\*]+?)\b(dim_\w+)\s*\(([^)]*)\)", txt)}


@pytest.mark.parametrize("fn", declared_symbols(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
def test_ctypes_prototypes_match_the_header(root, fn):
    """Return kind, argument count and argument kinds (pointer / 32-bit int / 64-bit int / 64-bit unsigned / float) of each
    entry in _capi.SIGNATURES equal the header's prototype: a wrong argtypes list would misread the call's arguments
    without any error."""
    import ctypes as C
    from deepim_b200 import _capi
    ret, params = header_prototypes(root)[fn]
    restype, argtypes = _capi.SIGNATURES[fn]
    if params == ["void"]:
        params = []

    def kind_c(decl):
        if "*" in decl:
            return "ptr"
        return {"void": "void", "int32_t": "i32", "int64_t": "i64", "uint64_t": "u64", "float": "f32"}[decl.split()[0]]

    def kind_py(t):
        if t is None:
            return "void"
        if t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer):
            return "ptr"
        return {C.c_int32: "i32", C.c_int64: "i64", C.c_uint64: "u64", C.c_float: "f32"}[t]

    assert kind_c(ret) == kind_py(restype), (fn, ret)
    assert len(argtypes) == len(params), (fn, params)
    assert [kind_c(p) for p in params] == [kind_py(t) for t in argtypes], fn


def test_no_cpu_fallback_ctx_create_fails_loudly_without_gpu(root):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from deepim_b200 import _capi
    h = ctypes.c_void_p()
    rc = _capi.lib.dim_ctx_create(0, 1, 480, 640, 1, 8, 8, ctypes.byref(h))
    assert rc != 0
    assert b"no CPU fallback" in _capi.lib.dim_last_error()
    from deepim_b200.context import Context
    with pytest.raises(_capi.DeepIMError):
        Context(0)


def test_product_never_imports_or_links_the_oracle(root):
    pkg = os.path.join(root, "mx-deepim_b200")
    bad = []
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M) or "liboracle" in src or "deepim_oracle" in src:
                    bad.append(os.path.join(dp, f))
    assert not bad, bad
    # and the shared library has no dependency on it
    so = os.path.join(pkg, "libdeepim_b200.so")
    assert b"liboracle" not in open(so, "rb").read()


def test_operator_surface_matches_reference_signatures():
    # SURVEY 8(b): names, argument / output lists and string attrs of deepim/operator_py/*.py
    from deepim_b200 import operator_py as op
    K = "[572.4114 0 325.2611 0 573.57043 242.04899 0 0 1]"
    expect = {
        "ZoomMask": (dict(K=K), ["mask_observed", "mask_gt_observed", "mask_rendered", "src_pose"],
                     ["zoom_mask_observed", "zoom_mask_gt_observed", "zoom_mask_rendered", "zoom_factor"]),
        "ZoomImageWithFactor": (dict(pixel_means="[123.68 116.779 103.939]"),
                                ["zoom_factor", "image_observed", "image_rendered"],
                                ["zoom_image_observed", "zoom_image_rendered"]),
        "ZoomMaskWithFactor": (dict(b_inv_zoom="True"), ["zoom_factor", "mask"], ["zoom_mask"]),
        "ZoomFlow": (dict(b_inv_zoom="False"), ["zoom_factor", "flow", "flow_weights"], ["zoom_flow", "zoom_flow_weights"]),
        "ZoomTrans": (dict(b_inv_zoom="True"), ["zoom_factor", "trans_delta"], ["zoom_trans_delta"]),
        "ZoomDepth": (dict(), ["zoom_factor", "depth_observed", "depth_rendered"],
                      ["zoom_depth_observed", "zoom_depth_rendered"]),
        "Transform3D": (dict(T_means="[0 0 0]", T_stds="[1 1 1]", rot_coord="CAMERA"),
                        ["point_cloud", "rotation", "translation", "pose_src"], ["transformed_3d_points"]),
        "FlowUpdater": (dict(K=K), ["depth_src", "depth_tgt", "pose_src", "pose_tgt"], ["flow", "flow_weights"]),
        "ZoomImage": (dict(K=K, pixel_means="[123.68 116.779 103.939]"), ["image_observed", "image_rendered", "src_pose"],
                      ["zoom_image_observed", "zoom_image_rendered", "zoom_factor"]),
        "GroupPicker": (dict(group_num="13"), ["input_data", "group_idx"], ["picked_data"]),
    }
    for name, (kw, args, outs) in expect.items():
        prop = op.REGISTRY[name](**kw)
        assert prop.list_arguments() == args and prop.list_outputs() == outs, name
    inv = op.REGISTRY["ZoomFlow"](b_inv_zoom="True")
    assert inv.list_arguments() == ["zoom_factor", "flow"] and inv.list_outputs() == ["zoom_flow"]
    zm = op.REGISTRY["ZoomMask"](K=K, width="640", height="480")
    np.testing.assert_allclose(zm.K[0], [572.4114, 0, 325.2611], rtol=1e-7)
    assert zm.infer_shape([[4, 1, 480, 640]] * 3 + [[4, 3, 4]])[1][-1] == [4, 4]
    zi = op.REGISTRY["ZoomImageWithFactor"](pixel_means="[123.68 116.779 103.939]")
    np.testing.assert_allclose(zi.pixel_means, [103.939, 116.779, 123.68], rtol=1e-7)  # reversed, l.79-81
    assert op.REGISTRY["GroupPicker"](group_num="13").infer_shape([[4, 52], [4, 1]])[1] == [[4, 4]]  # group_picker.py:73-79
    with pytest.raises(RuntimeError):
        op.create("ZoomTrans", b_inv_zoom="True")  # no Context set -> loud


def test_shard_range_and_chunks():
    from deepim_b200 import sharding
    for n in (0, 1, 7, 64, 65, 128):
        for world in (1, 2, 3, 8):
            rs = [sharding.shard_range(n, r, world) for r in range(world)]
            assert rs[0][0] == 0 and rs[-1][1] == n
            assert all(rs[i][1] == rs[i + 1][0] for i in range(world - 1))
            sizes = [b - a for a, b in rs]
            assert max(sizes) - min(sizes) <= 1
    assert sharding.chunks(3, 40, 16) == [(3, 19), (19, 35), (35, 40)]
    assert sharding.chunks(5, 5, 16) == []
    with pytest.raises(ValueError):
        sharding.shard_range(4, 2, 2)


def test_mxnet_params_reader_writer(tmp_path):
    """MXNet .params container (mx.nd.save dict; lib/utils/load_model.py:10-30): writer/reader round trip, the legacy
    and V1 record layouts, and a byte string assembled by hand from the documented layout.  Format parity is unpinned
    (no sample checkpoint in the reference, MXNet not installable): see the module docstring."""
    import struct
    from deepim_b200 import mx_params, synth
    w = synth.make_weights(0)
    small = {k: w[k] for k in ("flow_conv1_weight", "flow_conv1_bias", "rot_weight", "trans_bias")}
    mx_params.save_checkpoint(str(tmp_path / "net"), 8, small, {"bn_moving_mean": np.arange(4, dtype=np.float32)})
    arg, aux = mx_params.load_checkpoint(str(tmp_path / "net"), 8)
    assert set(arg) == set(small) and list(aux) == ["bn_moving_mean"]
    for k in small:
        assert arg[k].dtype == np.float32 and np.array_equal(arg[k], small[k])
    # hand-assembled: one V2 float32 (2,3), one V1 int32 (2,), one legacy float64 (1,2)
    a0, a1, a2 = np.arange(6, dtype=np.float32).reshape(2, 3), np.array([7, -9], np.int32), np.array([[0.5, 1.5]])
    rec0 = struct.pack("<IiI2qiii", 0xF993FAC9, 0, 2, 2, 3, 1, 0, 0) + a0.tobytes()
    rec1 = struct.pack("<II1qiii", 0xF993FAC8, 1, 2, 2, 0, 4) + a1.tobytes()
    rec2 = struct.pack("<I2Iiii", 2, 1, 2, 1, 0, 1) + a2.tobytes()
    names = [b"arg:a0", b"arg:a1", b"aux:a2"]
    blob = struct.pack("<QQQ", 0x112, 0, 3) + rec0 + rec1 + rec2 + struct.pack("<Q", 3) + b"".join(struct.pack("<Q", len(n)) + n for n in names)
    d = mx_params.load(blob)
    assert np.array_equal(d["arg:a0"], a0) and np.array_equal(d["arg:a1"], a1) and np.array_equal(d["aux:a2"], a2)
    with pytest.raises(ValueError):
        mx_params.load(b"\x00" * 32)
    with pytest.raises(ValueError):
        mx_params.load(blob[:-40])


def test_lm6d_disk_formats_round_trip(tmp_path):
    """LM6d_refine on-disk formats (lib/dataset/LM6D_REFINE.py:112-196, render_py_multi.py:69-76): OBJ un-rolled per
    face-vertex like glumpy.objload renders identically, uint16 depth / DEPTH_FACTOR, pose files with a header line."""
    import lm6d_fixture
    from deepim_b200 import lm6d_io, synth
    from oracle import oracle as O
    classes, meshes = lm6d_fixture.build(str(tmp_path), n_per_class=1)
    ds = lm6d_io.LM6DRefine(str(tmp_path), classes, "val")
    assert abs(ds.diameters["cube"] - meshes["cube"].diameter) < 1e-6
    m = ds.mesh("cube")
    assert len(m.verts) == 3 * len(meshes["cube"].faces) and np.array_equal(m.tex, meshes["cube"].tex)
    (pair,) = ds.pairs("cube")
    rec = ds.load_pair("cube", pair)
    assert rec["image_observed"].dtype == np.uint8 and rec["image_observed"].shape == (480, 640, 3)
    a = O.render(m, rec["pose_rendered"], synth.K_LINEMOD)
    b = O.render(meshes["cube"], rec["pose_rendered"], synth.K_LINEMOD)
    assert np.array_equal(a["bgr"], b["bgr"]) and np.array_equal(a["depth"], b["depth"])    # same pixels from the un-rolled mesh
    assert np.abs(rec["depth_rendered"] - b["depth"]).max() <= 0.5 / lm6d_io.DEPTH_FACTOR + 1e-6   # uint16 millimetres
    assert np.abs(rec["pose_observed"] - np.loadtxt(os.path.join(str(tmp_path), "data", "gt_observed", "cube", "000000-pose.txt"),
                                                    skiprows=1)).max() == 0
    assert ds.points("glue").shape[1] == 3


def test_trainer_flat_parameter_layout():
    """The flat fp32 parameter vector of the training step (dim_train_param_info; no GPU needed for the table):
    57 749 164 values = SURVEY 8(d)'s 230 996 656-byte gradient all-reduce, reference tensor order, fc6 kept in NHWC order."""
    from deepim_b200 import synth, trainer
    tab = trainer.param_table()
    assert sum(n for _, n in tab) == 57749164 and 4 * 57749164 == 230996656
    assert [k for k, _ in tab[-2:]] == ["upsampling_weight", "mask_upsampling_weight"]
    w = synth.make_train_weights(3)
    # the table the library reports (dim_train_param_info) names exactly the tensors of deepIM_flownet.py's training graph, with
    # their element counts
    assert {k: n for k, n in tab} == {k: int(np.prod(v.shape)) for k, v in w.items()}
    flat = trainer.flatten_params(w)
    back = trainer.unflatten_params(flat, w)
    assert all(np.array_equal(back[k], w[k]) for k in w)
    off = 0
    for name, n in tab:
        if name == "fc6_weight":   # stored (out, h*10+w, c): element (o, c*80+hw) of MXNet's layout sits at (o, hw, c)
            f6 = flat[off:off + n].reshape(256, 80, 1024)
            assert f6[5, 17, 300] == w["fc6_weight"][5, 300 * 80 + 17]
        off += n
    # depth input without the mask channels is no network of this library: its table is refused, as the context switches are
    from deepim_b200 import _capi
    name, wn, bn = ctypes.c_char_p(), ctypes.c_int64(), ctypes.c_int64()
    assert _capi.lib.dim_train_param_info(1, 0, 0, ctypes.byref(name), ctypes.byref(wn), ctypes.byref(bn)) != 0
    assert b"input_mask = 0" in _capi.lib.dim_last_error()


def test_simpson_rule_and_obj_parser(tmp_path):
    """pose_eval.simpson = scipy.integrate.simps(even='avg') of the reference's era (LM6D_REFINE.py:462-466 integrates 1000
    samples); the OBJ reader handles vn records, negative indices and polygon fans (glumpy.objload conventions)."""
    from deepim_b200 import lm6d_io
    from deepim_b200.pose_eval import simpson
    x = np.linspace(0.0, 1.0, 1001)
    assert abs(simpson(x ** 3, x[1] - x[0]) - 0.25) < 1e-12          # odd sample count: exact for cubics
    y = np.linspace(0.0, 0.0999, 1000) ** 2                          # the evaluator's grid: 1000 samples, dx = 1e-4
    first = simpson(y[:-1], 1e-4) + 0.5e-4 * (y[-1] + y[-2])
    last = simpson(y[1:], 1e-4) + 0.5e-4 * (y[0] + y[1])
    assert abs(simpson(y, 1e-4) - 0.5 * (first + last)) < 1e-18 and abs(simpson(y, 1e-4) - 0.0999 ** 3 / 3) < 1e-9
    obj = tmp_path / "m.obj"
    obj.write_text("v 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nvt 0 0\nvt 1 0\nvt 1 1\nvt 0 1\nvn 0 0 1\n"
                   "f 1/1/1 2/2/1 3/3/1 4/4/1\nf -4/-4/-1 -3/-3/-1 -2/-2/-1\n")
    m = lm6d_io.load_textured_obj(str(obj))
    assert m.faces.shape == (3, 3) and m.verts.shape == (9, 3)       # quad -> 2 triangles (fan) + 1 triangle, un-rolled
    assert np.array_equal(m.verts[3:6], np.array([[0, 0, 0], [1, 1, 0], [0, 1, 0]], np.float32))
    assert np.array_equal(m.verts[6:9], m.verts[[0, 1, 2]]) and np.array_equal(m.normals, np.tile([[0, 0, 1]], (9, 1)))
    assert np.array_equal(m.uvs[2], [1, 1])


def test_symbol_json_reader_and_architecture_check(tmp_path):
    """<prefix>-symbol.json (MXNet's graph file next to <prefix>-%04d.params): read the node / attribute layout of MXNet >= 1.0
    ("attrs") and of older files ("attr" / "param"), and refuse a checkpoint whose graph is not the FlowNetS tower."""
    import json
    from deepim_b200 import mx_params, synth
    path = mx_params.save_symbol_json(os.path.join(str(tmp_path), "deepim-symbol.json"))
    sym = mx_params.load_symbol_json(path)
    assert mx_params.check_flownet_symbol(sym)
    assert sym["arguments"][0] == "data" and "fc6_weight" in sym["arguments"] and "rot_bias" in sym["arguments"]
    assert [sym["nodes"][h]["name"] for h in sym["heads"]] == ["rot", "trans"]
    w = synth.make_weights(0)
    assert all(a in w for a in sym["arguments"] if a != "data")          # argument names = checkpoint keys (load_model.py:19-27)
    g = json.load(open(path))
    for n in g["nodes"]:                                                  # pre-1.0 spelling of the attribute dict
        if "attrs" in n:
            n["attr"] = n.pop("attrs")
    assert mx_params.check_flownet_symbol(mx_params.load_symbol_json(json.dumps(g)))
    for n in g["nodes"]:
        if n["name"] == "conv3":
            n["attr"]["stride"] = "(1, 1)"
    with pytest.raises(ValueError):
        mx_params.check_flownet_symbol(mx_params.load_symbol_json(json.dumps(g)))
    with pytest.raises(ValueError):
        mx_params.load_symbol_json(json.dumps({"foo": 1}))
