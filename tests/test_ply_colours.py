"""CPU: vertex-coloured meshes.  lm6d_io.load_ply against the reference's PLY reader (tests/golden/ref_ply.npz), in ASCII
and binary with every scalar type, and its refusals; a textured PLY renders like the OBJ of the same model; the coloured
renders of the CPU checker (tests/colour_oracle.c: unlit with and without uint8 truncation, ModelNet- and Py_Light-lit)
against the float64 ray caster on the rasteriser's test scenes; one constant vertex colour against a constant texture."""
import os
import struct

import numpy as np
import pytest

from deepim_b200 import lm6d_io, synth
from oracle import oracle as O

import colour_oracle as CO
import colour_scenes as CS
import raster_ref as RR
import raster_scenes as RS

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_ply.npz")
SCENES = RS.geometry_scenes() + RS.mesh_scenes() + [RS.batch16_scene()]
FACTOR = 1000.0


# ------------------------------------------------------------------------------------------------------- the reader
@pytest.mark.parametrize("case", range(4))
def test_load_ply_matches_the_reference_reader(tmp_path, case):
    g = np.load(GOLDEN)
    path = tmp_path / ("case%d.ply" % case)
    path.write_bytes(g["case%d_ply" % case].tobytes())
    scale = 1e-3 if case == 3 else 1.0
    m = lm6d_io.load_ply(str(path), scale=scale)
    pts = g["case%d_pts" % case]
    assert np.array_equal(m.verts, (pts * scale).astype(np.float32))
    assert np.array_equal(m.faces, g["case%d_faces" % case].astype(np.int32))
    assert m.uvs is None and m.tex is None
    if "case%d_colors" % case in g:
        assert np.array_equal(m.colours, g["case%d_colors" % case].astype(np.float32) / np.float32(255))
    else:
        assert np.array_equal(m.colours, np.full((len(pts), 3), 0.5, np.float32))  # the SIXD renderer's grey
    if "case%d_normals" % case in g:
        assert np.array_equal(m.normals, g["case%d_normals" % case].astype(np.float32))
    else:
        assert getattr(m, "normals", None) is None


def _model(seed=4, V=30, F=40):
    rs = np.random.RandomState(seed)
    return (rs.randint(-30000, 30000, (V, 3)), rs.uniform(-1, 1, (V, 3)).astype(np.float32), rs.randint(0, 256, (V, 4)),
            rs.randint(0, V, (F, 3)))


# vertex: x y z int, nx ny nz double, quality short, red green blue alpha uchar; an extra element before and after the faces
VPROPS = [("int", "x"), ("int", "y"), ("int", "z"), ("double", "nx"), ("double", "ny"), ("double", "nz"), ("short", "quality"),
          ("uchar", "red"), ("uchar", "green"), ("uchar", "blue"), ("uchar", "alpha")]
VFMT = "<iiidddhBBBB"


def write_ply(path, binary, face_key="vertex_indices", fmt=None, faces=None, vprops=VPROPS, comments=()):
    pos, nrm, col, f = _model()
    faces = f if faces is None else faces
    fmt = fmt or ("binary_little_endian 1.0" if binary else "ascii 1.0")
    head = ["ply", "format " + fmt] + ["comment " + c for c in comments]
    head += ["element camera 2", "property float fov", "property list uchar short tags"]
    head += ["element vertex %d" % len(pos)] + ["property %s %s" % p for p in vprops]
    head += ["element face %d" % len(faces), "property list uchar int " + face_key]
    head += ["element edge 3", "property int vertex1", "property list ushort uint more", "end_header"]
    body = b""
    cams = [(1.5, [1, -2]), (0.25, [7])]
    edges = [(0, [1, 2, 3]), (5, []), (9, [4])]
    if binary:
        for fov, tags in cams:
            body += struct.pack("<fB", fov, len(tags)) + struct.pack("<%dh" % len(tags), *tags)
        for p, n, c in zip(pos, nrm, col):
            body += struct.pack(VFMT, *p, *n.astype(np.float64), 3, *c)
        for t in faces:
            body += struct.pack("<B", len(t)) + struct.pack("<%di" % len(t), *t)
        for a, more in edges:
            body += struct.pack("<iH", a, len(more)) + struct.pack("<%dI" % len(more), *more)
    else:
        lines = ["%r %d %s" % (fov, len(tags), " ".join(map(str, tags))) for fov, tags in cams]
        lines += ["%d %d %d %.17g %.17g %.17g 3 %d %d %d %d" % (*p, *n.astype(np.float64), *c) for p, n, c in zip(pos, nrm, col)]
        lines += ["%d %s" % (len(t), " ".join(map(str, t))) for t in faces]
        lines += ["%d %d %s" % (a, len(more), " ".join(map(str, more))) for a, more in edges]
        body = ("\n".join(lines) + "\n").encode()
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode() + body)
    return pos, nrm, col, faces


@pytest.mark.parametrize("face_key", ["vertex_indices", "vertex_index"])
def test_ascii_and_binary_load_the_same_arrays(tmp_path, face_key):
    pos, nrm, col, faces = write_ply(tmp_path / "a.ply", False, face_key)
    write_ply(tmp_path / "b.ply", True, face_key)
    a = lm6d_io.load_ply(str(tmp_path / "a.ply"), scale=1e-3)
    b = lm6d_io.load_ply(str(tmp_path / "b.ply"), scale=1e-3)
    for k in ("verts", "colours", "normals", "faces"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    assert np.array_equal(a.verts, (pos.astype(np.float64) * 1e-3).astype(np.float32))
    assert np.array_equal(a.colours, col[:, :3].astype(np.float32) / np.float32(255))  # alpha ignored
    assert np.array_equal(a.normals, nrm)
    assert np.array_equal(a.faces, faces)


def test_float_colours_are_taken_as_they_are(tmp_path):
    """a float colour property is not divided by 255, however dark the model"""
    p = tmp_path / "f.ply"
    p.write_text("ply\nformat ascii 1.0\nelement vertex 3\nproperty float x\nproperty float y\nproperty float z\n"
                 "property float red\nproperty float green\nproperty float blue\nelement face 1\n"
                 "property list uchar int vertex_indices\nend_header\n0 0 0 0.25 0.5 1\n1 0 0 0 0 0\n0 1 0 1 1 1\n3 0 1 2\n")
    m = lm6d_io.load_ply(str(p))
    assert np.array_equal(m.colours, np.float32([[0.25, 0.5, 1], [0, 0, 0], [1, 1, 1]]))


@pytest.mark.parametrize("what", ["big endian", "quad", "no z", "index out of range", "negative index", "missing texture"])
def test_load_ply_refusals(tmp_path, what):
    p = tmp_path / "bad.ply"
    if what == "big endian":
        write_ply(p, True, fmt="binary_big_endian 1.0")
    elif what == "quad":
        write_ply(p, False, faces=[[0, 1, 2], [0, 1, 2, 3]])
    elif what == "no z":
        write_ply(p, False, vprops=[("int", "x"), ("int", "y"), ("int", "w")] + VPROPS[3:])
    elif what == "index out of range":
        write_ply(p, True, faces=[[0, 1, 30]])
    elif what == "negative index":
        write_ply(p, False, faces=[[0, -1, 2]])
    else:
        write_ply(p, False, vprops=VPROPS[:7] + [("float", "texture_u"), ("float", "texture_v"), ("uchar", "blue"),
                                                 ("uchar", "alpha")], comments=["TextureFile nowhere.png"])
    with pytest.raises(ValueError):
        lm6d_io.load_ply(str(p))


def test_textured_ply_renders_like_the_obj(tmp_path):
    """the same textured model as OBJ (un-rolled per face corner) and as PLY (indexed): identical renders"""
    m = synth.make_blob(nlat=20, nlon=40, seed=3)
    lm6d_io.write_textured_obj(m, str(tmp_path / "m" / "textured.obj"), str(tmp_path / "m" / "tex.png"))
    with open(tmp_path / "m" / "model.ply", "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\ncomment TextureFile tex.png\nelement vertex %d\nproperty float x\n"
                 "property float y\nproperty float z\nproperty float texture_u\nproperty float texture_v\nelement face %d\n"
                 "property list uchar int vertex_indices\nend_header\n" % (len(m.verts), len(m.faces))).encode())
        f.write(np.concatenate([m.verts, m.uvs], 1).astype("<f4").tobytes())
        f.write(np.concatenate([np.full((len(m.faces), 1), 3, np.uint8).view(np.uint8),
                                m.faces.astype("<i4").view(np.uint8).reshape(-1, 12)], 1).tobytes())
    obj = lm6d_io.load_textured_obj(str(tmp_path / "m" / "textured.obj"), str(tmp_path / "m" / "tex.png"))
    ply = lm6d_io.load_ply(str(tmp_path / "m" / "model.ply"))
    assert ply.colours is None and np.array_equal(ply.tex, obj.tex) and len(ply.verts) < len(obj.verts)
    for k, pose in enumerate(synth.sample_pose_pairs(3, 8)[0]):
        a, b = O.render(obj, pose, synth.K_LINEMOD), O.render(ply, pose, synth.K_LINEMOD)
        assert a["mask"].sum() > 1000
        for n in ("bgr", "depth", "image", "mask", "bbox"):
            assert np.array_equal(a[n], b[n]), (k, n)


# ---------------------------------------------------------------------------------- the coloured renders vs float64
def check_scene_colours(s):
    rep = RR.Report(repr(s))
    for c, pose, lpos, inten, ratio in s.inst:
        m = s.meshes[c]
        ref = RR.Render(m, pose, s.K, s.H, s.W, s.zn, s.zf, m.normals)
        geo = dict(zn=s.zn, zf=s.zf, H=s.H, W=s.W)
        for trunc in (True, False):
            o = CO.render(m, pose, s.K, trunc_u8=trunc, **geo)
            RR.check_render(rep, ref, o["depth"], o["mask"])
            CS.check_colours(rep, ref, o["bgr"], trunc)
        o = CO.render_lit(m, m.normals, pose, s.K, lpos, inten, ratio, **geo)
        RR.check_render(rep, ref, o["depth"], o["mask"])
        CS.check_lit_colours(rep, ref, o["bgr"], lpos, inten, ratio, "modelnet")
        o = CO.render_dataset(m, pose, s.K, lpos, inten, ratio, depth_factor=FACTOR, **geo)
        CS.check_lit_colours(rep, ref, o["lit_bgr"], lpos, inten, ratio, "py_light")
        CS.check_colours(rep, ref, o["bgr"], True)
        RR.check_render(rep, ref, o["label"], label=True)
        RR.check_u16(rep, ref, o["depth"], o["label"], FACTOR)
    return rep


@pytest.mark.parametrize("s", SCENES, ids=repr)
def test_coloured_oracle_against_float64(s):
    rep = check_scene_colours(CS.coloured_scene(s))
    print(rep, "u8 colour ambiguous", getattr(rep, "ambiguous_colour", 0))
    assert rep.ok, str(rep)


@pytest.mark.parametrize("level", [0, 1, 77, 128, 254, 255])
def test_constant_colour_against_constant_texture(level):
    """one vertex colour k / 255 everywhere against a texture of k: the same geometry outputs, colours within one level
    (the float32 interpolation can land just below k before the uint8 truncation)"""
    ms = RS.meshes()
    for name, pose in zip(("cube", "c2"), synth.sample_pose_pairs(2, 5)[0]):
        t = ms[name]
        tex = synth.Mesh(t.verts, t.uvs, t.faces, np.full((4, 4, 3), level, np.uint8))
        col = synth.Mesh(t.verts, None, t.faces, None, colours=np.full((len(t.verts), 3), np.float32(level) / np.float32(255)))
        for trunc in (True, False):
            a, b = O.render(tex, pose, RS.K_LM, trunc_u8=trunc), CO.render(col, pose, RS.K_LM, trunc_u8=trunc)
            for n in ("depth", "mask", "bbox"):
                assert np.array_equal(a[n], b[n]), (name, n)
            assert a["mask"].sum() > 100
            assert np.abs(a["bgr"] - b["bgr"]).max() <= 1.0
            assert np.abs(a["image"] - b["image"]).max() <= 1.0 + 1e-4


def test_mesh_has_one_colour_source():
    m = synth.make_cube()
    with pytest.raises(ValueError):
        synth.Mesh(m.verts, m.uvs, m.faces, m.tex, colours=np.zeros((len(m.verts), 3)))
    with pytest.raises(ValueError):
        synth.Mesh(m.verts, None, m.faces, None)
