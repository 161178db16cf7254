"""The CUDA library (through the C ABI) against the fixtures produced by the reference's UNMODIFIED custom operators
(tests/golden/ref_mx_*.npz, made by tests/golden/make_golden_mx.py under the numpy-backed mxnet stand-in): the same inputs,
compared with the reference's outputs directly -- not through the oracle.  Bit-exact for the 8 integer zoom bbox indices,
zoom_factor, every rounded mask / weight plane and ZoomTrans; <= 1 ulp for the sampled float planes; float32 rounding for
Transform3D.  Run with -m gpu on an H100; reads nothing outside the repo."""
import hashlib
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from deepim_b200.context import Context  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import mx_cases as C  # noqa: E402

DEV = torch.device("cuda", 0)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def load(name):
    return np.load(os.path.join(HERE, "golden", name))


def ulp_diff(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    sp = np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float32))
    return float(np.max(np.abs(a.astype(np.float64) - b.astype(np.float64)) / sp))


def test_zoom_mask_full_frame_against_reference_operator():
    g = load("ref_mx_zoom_full.npz")
    B, H, W = int(g["B"]), int(g["H"]), int(g["W"])
    c = C.zoom_case(int(g["seed"]), B, H, W)
    ctx = Context(0, max_batch=B, height=H, width=W, max_classes=1, max_verts=8, max_faces=8)
    zo, zg, zr, zf, bbox, status = ctx.zoom_mask(dev(c["mo"]), dev(c["mo"]), dev(c["mr"]), dev(c["pose"]), c["K"])
    assert np.array_equal(bbox.cpu().numpy(), g["bbox"])                 # the 8 integer zoom bbox indices
    assert np.array_equal(zf.cpu().numpy(), g["zoom_factor"])            # float32 bit patterns
    assert np.array_equal(np.packbits(zo.cpu().numpy().astype(np.uint8)), g["zm_obs"])
    assert np.array_equal(np.packbits(zr.cpu().numpy().astype(np.uint8)), g["zm_ren"])
    assert status.cpu().numpy().tolist() == [0] * B
    ctx.close()


def test_zoom_family_small_frame_against_reference_operators():
    g = load("ref_mx_zoom_small.npz")
    B, H, W = int(g["B"]), int(g["H"]), int(g["W"])
    c = C.zoom_case(int(g["seed"]), B, H, W)
    ctx = Context(0, max_batch=B, height=H, width=W, max_classes=1, max_verts=8, max_faces=8)
    zo, zg, zr, zf, bbox, _ = ctx.zoom_mask(dev(c["mo"]), dev(c["mo"]), dev(c["mr"]), dev(c["pose"]), c["K"])
    assert np.array_equal(bbox.cpu().numpy(), g["bbox"]) and np.array_equal(zf.cpu().numpy(), g["zoom_factor"])
    for got, key in ((zo, "zm_obs"), (zg, "zm_gt"), (zr, "zm_ren")):
        assert np.array_equal(got.cpu().numpy(), g[key].astype(np.float32)), key
    zio, zir = ctx.zoom_image_with_factor(zf, dev(c["img_o"]), dev(c["img_r"]), C.PIXEL_MEANS_RGB)
    assert ulp_diff(zio.cpu().numpy(), g["zio"]) <= 1 and ulp_diff(zir.cpu().numpy(), g["zir"]) <= 1
    for inv in (False, True):
        got = ctx.zoom_mask_with_factor(zf, dev(c["depth"]), inv).cpu().numpy()
        assert np.array_equal(got, g["zmwf_inv%d" % inv].astype(np.float32))
    fl, fw = ctx.zoom_flow(zf, dev(c["flow"]), dev(c["fw"]), False)
    assert ulp_diff(fl.cpu().numpy(), g["zflow"]) <= 1
    assert np.array_equal(fw.cpu().numpy(), g["zflow_w"].astype(np.float32))
    fl_inv, _ = ctx.zoom_flow(zf, dev(c["flow"]), None, True)
    assert ulp_diff(fl_inv.cpu().numpy(), g["zflow_inv"]) <= 1
    zd, zd2 = ctx.zoom_depth(zf, dev(c["depth"]), dev(c["depth"]))
    assert ulp_diff(zd.cpu().numpy(), g["zdepth"]) <= 1 and torch.equal(zd, zd2)
    zi = ctx.zoom_image(dev(c["img_o"]), dev(c["img_r"]), dev(c["pose"]), c["K"], C.PIXEL_MEANS_RGB)
    assert np.array_equal(zi[2].cpu().numpy(), g["zimg_factor"])
    assert hashlib.sha256(zi[0].cpu().numpy().tobytes()).digest() == g["zimg_o_sha"].tobytes()
    assert hashlib.sha256(zi[1].cpu().numpy().tobytes()).digest() == g["zimg_r_sha"].tobytes()
    tr = g["trans_in"]
    for inv in (False, True):
        assert np.array_equal(ctx.zoom_trans(zf, dev(tr), inv).cpu().numpy(), g["ztrans_inv%d" % inv])
        for zg_ in (False, True):
            got = ctx.zoom_trans_backward(zf, dev(tr[::-1].copy()), inv, zg_).cpu().numpy()
            assert np.array_equal(got, g["ztrans_bwd_inv%d_zg%d" % (inv, int(zg_))])
    ctx.close()


def test_transform3d_against_reference_operator():
    g = load("ref_mx_transform3d.npz")
    c = C.t3d_case(int(g["seed"]))
    ctx = Context(0, max_batch=4, height=96, width=128, max_classes=1, max_verts=8, max_faces=8)
    for coord in ("MODEL", "CAMERA"):
        fw = ctx.transform3d(dev(c["pts"]), dev(c["q"]), dev(c["t"]), dev(c["pose_src"]), c["T_means"], c["T_stds"], coord.lower())
        assert np.abs(fw.cpu().numpy() - g["fwd_" + coord]).max() < 2e-6
        rg, tg = ctx.transform3d_backward(dev(c["og"]), dev(c["pts"]), dev(c["q"]), dev(c["t"]), dev(c["pose_src"]), c["T_means"],
                                          c["T_stds"], coord.lower())
        assert np.abs(rg.cpu().numpy() - g["rot_grad_" + coord]).max() < 1e-4 * max(1.0, np.abs(g["rot_grad_" + coord]).max())
        assert np.abs(tg.cpu().numpy() - g["trans_grad_" + coord]).max() < 1e-4 * max(1.0, np.abs(g["trans_grad_" + coord]).max())
        assert not rg.cpu().numpy()[3].any()     # un-normalised quaternion: zero gradient (transform3d.py:221-222)
    ctx.close()


def test_update_data_batch_against_reference_function():
    """mask_observed := end-exclusive box of the new rendered mask (dim_update_mask_box) and image_rendered := transform(bgr)
    (dim_transform_image_u8) against lib/pair_matching/data_pair.py:update_data_batch run on the same inputs."""
    g = load("ref_mx_update_data_batch.npz")
    H, W = g["mask_rendered_0"].shape[2:]
    ctx = Context(0, max_batch=2, height=H, width=W, max_classes=1, max_verts=8, max_faces=8)
    bbs = []
    for b in range(2):
        m = g["mask_rendered_%d" % b][0, 0]
        ys, xs = np.nonzero(m)
        bbs.append([xs.min(), xs.max(), ys.min(), ys.max()])
    box = ctx.update_mask_box(dev(np.array(bbs, np.int32))).cpu().numpy()
    img = ctx.transform_image_u8(dev(np.stack([g["img_bgr_0"], g["img_bgr_1"]])), (103.939, 116.779, 123.68)).cpu().numpy()
    for b in range(2):
        assert np.array_equal(box[b, 0], g["mask_observed_%d" % b][0, 0].astype(np.float32))
        assert np.array_equal(img[b], g["image_rendered_%d" % b][0])
    ctx.close()
