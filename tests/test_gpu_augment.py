"""GPU: dim_replace_background and dim_mask_dilate bit for bit against the live reference's outputs
(tests/golden/make_golden_augment.py), their error paths, and make_device_batch(background=..., mask_dilate=...) feeding
fit_batch."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import augment, synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.trainer import Trainer, fit_batch, make_device_batch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
BG = np.load(os.path.join(HERE, "golden", "ref_background.npz"))
DIL = np.load(os.path.join(HERE, "golden", "ref_mask_dilate.npz"))
H, W = 480, 640
MAXB = 16
MEANS_RGB = BG["pixel_means_bgr"][::-1].copy()
PHOTOS = [BG["photo%d" % i] for i in range(len(BG["photo_shapes"]))]


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, max_batch=MAXB, max_classes=2, max_verts=6000, max_faces=11000)
    augment.BackgroundBank(c, PHOTOS)
    yield c
    c.close()


def case_inputs(cases):
    obs = torch.from_numpy(np.stack([BG["observed"]] * len(cases)).astype(np.float32)).cuda()  # one observed image for every case
    mask = torch.from_numpy(np.stack([BG["mask"][i] for i in cases]).astype(np.float32)[:, None]).cuda()
    return obs, mask, np.asarray([BG["bank_index"][i] for i in cases], np.int32)


def blob_of(comp_u8):
    """transform (image.py:583-594) as the reference computes it, cast to float32"""
    c = comp_u8.astype(np.float64)
    return np.stack([c[..., 2 - k] - BG["pixel_means_bgr"][2 - k] for k in range(3)], 1).astype(np.float32)


def test_replace_background_bit_identical_to_the_reference(ctx):
    cases = list(range(len(BG["bank_index"])))
    obs, mask, idx = case_inputs(cases)
    img, comp = ctx.replace_background(obs, mask, idx, MEANS_RGB, want_composite=True)
    comp = comp.cpu().numpy()
    for j, i in enumerate(cases):
        np.testing.assert_array_equal(comp[j], BG["composite"][i], err_msg="case %d (photo %s)" % (i, BG["bank_index"][i]))
    np.testing.assert_array_equal(img.cpu().numpy(), blob_of(BG["composite"][cases]))


def test_keep_index_equals_transform_image_u8(ctx):
    obs, mask, _ = case_inputs([0, 1])
    img = ctx.replace_background(obs, mask, np.array([-1, -1], np.int32), MEANS_RGB)
    ref = ctx.transform_image_u8(obs.to(torch.uint8), MEANS_RGB)
    assert torch.equal(img, ref)


@pytest.mark.parametrize("B", [1, 3, 16])
def test_mixed_batch(ctx, B):
    n = len(BG["bank_index"])
    cases = [(3 * j) % n for j in range(B)]
    obs, mask, _ = case_inputs(cases)
    idx = np.asarray([BG["bank_index"][i] if j % 2 == 0 else -1 for j, i in enumerate(cases)], np.int32)
    img, comp = ctx.replace_background(obs, mask, idx, MEANS_RGB, want_composite=True)
    comp = comp.cpu().numpy()
    for j, i in enumerate(cases):
        want = BG["composite"][i] if idx[j] >= 0 else BG["observed"]
        np.testing.assert_array_equal(comp[j], want, err_msg="instance %d" % j)
    np.testing.assert_array_equal(img.cpu().numpy(), blob_of(comp))


def test_mask_dilate_bit_identical_to_the_reference(ctx):
    n = len(DIL["seed"])
    for lo in range(0, n, MAXB):
        sl = slice(lo, min(n, lo + MAXB))
        draws = np.concatenate([augment.mask_dilate_draws(1, np.random.RandomState(int(s))) for s in DIL["seed"][sl]])
        m = torch.from_numpy(DIL["mask"][sl][:, None].copy()).cuda()
        out = ctx.mask_dilate(m, draws).cpu().numpy()[:, 0]
        np.testing.assert_array_equal(out.astype(np.float64), DIL["out"][sl])


def test_error_paths(ctx):
    obs, mask, _ = case_inputs([0])
    with pytest.raises(capi.DeepIMError, match="not uploaded"):
        ctx.replace_background(obs, mask, np.array([len(PHOTOS)], np.int32), MEANS_RGB)
    big = torch.zeros((MAXB + 1, H, W, 3), device="cuda")
    with pytest.raises(capi.DeepIMError, match="max_batch"):
        ctx.replace_background(big, torch.zeros((MAXB + 1, 1, H, W), device="cuda"), np.full(MAXB + 1, -1, np.int32),
                               MEANS_RGB)
    with pytest.raises(capi.DeepIMError, match="max_batch"):
        ctx.mask_dilate(torch.zeros((MAXB + 1, 1, H, W), device="cuda"), np.zeros((MAXB + 1, 5), np.int32))
    idx = np.zeros(1, np.int32)
    rc = capi.lib.dim_replace_background(ctx._h, None, capi.C.c_void_p(mask.data_ptr()), idx.ctypes.data, 1,
                                         capi.farr(MEANS_RGB, 3, capi.C.c_double), capi.C.c_void_p(obs.data_ptr()), None, None)
    assert rc != 0 and b"NULL" in capi.lib.dim_last_error()
    rc = capi.lib.dim_mask_dilate(ctx._h, capi.C.c_void_p(mask.data_ptr()), None, 1, capi.C.c_void_p(mask.data_ptr()), None)
    assert rc != 0 and b"NULL" in capi.lib.dim_last_error()
    d = torch.zeros((1, 5), dtype=torch.int32, device="cuda")
    rc = capi.lib.dim_mask_dilate(ctx._h, capi.C.c_void_p(mask.data_ptr()), capi.C.c_void_p(d.data_ptr()), 1,
                                  capi.C.c_void_p(mask.data_ptr()), None)
    assert rc != 0 and b"in place" in capi.lib.dim_last_error()
    with pytest.raises(capi.DeepIMError, match="INTER_AREA"):
        capi.check(capi.lib.dim_bg_upload(ctx._h, 0, np.zeros((960, 1279, 3), np.uint8).ctypes.data, 960, 1279))
    empty = Context(0, max_batch=1, max_classes=1, max_verts=100, max_faces=100)
    try:
        with pytest.raises(capi.DeepIMError, match="bank is empty"):
            empty.replace_background(obs, mask, np.zeros(1, np.int32), MEANS_RGB)
        assert torch.equal(empty.replace_background(obs, mask, np.full(1, -1, np.int32), MEANS_RGB),
                           empty.transform_image_u8(obs.to(torch.uint8), MEANS_RGB))
    finally:
        empty.close()


def make_ctx(meshes, B):
    c = Context(0, max_batch=B, max_classes=2, max_verts=6000, max_faces=11000)
    for i, m in enumerate(meshes):
        c.upload_mesh(i, m)
    return c, augment.BackgroundBank(c, PHOTOS[:4])


def test_make_device_batch_with_augmentation_trains():
    K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
    B = 2
    meshes = [synth.make_cube(), synth.make_blob()]
    c, bank = make_ctx(meshes, B)
    try:
        plain, _, _, _ = make_device_batch(c, meshes, B, 11, K, MEANS)
        aug, _, _, _ = make_device_batch(c, meshes, B, 11, K, MEANS, background=(bank, 7), mask_dilate=7)
        # the augmented blobs differ from the plain ones exactly where the augmentation acts
        fg = plain["mask_gt_observed"] != 0
        io, ip = aug["image_observed"], plain["image_observed"]
        assert torch.equal(io.masked_select(fg.expand_as(io)), ip.masked_select(fg.expand_as(ip)))
        assert not torch.equal(io, ip)
        assert (aug["mask_observed"] >= plain["mask_observed"]).all() and not torch.equal(aug["mask_observed"], plain["mask_observed"])
        for k in ("image_rendered", "mask_gt_observed", "src_pose", "flow"):
            assert torch.equal(aug[k], plain[k]), k
    finally:
        c.close()
    # three augmented batches through one bf16 trainer: finite objectives, the observed mask and image fixed across the inner
    # iterations, and (as the existing fit_batch tests assert for a fresh trainer on seed 11) the objective of the first
    # batch falls over its inner iterations
    c, bank = make_ctx(meshes, B)
    try:
        tr = Trainer(c, synth.make_train_weights(0), precision="bf16")
        seen = []
        zoom_front = tr.zoom_front

        def recording_zoom_front(b, K_):
            seen.append((b["mask_observed"].clone(), b["image_observed"].clone()))
            return zoom_front(b, K_)

        tr.zoom_front = recording_zoom_front
        objs = []
        for s in (11, 12, 13):
            batch, cls, tgt, depth = make_device_batch(c, meshes, B, s, K, MEANS, background=(bank, s), mask_dilate=s)
            mo, im = batch["mask_observed"].clone(), batch["image_observed"].clone()
            del seen[:]
            o = fit_batch(tr, batch, cls, tgt, depth, K, n_inner=4).cpu().numpy()
            assert o.shape == (4,) and np.isfinite(o).all(), o
            assert len(seen) == 4 and all(torch.equal(m, mo) and torch.equal(i, im) for m, i in seen)
            objs.append(o)
        assert objs[0][-1] < objs[0][0], objs
    finally:
        c.close()
