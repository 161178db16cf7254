"""Generate the augmentation fixtures from the LIVE reference (runs only where /root/reference exists).

    python tests/golden/make_golden_augment.py   # rewrites tests/golden/ref_mask_dilate.npz, ref_background.npz

mask dilation: lib/utils/mask_dilate.mask_dilate under np.random.seed(s), on masks with boxes touching each border, a blob
and non-binary values.
background replacement: lib/utils/image.get_pair_image(pairdb, config, "train") on temporary files -- a config stand-in
and a fake VOCdevkit/VOC2012 tree whose photos are PNG bytes under .jpg names (cv2.imread decodes by content, so the
fixture does not depend on a JPEG decoder).  Each case lists one photo in diningtable_trainval.txt, so the photo a case
uses is known; random and np.random are seeded before each call.  The resized photo the reference composites is captured
by wrapping the module's resize().
Nothing from the reference is copied: this script only *calls* it and stores inputs/outputs.
"""
import os
import random
import sys
import tempfile
from types import SimpleNamespace

import cv2
import numpy as np

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
H, W = 480, 640
PIXEL_MEANS_BGR = np.array([103.06, 115.90, 123.15])  # the shipped yaml's network.PIXEL_MEANS (B, G, R)
# photo shapes: landscape (VOC's 375x500), portrait, square, a landscape narrower than 4:3 (stays 600 wide), a portrait
# that comes out 639 wide, a crop that hits the round(scale * max) > 640 cap, a downscaled one, exact 1/2 scale (cv2's INTER_AREA
# switch, equal to the linear result on full 2x2 cells)
PHOTOS = [(375, 500), (500, 333), (400, 400), (480, 600), (300, 350), (301, 700), (600, 900), (960, 1280), (700, 400)]


def texture(rng, h, w):
    """uint8 [h, w, 3] of random 15x19 blocks of 4 levels (0 and 255 among them): every resize tap pattern occurs at the
    block edges, and the fixtures stay small once compressed"""
    blocks = (rng.integers(0, 4, (h // 15 + 1, w // 19 + 1, 3)) * 85).astype(np.uint8)
    return np.ascontiguousarray(blocks.repeat(15, 0).repeat(19, 1)[:h, :w])


def import_reference():
    if not os.path.isdir(REF):
        raise SystemExit("reference not present; fixtures are committed, nothing to do")
    sys.path.insert(0, REF)
    from lib.utils import image as image_mod
    from lib.utils.mask_dilate import mask_dilate
    return image_mod, mask_dilate


def dilate_masks(rng):
    out = []
    for y0, y1, x0, x1 in ((0, 60, 200, 300), (420, 480, 100, 250), (150, 260, 0, 40), (300, 420, 590, 640), (200, 290, 280, 410)):
        m = np.zeros((H, W), np.float64)
        m[y0:y1, x0:x1] = 1.0
        out.append(m)
    yy, xx = np.mgrid[0:H, 0:W]
    out.append((((yy - 240) / 90.0) ** 2 + ((xx - 330) / 140.0) ** 2 < 1).astype(np.float64))  # blob
    m = np.zeros((H, W), np.float64)  # non-binary values (exact in float32)
    m[100:200, 100:260] = rng.choice([0.5, 1.0, 2.0, 3.0, -1.0, 0.25, 0.0], size=(100, 160))
    out.append(m)
    return out


def main():
    image_mod, mask_dilate = import_reference()
    rng = np.random.default_rng(20261016)

    masks, seeds, outs = [], [], []
    for i, m in enumerate(dilate_masks(rng)):
        for s in (3 * i, 3 * i + 1, 3 * i + 2):
            np.random.seed(s)
            outs.append(mask_dilate(m.copy()))
            masks.append(m)
            seeds.append(s)
    np.savez_compressed(os.path.join(HERE, "ref_mask_dilate.npz"), mask=np.asarray(masks, np.float32),
                        seed=np.asarray(seeds, np.int64), out=np.asarray(outs, np.float64))

    photos = [texture(rng, h, w) for h, w in PHOTOS]
    calls = []
    real_resize = image_mod.resize

    def resize(im, target_size, max_size, *a, **k):
        r, s = real_resize(im, target_size, max_size, *a, **k)
        calls.append((im.shape, r, s))
        return r, s

    image_mod.resize = resize
    cases = []  # (photo index or -1, data_syn, ratio, seed)
    for p in range(len(PHOTOS)):
        cases.append((p, True, 0.0, 100 + p))
    cases += [(1, False, 1.0, 200), (2, False, 0.0, 201)]
    obs = texture(rng, H, W)  # one observed image for every case (stored once)
    rec = {k: [] for k in ("bank_index", "mask", "composite", "resized", "crop_hw", "dst_hw", "fx", "seed")}
    with tempfile.TemporaryDirectory() as root:
        voc = os.path.join(root, "VOCdevkit", "VOC2012")
        os.makedirs(os.path.join(voc, "ImageSets", "Main"))
        os.makedirs(os.path.join(voc, "JPEGImages"))
        for i, ph in enumerate(photos):
            cv2.imwrite(os.path.join(voc, "JPEGImages", "bg%04d.png" % i), ph)
            os.replace(os.path.join(voc, "JPEGImages", "bg%04d.png" % i), os.path.join(voc, "JPEGImages", "bg%04d.jpg" % i))
        for ci, (p, syn, ratio, seed) in enumerate(cases):
            with open(os.path.join(voc, "ImageSets", "Main", "diningtable_trainval.txt"), "w") as f:
                f.write("bg%04d -1\nbg%04d  1\n" % ((p + 1) % len(photos), p))
            mask = np.zeros((H, W), np.uint8)
            yy, xx = np.mgrid[0:H, 0:W]
            mask[((yy - 200 - 7 * ci) / 110.0) ** 2 + ((xx - 300 - 11 * ci) / 170.0) ** 2 < 1] = 1 + ci
            for name, a in (("obs.png", obs), ("ren.png", obs[::-1].copy()), ("mask.png", mask)):
                cv2.imwrite(os.path.join(root, name), a)
            config = SimpleNamespace(SCALES=[(H, W)], TRAIN=SimpleNamespace(REPLACE_OBSERVED_BG_RATIO=ratio),
                                     dataset=SimpleNamespace(root_path=root),
                                     network=SimpleNamespace(PIXEL_MEANS=PIXEL_MEANS_BGR))
            pair = {"img_flipped": False, "image_observed": os.path.join(root, "obs.png"),
                    "image_rendered": os.path.join(root, "ren.png"), "data_syn": syn,
                    "mask_gt_observed": os.path.join(root, "mask.png")}
            random.seed(seed)
            np.random.seed(seed)
            del calls[:]
            ims_obs, _, _ = image_mod.get_pair_image([pair], config, "train")
            replaced = len(calls) == 3  # observed, rendered, then the photo's crop
            rec["bank_index"].append(p if replaced else -1)
            rec["mask"].append(mask)
            # the tensor is stored as the uint8 composite it was made from (a tenth of the bytes), after checking that
            # transform() of that composite gives the reference's tensor exactly
            t = ims_obs[0][0]
            comp = np.rint(t[::-1].transpose(1, 2, 0) + PIXEL_MEANS_BGR).astype(np.uint8)
            assert np.array_equal(image_mod.transform(comp, PIXEL_MEANS_BGR)[0], t)
            rec["composite"].append(comp)
            res = np.zeros((H, W, 3), np.uint8)
            crop_hw, dst_hw, fx = (0, 0), (0, 0), 0.0
            if replaced:
                shp, r, fx = calls[2]
                res[:r.shape[0], :r.shape[1]] = r
                crop_hw, dst_hw = shp[:2], r.shape[:2]
            rec["resized"].append(res)
            rec["crop_hw"].append(crop_hw)
            rec["dst_hw"].append(dst_hw)
            rec["fx"].append(fx)
            rec["seed"].append(seed)
    out = {k: np.asarray(v) for k, v in rec.items()}
    out["observed"] = obs
    out["pixel_means_bgr"] = PIXEL_MEANS_BGR
    out["photo_shapes"] = np.asarray(PHOTOS, np.int32)
    for i, ph in enumerate(photos):
        out["photo%d" % i] = ph
    np.savez_compressed(os.path.join(HERE, "ref_background.npz"), **out)
    print("wrote", len(seeds), "dilation cases and", len(cases), "background cases")


if __name__ == "__main__":
    main()
