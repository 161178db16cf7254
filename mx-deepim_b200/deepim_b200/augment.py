"""Train-time augmentation of the observed inputs, on the device: background replacement of synthetic observed images
(lib/utils/image.py:96-157) and observed-mask dilation (lib/utils/mask_dilate.py, TRAIN.MASK_DILATE).

The random draws are the caller's.  The reference draws them inside its multiprocessing.Pool workers, so its own sequence
is not reproducible; the helpers below consume a generator in the reference's call order, so that seeding it like the
reference's global state reproduces one live call."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._capi import check, lib


class BackgroundBank:
    """BGR uint8 photos [h, w, 3] (as cv2.imread decodes them) uploaded once to ctx's background bank at indices
    0 .. len(images) - 1 (dim_bg_upload)."""

    def __init__(self, ctx, images):
        self.ctx = ctx
        self.shapes = []
        for i, im in enumerate(images):
            a = np.ascontiguousarray(im, np.uint8)
            if a.ndim != 3 or a.shape[2] != 3:
                raise ValueError("background %d: expected a BGR uint8 [h, w, 3] image, got shape %s" % (i, a.shape))
            check(lib.dim_bg_upload(ctx._h, i, a.ctypes.data, a.shape[0], a.shape[1]))
            self.shapes.append(a.shape[:2])

    def __len__(self):
        return len(self.shapes)


def background_geometry(H, W, bh, bw):
    """(crop_h, crop_w, dst_h, dst_w, fx) of a bh x bw photo on an H x W canvas (dim_bg_geometry: image.py:108-145 and
    resize, image.py:552-572, in float64)."""
    out4, scale = (C.c_int32 * 4)(), C.c_double()
    check(lib.dim_bg_geometry(H, W, bh, bw, out4, C.byref(scale)))
    return tuple(out4) + (scale.value,)


def mask_dilate_draws(B, rs, max_thickness=10):
    """int32 [B, 5] draws of dim_mask_dilate: direction, then the thickness of the down, up, right and left shift (0 =
    skipped), taken from the legacy np.random.RandomState `rs` in mask_dilate's call order (randint(10), then one
    randint(max_thickness) + 1 per applied side), one instance after the other."""
    out = np.zeros((B, 5), np.int32)
    for b in range(B):
        d = rs.randint(10)
        out[b, 0] = d
        for k, skip in enumerate(((0, 1, 4), (1, 2, 5), (2, 3, 6), (0, 3, 7))):
            if d not in skip:
                out[b, 1 + k] = rs.randint(max_thickness) + 1
    return out


def background_draws(B, rng, n_bank, data_syn=True, ratio=0.0):
    """int32 [B] bank indices of dim_replace_background (-1 = keep the observed image), as image.py:97-113 decides: a
    synthetic instance (data_syn) always gets a photo, a real one with probability `ratio`
    (TRAIN.REPLACE_OBSERVED_BG_RATIO); the photo is uniform over the bank.  rng: a np.random.RandomState; data_syn: one
    bool for the batch or one per instance."""
    syn = np.broadcast_to(np.asarray(data_syn, bool), (B,))
    out = np.full(B, -1, np.int32)
    for b in range(B):
        if syn[b] or rng.rand() < ratio:
            if n_bank < 1:
                raise ValueError("background_draws: the bank is empty")
            out[b] = rng.randint(n_bank)
    return out
