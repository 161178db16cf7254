"""CPU: the host side of the train-time augmentation (deepim_b200.augment) against fixtures made by the live reference
(tests/golden/make_golden_augment.py): the mask-dilation draws, the background crop / resize geometry, and the composite
of image.py:147-157 restated in numpy."""
import os

import numpy as np
import pytest

from deepim_b200 import augment

HERE = os.path.dirname(os.path.abspath(__file__))
BG = np.load(os.path.join(HERE, "golden", "ref_background.npz"))
DIL = np.load(os.path.join(HERE, "golden", "ref_mask_dilate.npz"))
H, W = 480, 640


def dilate_with_draws(mask, d):
    """mask_dilate.py:19-47 driven by one row of mask_dilate_draws instead of np.random"""
    out = mask.astype(np.float64).copy()
    t = d[1:]
    if t[0]:
        out[t[0]:] += np.logical_and(mask[:-t[0]] != 0, mask[t[0]:] == 0)
    if t[1]:
        out[:-t[1]] += np.logical_and(mask[t[1]:] != 0, mask[:-t[1]] == 0)
    if t[2]:
        out[:, t[2]:] += np.logical_and(mask[:, :-t[2]] != 0, mask[:, t[2]:] == 0)
    if t[3]:
        out[:, :-t[3]] += np.logical_and(mask[:, t[3]:] != 0, mask[:, :-t[3]] == 0)
    out[out > 1] = 1
    return out


def test_mask_dilate_draws_reproduce_the_seeded_reference():
    for m, s, ref in zip(DIL["mask"], DIL["seed"], DIL["out"]):
        d = augment.mask_dilate_draws(1, np.random.RandomState(int(s)))[0]
        assert d.dtype == np.int32
        assert 0 <= d[0] < 10 and all(t == 0 or 1 <= t <= 10 for t in d[1:])
        np.testing.assert_array_equal(dilate_with_draws(m, d), ref)


def test_mask_dilate_draws_follow_the_call_order():
    rs, ref = np.random.RandomState(5), np.random.RandomState(5)
    got = augment.mask_dilate_draws(4, rs)
    for row in got:
        d = ref.randint(10)
        assert row[0] == d
        for k, skip in enumerate(((0, 1, 4), (1, 2, 5), (2, 3, 6), (0, 3, 7))):
            assert row[1 + k] == (0 if d in skip else ref.randint(10) + 1)
    assert rs.randint(1 << 30) == ref.randint(1 << 30)  # nothing more was consumed


def test_dilation_grows_a_box_into_a_cross():
    m = np.zeros((H, W), np.float32)
    m[100:200, 300:400] = 1
    out = dilate_with_draws(m, np.array([9, 3, 4, 5, 6]))
    assert out[96, 300] == 1 and out[95, 300] == 0  # the up shift (4 px) fills rows 96..99 above the box
    assert out[150, 294] == 1 and out[150, 293] == 0  # the left shift (6 px)
    assert out[96, 299] == 0 and out[202, 405] == 0  # corners stay empty: every shift reads the original box


def test_background_geometry_matches_every_fixture_case():
    for i in np.flatnonzero(BG["bank_index"] >= 0):
        bh, bw = BG["photo_shapes"][BG["bank_index"][i]]
        ch, cw, dh, dw, fx = augment.background_geometry(H, W, int(bh), int(bw))
        assert (ch, cw) == tuple(BG["crop_hw"][i]), i
        assert (dh, dw) == tuple(BG["dst_hw"][i]), i
        assert fx == BG["fx"][i], i


def test_background_geometry_refuses_what_it_cannot_reproduce():
    with pytest.raises(Exception, match="INTER_AREA"):
        augment.background_geometry(H, W, 960, 1279)  # scale exactly 1/2 with an odd crop side
    assert augment.background_geometry(H, W, 960, 1280)[2:4] == (480, 640)


def test_composite_restated_in_numpy_equals_the_fixture():
    for i in range(len(BG["bank_index"])):
        obs, mask, comp = BG["observed"], BG["mask"][i], BG["composite"][i]  # one observed image for every case
        if BG["bank_index"][i] < 0:
            np.testing.assert_array_equal(comp, obs)
            continue
        dh, dw = BG["dst_hw"][i]
        bg = np.zeros((H, W, 3), np.uint8)
        bg[:dh, :dw] = BG["resized"][i][:dh, :dw]
        res = bg.copy()
        fg = np.dstack([mask] * 3) != 0
        res[fg] = obs[fg]
        np.testing.assert_array_equal(res, comp)
        assert (BG["resized"][i][dh:] == 0).all() and (BG["resized"][i][:, dw:] == 0).all()


def test_background_draws():
    rs = np.random.RandomState(3)
    idx = augment.background_draws(6, rs, 4, data_syn=True)
    ref = np.random.RandomState(3)
    assert idx.tolist() == [ref.randint(4) for _ in range(6)]
    assert (augment.background_draws(5, np.random.RandomState(0), 4, data_syn=False, ratio=0.0) == -1).all()
    mixed = augment.background_draws(4, np.random.RandomState(1), 4, data_syn=[True, False, True, False], ratio=1.0)
    assert (mixed >= 0).all()
    with pytest.raises(ValueError, match="empty"):
        augment.background_draws(1, np.random.RandomState(0), 0)
