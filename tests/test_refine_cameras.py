"""CPU: one camera per frame on the host side -- the batch plan carries each batch's cameras with its frames, the shape
checks of Context's per-frame K, and lm6d_io's per-pair `-K.txt`."""
import os

import numpy as np
import pytest


def cams(n, seed):
    rng = np.random.default_rng(seed)
    K = np.zeros((n, 3, 3), np.float32)
    K[:, 0, 0], K[:, 1, 1] = rng.uniform(500, 1100, n), rng.uniform(500, 1100, n)
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = rng.uniform(250, 400, n), rng.uniform(180, 300, n), 1.0
    return K


@pytest.mark.parametrize("n,n_frames,max_batch,seed", [(37, 11, 16, 0), (16, 6, 16, 1), (5, 1, 16, 2), (64, 64, 8, 3),
                                                       (100, 7, 13, 4)])
def test_plan_frame_batches_carries_the_cameras(n, n_frames, max_batch, seed):
    from deepim_b200.refiner import plan_frame_batches
    frame_of = np.random.default_rng(seed).integers(0, n_frames, size=n)
    K = cams(n_frames, seed)
    plan = plan_frame_batches(frame_of, n_frames, max_batch, K_frames=K.astype(np.float64))
    plain = plan_frame_batches(frame_of, n_frames, max_batch)
    assert len(plan) == len(plain)
    for (a, b, frames, local, k), (a2, b2, frames2, local2) in zip(plan, plain):
        assert (a, b) == (a2, b2) and np.array_equal(frames, frames2) and np.array_equal(local, local2)
        assert k.dtype == np.float32 and k.shape == (len(frames), 3, 3) and k.flags.c_contiguous
        assert np.array_equal(k, K[frames])
        assert np.array_equal(k[local], K[frame_of[a:b]])     # row local[i] is instance a + i's camera


def test_plan_frame_batches_camera_shape_is_checked():
    from deepim_b200.refiner import plan_frame_batches
    with pytest.raises(ValueError, match=r"K_frames: expected shape \(4, 3, 3\)"):
        plan_frame_batches([0, 1, 2, 3], 4, 16, K_frames=cams(3, 0))
    with pytest.raises(ValueError, match="K_frames: expected shape"):
        plan_frame_batches([0, 1], 2, 16, K_frames=np.zeros((2, 9), np.float32))


def test_context_per_frame_camera_shapes():
    torch = pytest.importorskip("torch")
    from deepim_b200.context import _per_frame_k
    one = np.eye(3, dtype=np.float32)
    assert _per_frame_k(one, 4) is False                      # [3,3]: one camera, K9
    assert _per_frame_k(one.reshape(9), 4) is False           # nine values, as before
    assert _per_frame_k(np.stack([one] * 4), 4) is True       # [F,3,3]: K_frames
    assert _per_frame_k(torch.from_numpy(np.stack([one] * 2)), 2) is True
    for bad in (np.stack([one] * 3), np.zeros((4, 3, 4), np.float32), np.zeros((4, 9, 1), np.float32)):
        with pytest.raises(ValueError, match=r"one camera per frame\), got"):
            _per_frame_k(bad, 4)


def test_load_pair_reads_the_frames_camera_and_falls_back_without_it(tmp_path):
    import lm6d_fixture
    from deepim_b200 import lm6d_io
    classes, _ = lm6d_fixture.build(str(tmp_path), n_per_class=2)
    ds = lm6d_io.LM6DRefine(str(tmp_path), classes, "val")
    pairs = ds.pairs(classes[1])
    K2 = np.array([[1066.778, 0.0, 312.9869], [0.0, 1067.487, 241.3109], [0.0, 0.0, 1.0]])
    np.savetxt(os.path.join(str(tmp_path), "data", "observed", pairs[1][0] + "-K.txt"), K2)
    with_k, without = ds.load_pair(classes[1], pairs[1]), ds.load_pair(classes[1], pairs[0])
    assert with_k["K"].shape == (3, 3) and with_k["K"].dtype == np.float64 and np.array_equal(with_k["K"], K2)
    assert "K" not in without
    assert set(with_k) - {"K"} == set(without)
