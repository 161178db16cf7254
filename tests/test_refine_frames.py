"""CPU: PoseRefiner.refine_frames' batch plan (plan_frame_batches) is right."""
import numpy as np
import pytest


@pytest.mark.parametrize("n,n_frames,max_batch,seed", [(37, 11, 16, 0), (16, 3, 16, 1), (5, 1, 16, 2), (64, 64, 8, 3),
                                                       (100, 7, 13, 4), (1, 1, 1, 5)])
def test_plan_frame_batches(n, n_frames, max_batch, seed):
    from deepim_b200.refiner import plan_frame_batches
    frame_of = np.random.default_rng(seed).integers(0, n_frames, size=n)
    plan = plan_frame_batches(frame_of, n_frames, max_batch)
    seen = np.concatenate([np.arange(a, b) for a, b, _, _ in plan])
    assert np.array_equal(seen, np.arange(n))                  # every instance once, batches in input order
    for a, b, frames, local in plan:
        assert 1 <= b - a <= max_batch and 1 <= len(frames) <= min(b - a, max_batch)
        assert local.dtype == np.int32 and local.shape == (b - a,)
        assert np.array_equal(frames[local], frame_of[a:b])    # local indices point at the right frames
        assert np.array_equal(frames, np.unique(frame_of[a:b]))  # only the frames the batch observes, each once


def test_plan_frame_batches_of_a_shard_and_bad_indices():
    from deepim_b200 import sharding
    from deepim_b200.refiner import plan_frame_batches
    frame_of = np.array([0, 0, 1, 1, 1, 2, 2, 0, 3, 3])
    lo, hi = sharding.shard_range(len(frame_of), 1, 2)            # rank 1 of 2: instances 5..9
    plan = plan_frame_batches(frame_of, 4, 3, lo, hi)
    assert [(a, b) for a, b, _, _ in plan] == [(5, 8), (8, 10)]
    assert [f.tolist() for _, _, f, _ in plan] == [[0, 2], [3]]   # a rank uploads only the frames of its slice
    assert plan_frame_batches(frame_of, 4, 3, 5, 5) == []
    with pytest.raises(ValueError, match="instance 3 has frame index 4: out of range"):
        plan_frame_batches([0, 1, 2, 4], 4, 16)
    with pytest.raises(ValueError, match="instance 0 has frame index -1"):
        plan_frame_batches([-1, 0], 4, 16)
