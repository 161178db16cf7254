"""Lighting of the ModelNet (unseen-object) configuration.

When config.dataset.dataset starts with "ModelNet" the reference renders every pose of its test loop
(deepim/core/tester.py:146-185) and of its train-time batch update (lib/pair_matching/batch_updater_py_multi.py:187-229)
with the Lambert-lit Render_Py_Light_ModelNet_Multi.  Per render, with `pose` the float64 pose being rendered:

    light_position = np.array([0, 1, 1]) * 0.5             # light index 2, hard-coded
    light_position[0] += pose[0, 3]; light_position[1] -= pose[1, 3]; light_position[2] -= pose[2, 3]
    light_intensity = np.random.uniform(0.9, 1.1, size=(3,))   # a fresh draw per render
    brightness_ratio = 0.7

glumpy casts both uniforms to float32.  The random intensity is an input here: sample_intensity draws it from a seeded
numpy Generator, the library takes whatever the caller passes.

A `lighting` argument of Context.refine / refine_host / train_update is a dict
    {"intensity": float32 [..., 3], "offset": (0, 0.5, 0.5), "brightness_ratio": 0.7}
(offset and brightness_ratio optional).  PoseRefiner, trainer.make_device_batch and trainer.fit_batch draw the intensities
themselves and take {"seed", "offset", "brightness_ratio"} (or a LightSource).
"""
from __future__ import annotations

import numpy as np

OFFSET = (0.0, 0.5, 0.5)   # light index 2 of the reference: [0, 1, 1] * 0.5
BRIGHTNESS_RATIO = 0.7     # brightness_ratios=[0.7], brightness_k = 0
INTENSITY_RANGE = (0.9, 1.1)


def sample_intensity(rng: np.random.Generator, shape) -> np.ndarray:
    """Light intensities for `shape` renders: float32 [*shape, 3], each channel U(0.9, 1.1) drawn in float64 (as
    np.random.uniform) and cast to float32 (as the glumpy uniform)."""
    shape = (int(shape),) if np.isscalar(shape) else tuple(int(s) for s in shape)
    return rng.uniform(INTENSITY_RANGE[0], INTENSITY_RANGE[1], size=shape + (3,)).astype(np.float32)


def modelnet_light_position(pose_f64, offset=OFFSET) -> np.ndarray:
    """Light position in the GL camera frame for poses [..., 3, 4]: float32(offset + (t_x, -t_y, -t_z)) computed in float64
    from the float64 pose (the reference's arithmetic happens before anything is cast to float32)."""
    p = np.asarray(pose_f64, np.float64)
    o = np.asarray(offset, np.float64)
    return np.stack([o[0] + p[..., 0, 3], o[1] - p[..., 1, 3], o[2] - p[..., 2, 3]], axis=-1).astype(np.float32)


def params(lighting: dict):
    """(offset as 3 floats, brightness_ratio) of a lighting dict, with the reference's defaults."""
    offset = tuple(float(v) for v in lighting.get("offset", OFFSET))
    if len(offset) != 3:
        raise ValueError("lighting['offset'] must have 3 values, got %d" % len(offset))
    return offset, float(lighting.get("brightness_ratio", BRIGHTNESS_RATIO))


class LightSource:
    """A seeded light of the ModelNet branch: offset / brightness ratio fixed, a fresh intensity per render."""

    def __init__(self, seed=0, offset=OFFSET, brightness_ratio=BRIGHTNESS_RATIO):
        self.rng = np.random.default_rng(seed)
        self.offset, self.brightness_ratio = params({"offset": offset, "brightness_ratio": brightness_ratio})

    @classmethod
    def of(cls, lighting):
        """None -> None; a LightSource -> itself; a dict {"seed", "offset", "brightness_ratio"} -> a new LightSource."""
        if lighting is None or isinstance(lighting, LightSource):
            return lighting
        unknown = set(lighting) - {"seed", "offset", "brightness_ratio"}
        if unknown:
            raise ValueError("unknown lighting keys %s (expected seed, offset, brightness_ratio)" % sorted(unknown))
        return cls(lighting.get("seed", 0), lighting.get("offset", OFFSET), lighting.get("brightness_ratio", BRIGHTNESS_RATIO))

    def draw(self, shape) -> np.ndarray:
        return sample_intensity(self.rng, shape)

    def lighting(self, intensity) -> dict:
        """The per-call lighting dict of the Context methods for the given intensities."""
        return {"intensity": intensity, "offset": self.offset, "brightness_ratio": self.brightness_ratio}
