"""CPU: the bf16x3 training step's C entry points, and the calibration of its GPU tolerances (tests/test_gpu_train_bf16x3.py)
by the CPU emulation of its storage format (tests/bf16x3_emulation.py) on the batch of tests/test_gpu_train.py.

Recorded on that batch (1 - cosine against the fp32 oracle, parameter gradients): emulate_bf16 2.6e-12 .. 7.2e-4 (conv6_weight),
emulate_bf16x3 <= 1.3e-7 (flow_conv1_weight), at least 330x closer on every tensor whose bf16 cosine is not exactly 1."""
import ctypes
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import train_oracle as T  # noqa: E402
from deepim_b200 import synth  # noqa: E402
import bf16x3_emulation as E  # noqa: E402
import gpu_train_check as G  # noqa: E402

K, MEANS = synth.K_LINEMOD, synth.PIXEL_MEANS_RGB
# the floor of tests/test_gpu_train_bf16x3.py's gradient rule 1 - cos <= max(0.1 (1 - cos_bf16), floor): the emulation's worst
# parameter gradient (1.3e-7) with room for the device's summation order
GRAD_FLOOR = 1e-6
# the device's 1 - cos may exceed the emulation's by this factor, or reach DEVICE_FLOOR: the emulation sums exactly, the
# tensor cores accumulate fp32 with their own rounding, so the device's activations carry ~1e-4 relative error where the
# emulation's carry ~1e-5, and LeakyReLU units that close to zero take the other slope (recorded: conv6_weight 1.7e-6 on the
# device, 9e-11 emulated)
DEVICE_MARGIN, DEVICE_FLOOR = 10.0, 5e-6


def test_precision_entry_points_are_exported():
    from deepim_b200 import _capi as capi
    lib = ctypes.CDLL(capi.LIB_PATH)
    for name in ("dim_train_set_precision", "dim_train_get_precision"):
        assert hasattr(lib, name), name
    assert capi.lib.dim_train_set_precision.argtypes == [ctypes.c_void_p, ctypes.c_int32]
    assert capi.lib.dim_train_set_precision.restype is ctypes.c_int32
    assert capi.lib.dim_train_get_precision.argtypes[0] is ctypes.c_void_p
    assert capi.lib.dim_train_get_precision.argtypes[1]._type_ is ctypes.c_int32
    assert capi.lib.dim_train_get_precision.restype is ctypes.c_int32
    # both refuse a NULL context with a message instead of crashing
    assert capi.lib.dim_train_set_precision(None, capi.PREC_BF16X3) != 0
    p = ctypes.c_int32()
    assert capi.lib.dim_train_get_precision(None, ctypes.byref(p)) != 0


def test_pair_rounding_is_the_split_of_the_device():
    import torch
    x = torch.from_numpy(np.random.default_rng(0).normal(0, 3, 4096).astype(np.float32))
    hi = x.bfloat16().float()
    r = E.round_pair(x)
    assert torch.equal(r, hi + (x - hi).bfloat16().float())
    assert ((r - x).abs() <= x.abs() * 2.0 ** -16).all()       # ~16 significant bits
    assert torch.equal(x.bfloat16().float(), hi)               # Tensor.bfloat16 is restored outside graph()


@pytest.fixture(scope="module")
def grads():
    meshes = [synth.make_cube(), synth.make_blob()]
    w = synth.make_train_weights(0)
    batch = G.make_batch(meshes, 2, 11)                      # the batch of the GPU tests and of the recorded device run
    zin, lab = T.zoom_inputs(batch, K, MEANS)
    _, g32 = T.graph(w, zin, lab, requires_grad=True)
    _, g16 = T.graph(w, zin, lab, requires_grad=True, emulate_bf16=True)
    _, g3 = E.graph(w, zin, lab, requires_grad=True)
    return g32, g16, g3


def test_bf16x3_emulation_is_far_closer_to_fp32_than_bf16(grads):
    g32, g16, g3 = grads
    rows = {}
    for k in sorted(g32):
        if k in T.FROZEN or k.startswith("dz_"):
            continue
        c16, c3 = G.cmp(g16[k], g32[k])["cos"], G.cmp(g3[k], g32[k])["cos"]
        rows[k] = (c16, c3)
        assert 1 - c3 <= max(0.01 * (1 - c16), 1e-12), (k, c16, c3)   # 100x closer (the GPU rule asks for 10x)
        assert 1 - c3 <= GRAD_FLOOR / 5, (k, c3)                       # and well inside the GPU test's floor
    print("\n%-28s %-12s %s" % ("tensor", "1-cos bf16", "1-cos bf16x3"))
    for k, (c16, c3) in rows.items():
        print("%-28s %.3e    %.3e" % (k, 1 - c16, 1 - c3))


def test_bf16x3_storage_explains_the_device_gradient_deviation(grads):
    """The device cosines of a bf16x3 step on the same batch (tests/golden/train_check_device_bf16x3.json: tools/gpu_train_check.py
    --precision bf16x3 on an H100) lie within DEVICE_MARGIN / DEVICE_FLOOR of the emulation's, and the device closes at least
    95 % of the bf16 emulation's gap to fp32 on every tensor: what is left is the cost of the pair storage and of the tensor
    cores' accumulation, not a missing hi / lo term (that would leave a bf16-sized error on the tensors behind it)."""
    g32, g16, g3 = grads
    rec = json.load(open(os.path.join(ROOT, "tests", "golden", "train_check_device_bf16x3.json")))
    assert rec["precision"] == "bf16x3"
    dev = rec["grads"]
    assert set(k for k in g32 if not k.startswith("dz_")) == set(dev)
    for k, d in dev.items():
        if k in T.FROZEN:
            continue
        e3, e16 = G.cmp(g3[k], g32[k])["cos"], G.cmp(g16[k], g32[k])["cos"]
        assert 1 - d["cos"] <= max(DEVICE_MARGIN * (1 - e3), DEVICE_FLOOR), (k, d["cos"], e3)
        assert 1 - d["cos"] <= 0.05 * (1 - e16) + 1e-7, (k, d["cos"], e16)
