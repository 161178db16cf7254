"""The inference network's kernels one at a time, in every precision: each encoder layer (flow_conv1 through conv1_kernel,
conv2 ... conv6_1 through conv_igemm_persistent_kernel) against a float64 convolution of exactly the 16-bit input the device
stored (the seeded blob for conv1, act[i] for layer i), and fc6 (fc6_mma_kernel) + fc7 + the rot / trans heads against
float64 from the stored act[10].  Batch sizes whose tiles span images and end mid-image; the zero border and the images past
the batch left untouched; a full batch of a tight allocation.  Bound (tests/kernel_ref.py):
|dev - ref| <= rho |ref| + kappa 2^-24 S element by element, rho the output storage (fp16 2^-11, bf16 2^-8, bf16x3 2^-15)."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "mx-deepim_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import kernel_ref as R  # noqa: E402
from oracle.train_oracle import ENC  # noqa: E402
from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402

pytestmark = pytest.mark.gpu

H, W, MAXB = 480, 640, 16
MODES = {"fp16": capi.PREC_FP16, "bf16": capi.PREC_BF16, "bf16x3": capi.PREC_BF16X3}
KAPPA = R.KAPPA_INFER  # kappa per kernel family (tests/kernel_ref.py); printed when the module ends (pytest -s)
SIZES = [(H, W)]  # SIZES[i]: the interior of act[i], the input of encoder layer i (filled from the weights' kernel sizes)


@pytest.fixture(scope="module")
def weights():
    w = synth.make_weights(0)
    del SIZES[1:]
    for name, s, p in ENC:
        k = w[name + "_weight"].shape[-1]
        SIZES.append(((SIZES[-1][0] + 2 * p - k) // s + 1, (SIZES[-1][1] + 2 * p - k) // s + 1))
    return w


def _open(weights, max_batch):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    c = Context(0, max_batch=max_batch)
    c.load_weights(weights)
    return c


@pytest.fixture(scope="module")
def ctx(weights):
    c = _open(weights, MAXB)
    yield c
    c.close()
    print("\ninference kernels, largest kappa needed: " + json.dumps({k: float("%.4g" % v) for k, v in sorted(R.OBSERVED.items())}))


@pytest.fixture(scope="module")
def ctx5(weights):
    c = _open(weights, 5)
    yield c
    c.close()


def _blobs(B, seed):
    g = torch.Generator().manual_seed(seed)
    zio = (torch.rand(B, 3, H, W, generator=g) - 0.5) * 255
    zir = (torch.rand(B, 3, H, W, generator=g) - 0.5) * 255
    zmo = (torch.rand(B, 1, H, W, generator=g) > 0.5).float()
    zmr = (torch.rand(B, 1, H, W, generator=g) > 0.5).float()
    return zio, zir, zmo, zmr


def _forward(ctx, mode, B, seed):
    dev = torch.device("cuda", 0)
    blobs = _blobs(B, seed)
    rot, trans = ctx.net_forward(*[t.to(dev) for t in blobs], MODES[mode])
    return blobs, rot, trans


def _act(ctx, mode, idx, n):
    """act[idx] as stored for the first n images: hi, lo (bf16x3; else None) float32 [n, rows, cols, C] incl. border, and
    its interior (py, px, H, W)"""
    hi, g = ctx.debug_activation(idx, n, fp16=mode == "fp16")
    lo = ctx.debug_activation(idx, n, lo=True)[0] if mode == "bf16x3" else None
    return hi, lo, (g[3], g[4]) + SIZES[idx]


def _check_layer(ctx, weights, mode, layer, B, n, seed=None):
    """runs the network on a seeded batch of B and checks layer `layer` from its stored input; returns the first n images of
    its output buffer (hi, lo)"""
    name = ENC[layer][0]
    blobs = _forward(ctx, mode, B, B if seed is None else seed)[0]
    hi, lo, geo = _act(ctx, mode, layer + 1, n)
    assert np.isfinite(hi).all(), (name, mode, B)
    if layer == 0:
        zio, zir, zmo, zmr = blobs
        x = R.operand(torch.cat([zio / 255.0, zir / 255.0, zmo, zmr], dim=1), mode)
    else:
        ihi, ilo, igeo = _act(ctx, mode, layer, B)
        x = R.interior(ihi, igeo, B), R.interior(ilo, igeo, B)
    R.check_conv_layer(weights, mode, layer, B, x, (hi, lo), geo)
    for half in (hi, lo):
        assert half is None or R.border_is_zero(half, geo, B), "%s wrote into the zero border (%s, B=%d)" % (name, mode, B)
    return hi, lo


LAYER_IDS = [name for name, _, _ in ENC]


@pytest.mark.parametrize("layer", range(10), ids=LAYER_IDS)
@pytest.mark.parametrize("mode", sorted(MODES))
def test_layer_matches_float64_and_keeps_borders(ctx, weights, mode, layer):
    """B = 1, 3, 16 on one context: row runs and tiles that end mid-image, span images, or leave a short last run"""
    # fill every image of the buffer first, so that a smaller batch writing past its last image would show
    _forward(ctx, mode, MAXB, 99)
    before = _act(ctx, mode, layer + 1, MAXB)[:2]
    for B in (1, 3, MAXB):
        got = _check_layer(ctx, weights, mode, layer, B, MAXB)
        if B < MAXB:
            for g, b0 in zip(got, before):
                assert g is None or np.array_equal(g[B:], b0[B:]), "%s wrote past image %d (%s)" % (ENC[layer][0], B - 1, mode)


@pytest.mark.parametrize("layer", range(10), ids=LAYER_IDS)
@pytest.mark.parametrize("mode", sorted(MODES))
def test_layer_full_batch_of_a_tight_allocation(ctx5, weights, mode, layer):
    """A full batch (B = max_batch) ends its input buffer at the batch's last input row.  For conv1 the run of rows that ends
    there is 3 strips longer than its output rows; max_batch = 5 puts that end 49 KB short of the 2 MiB granule the buffer's
    allocation is rounded to, less than the 62 KB of 3 strips: conv1 reads none of them.  The other layers' tiles past the
    last image are virtual rows, masked in the epilogue."""
    _check_layer(ctx5, weights, mode, layer, 5, 5)


@pytest.fixture(scope="module")
def ctx33(weights):
    c = _open(weights, 33)
    yield c
    c.close()


def _fc6_cases(ctx, weights, mode, batches):
    for B in batches:
        _, rot, trans = _forward(ctx, mode, B, 50 + B)
        hi, lo, _ = _act(ctx, mode, 10, B)
        R.check_fc6_heads(weights, mode, B, (hi, lo), rot, trans)


@pytest.mark.parametrize("mode", sorted(MODES))
def test_fc6_and_heads_match_float64(ctx, weights, mode):
    """rot / trans of net_forward against float64 fc6 -> fc7 -> heads from the stored act[10] (kernel_ref.check_fc6_heads).
    B = 1, 3, 9, 16: the batch is the M rows of mma.m16n8k16, B = 9 and 16 use both 8-row halves."""
    _fc6_cases(ctx, weights, mode, (1, 3, 9, MAXB))


@pytest.mark.parametrize("mode", sorted(MODES))
def test_fc6_and_heads_match_float64_above_16_instances(ctx33, weights, mode):
    """The same check past one M chunk of fc6_mma_kernel (bench.py's C5 configuration batches 128 instances): B = 17 (a
    one-row second chunk), 24, 32 (two full chunks) and 33 (three chunks, a one-row tail) on a max_batch = 33 context."""
    _fc6_cases(ctx33, weights, mode, (17, 24, 32, 33))
