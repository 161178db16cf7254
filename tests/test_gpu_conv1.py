"""flow_conv1 (conv1_kernel) on its own, in every precision, at batch sizes whose row runs end mid-image or leave a short
last run: the stored activation against a torch conv2d of the same 16-bit input blob, the zero border and the images past
the batch left untouched, every value finite."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "mx-deepim_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402

pytestmark = pytest.mark.gpu

H, W, MAXB = 480, 640, 16
# per precision: (mode, how the device rounds conv1's operands, bound on |act - ref| relative to max(1, |ref|max)).
# The reference sees the same rounded operands, so what is left is the 16-bit output rounding and the fp32 summation order.
MODES = {
    "fp16": (capi.PREC_FP16, lambda t: t.half().double(), 2.5e-3),
    "bf16": (capi.PREC_BF16, lambda t: t.bfloat16().double(), 8e-3),
    "bf16x3": (capi.PREC_BF16X3, lambda t: t.double(), 2e-4),
}


@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(0)


@pytest.fixture(scope="module")
def ctx(weights):
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    c = Context(0, max_batch=MAXB)
    c.load_weights(weights)
    yield c
    c.close()


def _blobs(B, seed):
    g = torch.Generator().manual_seed(seed)
    zio = (torch.rand(B, 3, H, W, generator=g) - 0.5) * 255
    zir = (torch.rand(B, 3, H, W, generator=g) - 0.5) * 255
    zmo = (torch.rand(B, 1, H, W, generator=g) > 0.5).float()
    zmr = (torch.rand(B, 1, H, W, generator=g) > 0.5).float()
    return zio, zir, zmo, zmr


def _act1(ctx, mode, n=MAXB):
    """conv2's bordered input buffer for the first n images (hi + lo in bf16x3)."""
    a, g = ctx.debug_activation(1, n, fp16=mode == "fp16")
    if mode == "bf16x3":
        a = a + ctx.debug_activation(1, n, lo=True)[0]
    return a, g


def _check_batch(ctx, weights, mode, B, n):
    """runs conv1 on a seeded batch of B; checks the first n images of its output buffer, returns them."""
    prec, rnd, tol = MODES[mode]
    dev = torch.device("cuda", 0)
    w = rnd(torch.from_numpy(np.asarray(weights["flow_conv1_weight"], np.float32))).to(dev)
    b = torch.from_numpy(np.asarray(weights["flow_conv1_bias"], np.float32)).double().to(dev)
    zio, zir, zmo, zmr = _blobs(B, B)
    ctx.net_forward(zio.to(dev), zir.to(dev), zmo.to(dev), zmr.to(dev), prec)
    act, g = _act1(ctx, mode, n)
    py, px, Ho, Wo = g[3], g[4], 240, 320  # g[5:7] are conv2's output extent
    assert np.isfinite(act).all(), (mode, B)
    x = rnd(torch.cat([zio / 255.0, zir / 255.0, zmo, zmr], dim=1)).to(dev)
    ref = F.leaky_relu(F.conv2d(x, w, b, stride=2, padding=3), 0.1).permute(0, 2, 3, 1).cpu().numpy()
    inner = act[:B, py:py + Ho, px:px + Wo, :]
    err = np.abs(inner - ref).max()
    assert err < tol * max(1.0, np.abs(ref).max()), (mode, B, err)
    border = act[:B].copy()
    border[:, py:py + Ho, px:px + Wo, :] = 0
    assert not border.any(), "conv1 wrote into the zero border (%s, B=%d)" % (mode, B)
    return act


@pytest.mark.parametrize("mode", sorted(MODES))
def test_conv1_matches_torch_and_keeps_borders(ctx, weights, mode):
    dev = torch.device("cuda", 0)
    # fill every image of the buffer first, so that a smaller batch writing past its last image would show
    ctx.net_forward(*[t.to(dev) for t in _blobs(MAXB, 99)], MODES[mode][0])
    before, _ = _act1(ctx, mode)
    for B in (1, 3, MAXB):
        act = _check_batch(ctx, weights, mode, B, MAXB)
        if B < MAXB:
            assert np.array_equal(act[B:], before[B:]), "conv1 wrote past image %d (%s)" % (B - 1, mode)


@pytest.mark.parametrize("mode", sorted(MODES))
def test_conv1_full_batch_of_a_tight_allocation(weights, mode):
    """A full batch (B = max_batch) ends its input buffer at the batch's last input row, and the run of rows that ends
    there is 3 strips longer than its output rows.  max_batch = 5 puts that end 49 KB short of the 2 MiB granule the
    buffer's allocation is rounded to, less than the 62 KB of 3 strips: conv1 reads none of them."""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    c = Context(0, max_batch=5)
    try:
        c.load_weights(weights)
        _check_batch(c, weights, mode, 5, 5)
    finally:
        c.close()
