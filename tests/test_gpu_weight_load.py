"""GPU: the two ways weights reach the inference network build the same operand packs.  One context loads a checkpoint with
Context.load_weights (dim_net_load), another with Trainer (dim_train_load_params, whose flat vector holds fc6 permuted to
(256, hw, c)); net_forward on the same zoomed inputs must return bit-identical rot / trans in bf16 (the hi packs), bf16x3
(hi and lo) and fp16 (the fp16 packs: each weight rounded once from fp32, also on a training context), for the mask,
image-only and RGB-D networks."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from deepim_b200 import _capi as capi  # noqa: E402
from deepim_b200 import synth  # noqa: E402
from deepim_b200.context import Context  # noqa: E402
from deepim_b200.trainer import Trainer  # noqa: E402

H, W, B = 480, 640, 3
NETS = {"mask": {}, "nomask": {"input_mask": False}, "rgbd": {"input_depth": True}}


def _inputs(net, seed):
    g = torch.Generator().manual_seed(seed)
    rand = lambda c: torch.rand(B, c, H, W, generator=g)
    args = [(rand(3) - 0.5) * 255, (rand(3) - 0.5) * 255]
    args += [None, None] if net == "nomask" else [(rand(1) > 0.5).float(), (rand(1) > 0.5).float()]
    depths = {"zoom_depth_observed": rand(1) * 2, "zoom_depth_rendered": rand(1) * 2} if net == "rgbd" else {}
    dev = lambda t: None if t is None else t.cuda()
    return [dev(t) for t in args], {k: dev(t) for k, t in depths.items()}


@pytest.mark.parametrize("net", sorted(NETS))
def test_net_load_and_train_load_build_the_same_packs(net):
    w = synth.make_train_weights(5, **NETS[net])
    a = Context(0, max_batch=B, **NETS[net])
    b = Context(0, max_batch=B, **NETS[net])
    try:
        a.load_weights(w)
        Trainer(b, w)
        args, depths = _inputs(net, 7)
        for prec in (capi.PREC_BF16, capi.PREC_BF16X3, capi.PREC_FP16):
            ra, ta = a.net_forward(*args, precision=prec, **depths)
            rb, tb = b.net_forward(*args, precision=prec, **depths)
            torch.cuda.synchronize()
            assert np.isfinite(ra.cpu().numpy()).all() and ra.abs().max().item() > 0
            assert torch.equal(ra, rb), (net, prec)
            assert torch.equal(ta, tb), (net, prec)
    finally:
        a.close()
        b.close()
