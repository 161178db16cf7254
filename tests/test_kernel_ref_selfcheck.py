"""CPU: the float64 backward references of tests/kernel_ref.py that the training-step kernel tests hold the device to are
the derivatives of their forward references (torch autograd, float64, small random inputs), and its Transform3D
restatement agrees with the oracle's.  A wrong reference would otherwise pass a wrong kernel."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import kernel_ref as R  # noqa: E402
from oracle import oracle as O  # noqa: E402


def rand(g, *shape):
    return torch.randn(*shape, generator=g, dtype=torch.float64)


def vjp(f, x, g):
    """g^T d f / d x by autograd"""
    x = x.detach().clone().requires_grad_(True)
    (out,) = torch.autograd.grad(f(x), x, g)
    return out


def close(a, b):
    assert a.shape == b.shape
    assert torch.allclose(a, b, rtol=1e-12, atol=1e-12 * float(b.abs().max())), float((a - b).abs().max())


@pytest.mark.parametrize("hw", [(3, 4), (5, 2)])
def test_upsample_bwd_is_the_adjoint(hw):
    """upsample_bwd = autograd of the cropped grouped k32 s16 deconvolution, for the flow (2 groups) and the mask kernel,
    at an image size that clips the footprints on every side"""
    g = torch.Generator().manual_seed(1)
    h, w = hw
    H, W = 16 * h - 3, 16 * w + 1 - 8  # footprints clipped at the bottom / right as well as by the crop at the top / left
    for C in (2, 1):
        k = rand(g, C, 1, 32, 32)
        x, d = rand(g, 2, C, h, w), rand(g, 2, C, H, W)
        assert R.upsample_fwd(x, k, H, W).shape == d.shape
        close(R.upsample_bwd(d, k, h, w), vjp(lambda t: R.upsample_fwd(t, k, H, W), x, d))


def test_thin_deconv_backward_and_weight_gradient():
    """deconv_dgrad and deconv_wgrad = autograd of deconv_fwd (k4 s2 cropped by 1) for the 2 -> 2 upsample_flow layers"""
    g = torch.Generator().manual_seed(2)
    x, w = rand(g, 3, 2, 4, 5), rand(g, 2, 2, 4, 4)
    Ho, Wo = 8, 9
    d = rand(g, 3, 2, Ho, Wo)
    fwd = lambda a, ww: R.deconv_fwd((a, None), (ww, None), Ho, Wo)[0]
    close(R.deconv_dgrad((d, None), (w, None), 4, 5)[0], vjp(lambda t: fwd(t, w), x, d))
    close(R.deconv_wgrad((x, None), (d, None))[0], vjp(lambda t: fwd(x, t), w, d))


def test_l2_normalize_backward():
    g = torch.Generator().manual_seed(3)
    x, d = rand(g, 5, 4), rand(g, 5, 4)
    x[4] *= 1e-6  # a row where eps matters
    close(R.l2_normalize_bwd(x, d), vjp(R.l2_normalize, x, d))


def test_point_matching_gradient():
    """pm_loss_grad = autograd of gs * sum pm_loss, zero where est = obs (MXNet's abs backward: sign(0) = 0)"""
    g = torch.Generator().manual_seed(4)
    est, obs = rand(g, 2, 3, 7), rand(g, 2, 3, 7)
    obs[:, :, 2] = est[:, :, 2]
    pw = (rand(g, 2, 3, 7) > 0).double()
    gs, norm = 0.375 / 1536, 0.25
    ref = R.pm_loss_grad(est, obs, pw, norm, gs)
    close(ref, vjp(lambda t: gs * R.pm_loss(t, obs, pw, norm).sum(), est, torch.tensor(1.0, dtype=torch.float64)))
    assert not ref[:, :, 2].any()


@pytest.mark.parametrize("rot_coord", ["MODEL", "CAMERA", "CAMERA_NEW"])
def test_transform3d_matches_oracle(rot_coord):
    """the float64 Transform3D forward / hand-written backward against the oracle's restatement of transform3d.py"""
    rng = np.random.default_rng(5)
    B, N = 3, 11
    P = rng.normal(size=(B, 3, N)).astype(np.float32) * 0.1
    q = rng.normal(size=(B, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[2] *= 1.5  # outside both thresholds: identity rotation, zero rotation gradient
    q = q.astype(np.float32)
    t = (rng.normal(size=(B, 3)) * 0.05).astype(np.float32)
    qs = rng.normal(size=(B, 4))
    ps = np.zeros((B, 3, 4), np.float32)
    ps[:, :, :3] = R.quat2mat_t3d(torch.from_numpy(qs / np.linalg.norm(qs, axis=1, keepdims=True))).numpy()
    ps[:, :, 3] = [[0.05 * b, -0.03, 0.9 + 0.1 * b] for b in range(B)]
    D = rng.normal(size=(B, 3, N)).astype(np.float32)
    Tm, Ts = (0.0625, -0.125, 0.03125), (0.5, 2.0, 0.75)
    T = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    ref, S = R.transform3d_fwd(T(P), T(q), T(t), T(ps), Tm, Ts, rot_coord)
    o = O.transform3d_forward(P, q, t, ps, Tm, Ts, rot_coord)
    assert (ref - T(o)).abs().max() <= 1e-5 * float(S.max())
    (rg, _), (tg, _) = R.transform3d_bwd(T(D), T(P), T(q), T(t), T(ps), Tm, Ts, rot_coord)
    org, otg = O.transform3d_backward(D, P, q, t, ps, Tm, Ts, rot_coord)
    np.testing.assert_allclose(rg.numpy(), org, rtol=1e-5, atol=1e-5 * np.abs(org).max())
    np.testing.assert_allclose(tg.numpy(), otg, rtol=1e-5, atol=1e-5 * np.abs(otg).max())
    assert not rg[2].any()
