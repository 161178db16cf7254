"""Teacher-forced float64 references for single device kernels (shared by the per-kernel GPU tests).

A kernel is checked against the same operation computed in float64 (torch / cuDNN on the GPU, not this project's kernels)
from exactly the operands the device stored: the bf16 / fp16 activation buffers it read, the operand packs as the
repack rounds them from the fp32 master, and the stored activation's sign as the LeakyReLU mask.  What remains between
the two is the fp32 accumulation order and the output rounding, which one element-wise bound covers:

    |y_dev - y_ref| <= rho * |y_ref| + kappa * 2^-24 * S

S is the same operation applied to |operands| (+ |addend|), rho the output storage's unit roundoff (bf16 2^-8, fp16 2^-11,
a bf16x3 hi / lo pair 2^-15, fp32 0) and kappa a constant per kernel family.  A buffer that is rounded more than once
(an in-place read-add-store) adds rho times the magnitude of each earlier stored value (`slack`)."""
import numpy as np
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

from oracle.train_oracle import DECONV_CROP, DECONV_STRIDE

U = 2.0 ** -24
RHO = {"fp32": 0.0, "bf16": 2.0 ** -8, "fp16": 2.0 ** -11, "bf16x3": 2.0 ** -15}
OBSERVED = {}  # kernel family -> largest kappa an element needed, max over every check of the session


def gpu(a):
    return torch.as_tensor(np.ascontiguousarray(a)).to("cuda", torch.float64)


def interior(buf, geo, B, c0=0, c1=None):
    """[B, C, H, W] float64 of the valid region of a bordered NHWC buffer [>=B, Hp, Wp, C]; geo = (py, px, H, W)"""
    if buf is None:
        return None
    py, px, H, W = geo
    return gpu(buf[:B, py:py + H, px:px + W, c0:c1]).permute(0, 3, 1, 2)


def border_is_zero(buf, geo, B):
    """every element of the first B images outside the H x W interior (all four sides, full depth) is zero"""
    py, px, H, W = geo
    b = buf[:B].copy()
    b[:, py:py + H, px:px + W] = 0
    return not b.any()


def s2d_decode(buf):
    """conv1's space-to-depth strip buffer (read as [B, rows, cols, 4 L]) -> the bordered image canvas [B, L, 2 rows, 2 cols].
    A buffer row is C / 8 planes of cols x 8 lanes; plane j holds space-to-depth channels 8j ... 8j + 7, and channel
    (ph*2 + pw) * L + c of row r, column q is channel c of image pixel (2r + ph, 2q + pw)."""
    B, rows, cols, C = buf.shape
    L = C // 4
    s2d = buf.reshape(B, rows, C // 8, cols, 8).transpose(0, 1, 3, 2, 4).reshape(B, rows, cols, 2, 2, L)
    return s2d.transpose(0, 5, 1, 3, 2, 4).reshape(B, L, 2 * rows, 2 * cols)


def operand(w, prec):
    """An fp32 master tensor as the device packs it: (hi, lo) float64; lo is None unless prec is bf16x3.
    bf16 RN: hi = bf16(w), lo = bf16(w - hi); fp16: hi = fp16(w)."""
    w32 = torch.as_tensor(np.ascontiguousarray(w, np.float32)).cuda()
    if prec == "fp16":
        return w32.half().double(), None
    hi = w32.bfloat16().float()
    return hi.double(), ((w32 - hi).bfloat16().double() if prec == "bf16x3" else None)


def fused(p):
    """a (hi, lo) pair as one fp32 operand (hi + lo is exact in fp32): for kernels that add the halves before multiplying"""
    return (p[0] if p[1] is None else p[0] + p[1]), None


def products(op, a, b):
    """op(a, b) of two (hi, lo) operands as the tensor-core passes form it: hi*hi, plus lo*hi and hi*lo when a lo half
    exists (bf16x3; the lo*lo term is not computed by the device and not by the reference).  Returns (ref, S), S being
    the same passes over |a| and |b|."""
    terms = [(a[0], b[0])]
    if a[1] is not None:
        terms.append((a[1], b[0]))
    if b[1] is not None:
        terms.append((a[0], b[1]))
    ref = sum(op(x, y) for x, y in terms)
    S = sum(op(x.abs(), y.abs()) for x, y in terms)
    return ref, S


def lrelu_mask(act_hi, slope=0.1):
    """the data-gradient epilogue's rule: !(a > 0) takes the slope, so a stored 0 does (bf16x3: the hi half decides)"""
    return torch.where(act_hi > 0, torch.ones_like(act_hi), torch.full_like(act_hi, slope))


# ------------------------------------------------------------------------------------- the operations
def conv_wgrad(x, gz, k, stride, pad):
    """dW (Cout, Cin, k, k) of a convolution from its input x [B, Cin, H, W] and pre-activation gradient gz [B, Cout, Ho, Wo]"""
    return products(lambda a, g: conv2d_weight(a, (g.shape[1], a.shape[1], k, k), g, stride=stride, padding=pad), x, gz)


def conv_dgrad(gz, w, in_shape, stride, pad):
    """dX [B, Cin, H, W] of a convolution from gz [B, Cout, Ho, Wo] and W (Cout, Cin, k, k)"""
    return products(lambda g, ww: conv2d_input(in_shape, ww, g, stride=stride, padding=pad), gz, w)


def deconv_canvas(d, Hi, Wi):
    """a cropped deconvolution output gradient [B, C, Ho, Wo] on the uncropped (2 Hi + 2) x (2 Wi + 2) canvas"""
    B, C, Ho, Wo = d.shape
    s, c = DECONV_STRIDE, DECONV_CROP
    full = d.new_zeros(B, C, s * Hi + 2, s * Wi + 2)
    full[:, :, c:c + Ho, c:c + Wo] = d
    return full


def deconv_fwd(x, w, Ho, Wo):
    """the cropped stride-2 deconvolution of x [B, Cin, Hi, Wi] with W (Cin, Cout, 4, 4), no bias"""
    c = DECONV_CROP
    return products(lambda a, ww: F.conv_transpose2d(a, ww, stride=DECONV_STRIDE)[:, :, c:c + Ho, c:c + Wo], x, w)


def deconv_wgrad(x, d):
    """dW (Cin, Cout, 4, 4) of a cropped deconvolution from its input x [B, Cin, Hi, Wi] and output gradient d"""
    Hi, Wi = x[0].shape[2:]
    return products(lambda a, g: conv2d_weight(deconv_canvas(g, Hi, Wi), (a.shape[1], g.shape[1], 4, 4), a,
                                               stride=DECONV_STRIDE), x, d)


def deconv_dgrad(d, w, Hi, Wi):
    """dX [B, Cin, Hi, Wi] of a cropped deconvolution from its output gradient d and W (Cin, Cout, 4, 4)"""
    return products(lambda g, ww: F.conv2d(deconv_canvas(g, Hi, Wi), ww, stride=DECONV_STRIDE), d, w)


# ------------------------------------------------------------------------------------- the bound
def at_pixel(idx):
    b, c, y, x = idx
    return "(image %d, y %d, x %d, channel %d)" % (b, y, x, c)


def wgrad_tiles(k, bn):
    """location of a weight-gradient entry (d0, d1, kh, kw) and the conv_wgrad_kernel tile that computed it: tap = kh*k + kw,
    M tile = d0 // 128, N tile = d1 // bn (make_wgrad puts d0 -- Cout of a convolution, Cin of a deconvolution -- on M).
    No K slice is named: every slice of the batch's pixels adds into every entry, so a wrong slice shows in every tile."""
    def where(idx):
        d0, d1, kh, kw = idx
        return "(%d, %d, %d, %d) = tap %d, M tile %d, N tile %d" % (d0, d1, kh, kw, kh * k + kw, d0 // 128, d1 // bn)
    return where


def wgrad_bn(n):
    """make_wgrad's N tile for an N-side width of n"""
    return 256 if n >= 256 else (128 if n >= 128 else (64 if n >= 64 else 32))


def check(family, name, dev, ref, S, rho, kappa, where=lambda idx: str(idx), slack=None):
    """Asserts |dev - ref| <= rho |ref| + slack + kappa 2^-24 S element by element (no outlier allowance) and records in
    OBSERVED[family] the largest kappa an element needed.  dev, ref, S: float64 tensors of one shape."""
    dev = torch.as_tensor(dev).to(ref.device, torch.float64)
    assert dev.shape == ref.shape, (name, tuple(dev.shape), tuple(ref.shape))
    assert torch.isfinite(dev).all(), "%s: non-finite device values" % name
    err = (dev - ref).abs()
    allow = rho * ref.abs() + (0.0 if slack is None else slack)
    scale = U * S
    over = (err - allow).clamp_min(0)
    need = torch.where(over > 0, over / scale, torch.zeros_like(over))  # inf where S = 0 and dev is not exactly ref
    obs = need.max().item()
    OBSERVED[family] = max(OBSERVED.get(family, 0.0), obs)
    bad = need > kappa
    if bool(bad.any()):
        i = int(torch.argmax(need).item())
        idx = tuple(int(v) for v in np.unravel_index(i, tuple(dev.shape)))
        places = sorted({where(tuple(int(v) for v in j)).split(" = ")[-1] for j in bad.nonzero()[:4096].tolist()})
        raise AssertionError(
            "%s: %d of %d entries exceed rho|ref| + %g * 2^-24 S; worst at %s: dev %.9g ref %.9g S %.6g needs kappa %.4g%s"
            % (name, int(bad.sum()), dev.numel(), kappa, where(idx), dev.flatten()[i].item(), ref.flatten()[i].item(),
               S.flatten()[i].item(), obs, "; bad entries in: " + ", ".join(places[:12]) if len(places) > 1 else ""))
    return obs
