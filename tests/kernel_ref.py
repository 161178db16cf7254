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


# the heads' fixed bilinear upsampling (deepIM_flownet.py:184-199, 329-344): a Deconvolution k32 s16 with one group per
# channel, then Crop(offset (8, 8)) to the image size
UP_K, UP_STRIDE, UP_CROP = 32, 16, 8


def upsample_fwd(x, w, H, W):
    """the upsampled, cropped map [B, C, H, W] of x [B, C, h, w]; w (C, 1, 32, 32).  Device-agnostic, like the other
    references below (float64 in, float64 out)."""
    c = UP_CROP
    return F.conv_transpose2d(x, w, stride=UP_STRIDE, groups=x.shape[1])[:, :, c:c + H, c:c + W]


def upsample_bwd(d, w, h, wd):
    """the adjoint of upsample_fwd: the gradient [B, C, h, wd] of the low-resolution map from the gradient d [B, C, H, W]
    of the cropped output (d placed on the uncropped canvas, then the stride-16 convolution with the same kernel)"""
    B, C, H, W = d.shape
    c = UP_CROP
    canvas = d.new_zeros(B, C, UP_STRIDE * (h - 1) + UP_K, UP_STRIDE * (wd - 1) + UP_K)
    canvas[:, :, c:c + H, c:c + W] = d
    return F.conv2d(canvas, w, stride=UP_STRIDE, groups=C)


L2_EPS = 1e-10  # L2Normalization(mode=instance): x / sqrt(sum x^2 + eps)


def l2_normalize(x):
    """L2Normalization of the rotation head, rows of x [B, 4]"""
    return x / torch.sqrt((x * x).sum(1, keepdim=True) + L2_EPS)


def l2_normalize_bwd(x, g):
    """its backward: d x from the output gradient g, (g - y (y . g)) / n with y = x / n, n = sqrt(sum x^2 + eps)"""
    n = torch.sqrt((x * x).sum(1, keepdim=True) + L2_EPS)
    y = x / n
    return (g - y * (y * g).sum(1, keepdim=True)) / n


def pm_loss(est, obs, pw, norm):
    """the L1 point-matching loss per element (deepIM_flownet.py:290-296): pw |(est - obs) / norm|"""
    return pw * ((est - obs) / norm).abs()


def pm_loss_grad(est, obs, pw, norm, gs):
    """its gradient under MakeLoss(grad_scale = gs): gs pw sign(d) / norm, sign(0) = 0 as MXNet's abs backward"""
    return gs * pw * torch.sign((est - obs) / norm) / norm


def quat2mat_t3d(q):
    """Transform3D's quat2mat_forward (transform3d.py:185-212) of q [B, 4] -> [B, 3, 3]: the identity where
    |Nq - 1| >= 1e-2"""
    w, x, y, z = q.unbind(1)
    Nq = (q * q).sum(1)
    s = 2.0 / Nq
    X, Y, Z = x * s, y * s, z * s
    M = torch.stack([1 - (y * Y + z * Z), x * Y - w * Z, x * Z + w * Y,
                     x * Y + w * Z, 1 - (x * X + z * Z), y * Z - w * X,
                     x * Z - w * Y, y * Z + w * X, 1 - (x * X + y * Y)], 1).reshape(-1, 3, 3)
    eye = torch.eye(3, dtype=q.dtype, device=q.device).expand_as(M)
    return torch.where(((Nq - 1).abs() < 1e-2)[:, None, None], M, eye)


def _t3d_common(t, pose_src, Tm, Ts):
    """T_transform (rot_coord model / camera): d = t Ts + Tm, z2 = src_z / exp(d_z), a_k = d_k + src_k / src_z, and
    the error scales of z2 (relative, in units of 2^-24: exp, the division and d_z's own rounding) and of a_k"""
    Tm, Ts = (torch.as_tensor(v, dtype=t.dtype, device=t.device) for v in (Tm, Ts))
    src = pose_src[:, :, 3]
    d = t * Ts + Tm
    z2 = src[:, 2] / torch.exp(d[:, 2])
    a = d[:, :2] + src[:, :2] / src[:, 2:3]
    e2 = 3 + (t[:, 2] * Ts[2]).abs() + Tm[2].abs()
    Sa = (t[:, :2] * Ts[:2]).abs() + Tm[:2].abs() + (src[:, :2] / src[:, 2:3]).abs()
    return Ts, z2, a, e2, Sa


def _t3d_camera_new(t, pose_src, Tm, Ts):
    """T_transform for rot_coord camera_new: (x, y) = src_z d + src_(x, y), and the scale of their fp32 evaluation"""
    Tm, Ts = (torch.as_tensor(v, dtype=t.dtype, device=t.device) for v in (Tm, Ts))
    src = pose_src[:, :, 3]
    d = t[:, :2] * Ts[:2] + Tm[:2]
    Sd = (t[:, :2] * Ts[:2]).abs() + Tm[:2].abs()
    return src[:, 2:3] * d + src[:, :2], src[:, 2:3].abs() * Sd + src[:, :2].abs()


def transform3d_fwd(P, q, t, pose_src, Tm, Ts, rot_coord):
    """Transform3D forward (transform3d.py:34-97; rot_coord 'MODEL', 'CAMERA' or 'CAMERA_NEW'): points P [B, 3, N] under the
    rotation q [B, 4] and the translation t [B, 3] relative to pose_src [B, 3, 4] -> (ref, S), S bounding the fp32
    evaluation"""
    Rd, Rs = quat2mat_t3d(q), pose_src[:, :, :3]
    model = rot_coord.lower() == "model"
    Rt, SRt = (Rs @ Rd, Rs.abs() @ Rd.abs()) if model else (Rd @ Rs, Rd.abs() @ Rs.abs())
    _, z2, a, e2, Sa = _t3d_common(t, pose_src, Tm, Ts)
    if rot_coord.lower() == "camera_new":
        xy, Sxy = _t3d_camera_new(t, pose_src, Tm, Ts)
        Tt = torch.cat([xy, z2[:, None]], 1)
        STt = torch.cat([Sxy, z2.abs()[:, None] * e2[:, None]], 1)
    else:
        Tt = torch.cat([z2[:, None] * a, z2[:, None]], 1)
        STt = z2.abs()[:, None] * torch.cat([e2[:, None] * a.abs() + Sa, e2[:, None]], 1)
    return Rt @ P + Tt[:, :, None], SRt @ P.abs() + STt[:, :, None]


def _quat2mat_bwd_coef(qn):
    """[B, 4, 9]: (w', x', y', z') of quat2mat_backward (transform3d.py:214-275) as a linear map of the row-major 3x3
    matrix gradient, for the normalised quaternion qn"""
    w, x, y, z = qn.unbind(1)
    o = torch.zeros_like(w)
    rows = [[o, -z, y, z, o, -x, -y, x, o],
            [o, y, z, y, -2 * x, -w, z, w, -2 * x],
            [-2 * y, x, w, x, o, z, -w, z, -2 * y],
            [-2 * z, -w, x, w, -2 * z, y, x, y, o]]
    return 2 * torch.stack([torch.stack(r, 1) for r in rows], 1)


def transform3d_bwd(D, P, q, t, pose_src, Tm, Ts, rot_coord):
    """Transform3D's hand-written backward (transform3d.py:99-281) of the output gradient D [B, 3, N] ->
    ((d rotation [B, 4], S), (d translation [B, 3], S)); the rotation gradient is zero where |Nq - 1| >= 1e-4"""
    Ts, z2, a, e2, Sa = _t3d_common(t, pose_src, Tm, Ts)
    Dt, SDt = D.sum(2), D.abs().sum(2)
    share = -Ts[2] * z2
    if rot_coord.lower() == "camera_new":  # x, y no longer depend on d_z: d_x, d_y scale by src_z
        sz = pose_src[:, 2, 3]
        tg = torch.stack([Dt[:, 0] * Ts[0] * sz, Dt[:, 1] * Ts[1] * sz, Dt[:, 2] * share], 1)
        Stg = torch.stack([SDt[:, 0] * (Ts[0] * sz).abs(), SDt[:, 1] * (Ts[1] * sz).abs(), e2 * SDt[:, 2] * share.abs()], 1)
    else:
        tg = torch.stack([Dt[:, 0] * Ts[0] * z2, Dt[:, 1] * Ts[1] * z2,
                          Dt[:, 0] * share * a[:, 0] + Dt[:, 1] * share * a[:, 1] + Dt[:, 2] * share], 1)
        Stg = e2[:, None] * torch.stack([SDt[:, 0] * (Ts[0] * z2).abs(), SDt[:, 1] * (Ts[1] * z2).abs(),
                                         share.abs() * (SDt[:, 0] * Sa[:, 0] + SDt[:, 1] * Sa[:, 1] + SDt[:, 2])], 1)
    RtD, SRtD = D @ P.transpose(1, 2), D.abs() @ P.abs().transpose(1, 2)
    Rs = pose_src[:, :, :3]
    if rot_coord.lower() == "model":  # camera and camera_new share R_delta R_src
        Dm, SDm = Rs.transpose(1, 2) @ RtD, Rs.abs().transpose(1, 2) @ SRtD
    else:
        Dm, SDm = RtD @ Rs.transpose(1, 2), SRtD @ Rs.abs().transpose(1, 2)
    Nq = (q * q).sum(1)
    Ns = torch.sqrt(Nq)[:, None]
    C = _quat2mat_bwd_coef(q / Ns)
    dq, Sdq = (C @ Dm.reshape(-1, 9, 1))[..., 0], (C.abs() @ SDm.reshape(-1, 9, 1))[..., 0]
    sh = Ns ** 3 * (q * dq).sum(1, keepdim=True)
    rg = Ns * dq - q * sh
    Srg = Ns * Sdq + q.abs() * Ns ** 3 * (q.abs() * Sdq).sum(1, keepdim=True)
    ok = ((Nq - 1).abs() < 1e-4)[:, None]
    return (torch.where(ok, rg, torch.zeros_like(rg)), torch.where(ok, Srg, torch.zeros_like(Srg))), (tg, Stg)


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


# ------------------------------------------------------------------------------------- inference network
# kappa per inference kernel family: 4 x the largest (|err| - rho |ref|) / (2^-24 S) observed over every case of
# tests/test_gpu_conv1.py, rounded up to two digits and at least 1 ("obs"; measured on an H100 80GB HBM3 at a 400 W power
# limit).  The same bounds hold at every SM count (tests/test_gpu_schedule.py): each output's K order is fixed by the kernel.
KAPPA_INFER = {
    "conv1": 24,       # obs 5.9     conv1_kernel
    "tower": 96,       # obs 24.0    conv_igemm_persistent_kernel, conv2 ... conv6_1
    "fc6_head": 1,     # obs 0.0042  fc6_mma_kernel + head_kernel (fc7, rot, trans in fp32); S carried through fc7 and the heads
}


def fc6_nhwc(a):
    """fc6 (256, c*80 + hw) in MXNet order -> (256, hw*1024 + c), the NHWC order of act[10] the kernels read"""
    return np.ascontiguousarray(np.asarray(a).reshape(256, 1024, 80).transpose(0, 2, 1)).reshape(256, 81920)


def check_fc6_heads(weights, mode, B, act10, rot, trans, tag="", zoom_factor=None):
    """rot / trans of net_forward against float64 fc6 -> fc7 -> heads from the stored act[10] = (hi, lo) float32 numpy
    [>= B, 8, 10, 1024]: fc6's operands as its 16-bit pack rounds them, fc7 / rot / trans from the fp32 weights.  The error
    scale S of fc6 is carried through fc7 and the heads by their absolute weights (LeakyReLU moves no difference up).
    zoom_factor [>= B, 4] (the refinement loop's se3): trans x and y are the head's outputs times wx in float32
    (invZoomTrans), so ref and S of those two are scaled by wx and the product's rounding, 2^-24 relative, is allowed."""
    lrelu = lambda v: F.leaky_relu(v, 0.1)
    W6 = operand(fc6_nhwc(weights["fc6_weight"]), mode)
    wb = {k: gpu(weights[k]) for k in ("fc6_bias", "fc7_weight", "fc7_bias", "rot_weight", "rot_bias", "trans_weight",
                                       "trans_bias")}
    hi, lo = act10
    a = gpu(hi[:B]).reshape(B, 81920), (None if lo is None else gpu(lo[:B]).reshape(B, 81920))
    z6, S6 = products(lambda x, w: x @ w.T, a, W6)
    h6, E6 = lrelu(z6 + wb["fc6_bias"]), S6 + wb["fc6_bias"].abs()
    w7 = wb["fc7_weight"]
    h7 = lrelu(h6 @ w7.T + wb["fc7_bias"])
    E7 = E6 @ w7.abs().T + h6.abs() @ w7.abs().T + wb["fc7_bias"].abs()
    for name, dev in (("rot", rot), ("trans", trans)):
        w, b = wb[name + "_weight"], wb[name + "_bias"]
        ref, S, slack = h7 @ w.T + b, E7 @ w.abs().T + h7.abs() @ w.abs().T + b.abs(), None
        if name == "trans" and zoom_factor is not None:
            s = torch.ones_like(ref)
            s[:, :2] = gpu(np.asarray(zoom_factor)[:B, :1])
            ref, S = ref * s, S * s.abs()
            slack = torch.zeros_like(ref)
            slack[:, :2] = U * ref[:, :2].abs()
        check("fc6_head", "%s (%s, B=%d%s)" % (name, mode, B, tag), dev, ref, S, 0.0, KAPPA_INFER["fc6_head"],
              lambda idx: "(image %d, output %d)" % idx, slack=slack)


def check_conv_layer(weights, mode, layer, B, x, out, geo, tag=""):
    """encoder layer `layer` (ENC order) against float64 from its stored input x = (hi, lo) float64 [B, Cin, H, W] (the
    interior; conv1: the decoded space-to-depth canvas, pad included) and its stored output buffer out = (hi, lo) float32
    numpy [>= B, rows, cols, C] with interior geo = (py, px, H, W).  Returns the largest kappa an element needed."""
    from oracle.train_oracle import ENC
    name, s, p = ENC[layer]
    w = operand(weights[name + "_weight"], mode)
    b = gpu(weights[name + "_bias"])[None, :, None, None]
    ref, S = products(lambda a, ww: F.conv2d(a, ww, stride=s, padding=p), x, w)
    dev = fused((interior(out[0], geo, B), interior(out[1], geo, B)))[0]
    fam = "conv1" if layer == 0 else "tower"
    return check(fam, "%s (%s, B=%d%s)" % (name, mode, B, tag), dev, F.leaky_relu(ref + b, 0.1), S + b.abs(), RHO[mode],
                 KAPPA_INFER[fam], at_pixel)


# ------------------------------------------------------------------------------------- training step
# kappa of the weight-gradient families (conv_wgrad_kernel / conv1_wgrad_kernel + wgrad_reduce), shared by
# tests/test_gpu_train_kernels.py and tests/test_gpu_schedule.py; see DESIGN.md section 6 for what each K-slice count needed
KAPPA_WGRAD = {
    "wgrad": 1300,          # obs 302.3  conv_wgrad_kernel + wgrad_reduce (WG_CONV, WG_DECONV)
    "conv1_wgrad": 190,     # obs 45.8   conv1_wgrad_kernel + WG_CONV1_ROW; RGB-D: conv_wgrad_kernel + WG_CONV1_RGBD
}


# the weight gradients whose fp32 reduction order follows the SM count (make_wgrad / run_wgrad_conv1 K slices)
SM_DEPENDENT_GRADS = ("flow_conv1_weight", "conv2_weight", "conv3_weight", "conv3_1_weight", "conv4_weight", "conv4_1_weight",
                      "conv5_weight", "conv5_1_weight", "conv6_weight", "conv6_1_weight", "deconv5_weight", "deconv4_weight")


def wgrad_slices(ctx, B):
    """{gradient: (K slices, pixel blocks per slice, pixel blocks)} of a B-image training step at the context's current SM
    count and precision (dim_train_debug_wgrad_slices; the order of SM_DEPENDENT_GRADS)"""
    import ctypes as C
    from deepim_b200 import _capi as capi
    out = (C.c_int32 * 36)()
    capi.check(capi.lib.dim_train_debug_wgrad_slices(ctx._h, B, out))
    return {n: tuple(out[3 * g:3 * g + 3]) for g, n in enumerate(SM_DEPENDENT_GRADS)}


def wgrad_slice_growth(slices, calibrated):
    """{gradient: how much longer the K range one fp32 accumulator sums is under `slices` than under `calibrated` (the
    schedule KAPPA_WGRAD was calibrated at: the device's SM count)}, at least 1.  The tensor cores' fp32 accumulation does
    not round to nearest, so its error grows with the number of K steps one accumulator takes, linearly as measured
    (DESIGN.md section 6); a weight gradient's kappa is scaled by this factor."""
    return {n: max(1.0, slices[n][1] / calibrated[n][1]) for n in slices}


class Run:
    """the device state of a training context after one forward_backward of B images; buffers are read lazily and cached"""

    def __init__(self, net, prec, B, ctx, tr):
        from oracle.train_oracle import ENC
        self.net, self.prec, self.B, self.ctx, self.tr = net, prec, B, ctx, tr
        self.s3 = prec == "bf16x3"
        self.grads = tr.grads_dict()
        self.params = tr.get_params()
        self.sizes = [(ctx.H, ctx.W)]  # sizes[i]: the interior of act[i] (the input of encoder layer i)
        for name, s, p in ENC:
            k = self.params[name + "_weight"].shape[-1]
            h, w = self.sizes[-1]
            self.sizes.append(((h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1))
        self._c = {}

    def _cached(self, key, f):
        if key not in self._c:
            self._c[key] = f()
        return self._c[key]

    def act_raw(self, i, lo=False):
        """act[i] as stored ([max_batch, rows, cols, C] float32 incl. border) and its interior (py, px, H, W)"""
        def f():
            buf, g = self.ctx.debug_activation(i, self.ctx.max_batch, lo=lo)
            return buf, (g[3], g[4]) + self.sizes[i]
        return self._cached(("act", i, lo), f)

    def act(self, i):
        """(hi, lo) interior of act[i] as float64 [B, C, H, W]; act[0] decoded from conv1's space-to-depth buffer"""
        def f():
            out = []
            for lo in ((False, True) if self.s3 else (False,)):
                buf, (py, px, H, W) = self.act_raw(i, lo)
                if i == 0:
                    out.append(gpu(s2d_decode(buf[:self.B])[:, :, py:py + H, px:px + W]))
                else:
                    out.append(interior(buf, (py, px, H, W), self.B))
            return out[0], (out[1] if self.s3 else None)
        return self._cached(("actp", i), f)

    def tbuf(self, tid, lo=False):
        return self._cached(("t", tid, lo), lambda: self.tr.debug_tensor(tid + (100 if lo else 0)))

    def pair(self, tid, c0=0, c1=None):
        """(hi, lo) interior of a bf16 training buffer as float64 [B, C, H, W]"""
        hi, geo = self.tbuf(tid)
        lo = self.tbuf(tid, True)[0] if self.s3 else None
        return interior(hi, geo, self.B, c0, c1), interior(lo, geo, self.B, c0, c1)

    def fp32(self, tid):
        """an fp32 training map [B, h, w, c] as float64 [B, c, h, w] (dh6 / h6: [B, 256])"""
        a = gpu(self.tbuf(tid)[:self.B])
        return a if a.dim() == 2 else a.permute(0, 3, 1, 2)

    def w(self, name):
        return operand(self.params[name], self.prec)

    def w_fc6(self):
        """fc6's operand pack, (256, hw*1024 + c): the NHWC order of ReLU10 the kernels read"""
        return operand(fc6_nhwc(self.params["fc6_weight"]), self.prec)

    def w32(self, name):
        return gpu(self.params[name]), None

    @property
    def rho(self):
        return RHO[self.prec]


def check_conv_wgrad(run, i, tag="", growth=1.0):
    """conv_wgrad_kernel + wgrad_reduce (WG_CONV) of encoder layer i = 1 ... 9: dW = conv2d_weight(act[i], gz[i])"""
    from oracle.train_oracle import ENC
    name, s, p = ENC[i]
    k = run.params[name + "_weight"].shape[-1]
    ref, S = conv_wgrad(run.act(i), run.pair(20 + i), k, s, p)
    return check("wgrad", "%s_weight (B=%d, %s%s)" % (name, run.B, run.prec, tag), run.grads[name + "_weight"], ref, S, 0.0,
                 KAPPA_WGRAD["wgrad"] * growth, wgrad_tiles(k, wgrad_bn(ref.shape[1])))


def check_conv1_wgrad(run, tag="", growth=1.0):
    """flow_conv1's weight gradient from the decoded space-to-depth input act[0] (stride 2, pad 3) and gz[0]: the
    row-GEMM kernel with WG_CONV1_ROW (D1 = 8, or 6 for the image-only network) or, RGB-D, the generic kernel with
    WG_CONV1_RGBD (D1 = 10).  The lanes past D1 hold exact zeros in the input and are absent from the gradient."""
    from oracle.train_oracle import ENC
    name, s, p = ENC[0]
    x = run.act(0)
    D1 = {"nomask": 6, "rgbd": 10}.get(run.net, 8)
    dev = run.grads[name + "_weight"]
    assert dev.shape == (64, D1, 7, 7)
    assert x[0].shape[1] == (16 if run.net == "rgbd" else 8)
    for half in x:
        assert half is None or not half[:, D1:].any(), "conv1 input lanes %d+ are not zero" % D1
    ref, S = conv_wgrad(x, run.pair(20), 7, s, p)

    def where(idx):
        co, ci, kh, kw = idx
        if run.net == "rgbd":
            return "(%d, %d, %d, %d) = tap %d" % (co, ci, kh, kw, (kh // 2) * 4 + kw // 2)
        return "(%d, %d, %d, %d) = filter row %d, M row %d" % (co, ci, kh, kw, kh // 2, (kw // 2) * 32 + (kh % 2) * 16 + (kw % 2) * 8 + ci)
    return check("conv1_wgrad", "flow_conv1_weight (%s, B=%d, %s%s)" % (run.net, run.B, run.prec, tag), dev, ref[:, :D1], S[:, :D1],
                 0.0, KAPPA_WGRAD["conv1_wgrad"] * growth, where)


def check_deconv_wgrad(run, name, tag="", growth=1.0):
    """conv_wgrad_kernel + WG_DECONV: deconv5 from act10b and the final dcat2[512:1024], deconv4 from cat2[:1026] and the
    final dcat3[512:768]"""
    x, d = {"deconv5_weight": (run.pair(15, 0, 1024), run.pair(12, 512, 1024)),
            "deconv4_weight": (run.pair(10, 0, 1026), run.pair(13, 512, 768))}[name]
    ref, S = deconv_wgrad(x, d)
    return check("wgrad", "%s (B=%d, %s%s)" % (name, run.B, run.prec, tag), run.grads[name], ref, S, 0.0, KAPPA_WGRAD["wgrad"] * growth,
                 wgrad_tiles(4, wgrad_bn(ref.shape[1])))
