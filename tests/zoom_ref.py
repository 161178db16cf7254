"""Float64 reference of the zoom stage (TEST INFRASTRUCTURE): boxes, zoom factor, the bilinear zoom in every gather mode,
the inverse-zoom affine, ZoomTrans and conv1's input channels.

An independent definition of what `zoom_gather_kernel`, `mask_bbox_kernel`, `obs_colour_box_kernel`, `zoom_factor_kernel`,
`box_mask_kernel`, `zoom_trans_kernel` and `zoom_fused_nhwc8_kernel` compute (and the oracle's `orc_zoom_plane`,
`orc_zoom_factor`, `orc_inv_zoom_affine`, `orc_box_mask`, `orc_zoom_trans`): float64 numpy, with no oracle import and
no float32 operation sequence.  Semantics, with the file each comes from (deepim/operator_py/ unless a path is given):

- Sampler (mx.sym.GridGenerator 'affine' + mx.sym.BilinearSampler, as zoom_mask.py:96-98 and every other op calls them;
  MXNet documents both as align_corners sampling): output pixel (i, j) of an H x W plane samples the source point
  x = ((wx (-1 + 2 j / (W - 1)) + tx) + 1) (W - 1) / 2, y likewise with (wy, ty, H, i).  The value is the bilinear
  interpolation on the integer pixel grid of the image extended by zeros: a tap outside [0, W-1] x [0, H-1] reads 0.  The
  affine is the float32 zoom factor (mx.nd.array of Python floats is float32), promoted exactly.
- Modes of zoom_gather_kernel (MODE 0 ... 6), defined from the operators:
  0 plain sample (zoom_depth.py:34-42);  1 round half away from zero, mx.nd.round (zoom_mask.py:105-107);
  2 binarise at 0.2 then round (zoom_mask_with_factor.py:36-62);  3 (img + mean) sampled, minus mean: the padding zero
  lives in the image-plus-mean domain, so an out-of-frame sample is -mean (zoom_image_with_factor.py:44-62);
  4 sample * wx (zoom_flow.py:55-64, b_inv_zoom);  5 round(sample - 0.45) (zoom_flow.py:66-71);  6 sample / wx
  (zoom_flow.py:55-64).  wx is the forward zoom factor's first entry in both flow modes.
- Thresholds against a float32 array compare in float32 (numpy 1.x value-based casting of a Python scalar, and MXNet's
  scalar ops in the array's dtype): binarise is `v > float32(0.2)` (zoom_mask.py:39-41), the mask box
  `sum_c(mask) > float32(0.3)` (zoom_mask.py:36-43), the image box `sum_c(image + mean) > float32(0.01)`
  (zoom_image.py:33-37), the flow-weight offset float32(0.45).
- Inverse-zoom affine (zoom_flow.py:35-44, zoom_mask_with_factor.py:43-52): float32 factors with Python numbers, so float64
  under numpy 1.x, then float32 in mx.nd.array.
- ZoomTrans (zoom_trans.py:22-74): float32 scalars times / over float32 wx, stored float32; backward with b_zoom_grad the
  same scaling, without it the identity.
- Boxes: inclusive min / max of the valid columns and rows (zoom_mask.py:51-58).  The observed rectangle of the fused
  loop is end-exclusive on the rendered box: mask_observed[y0:y1, x0:x1] = 1 (lib/pair_matching/data_pair.py:93-105).
- Zoom factor (zoom_mask.py:59-103; zoom_image.py:41-86 is the same code): c = K t, zoom centre c_x = c0 / c2, c_y = c1 / c2
  (or the observed box's centre when the rendered box is empty, l.70-77), crop = max(0.75 right, 0.75 left, up, down) 1.4 2,
  wx = wy = crop / H, tx = c_x / W 2 - 1, ty = c_y / H 2 - 1.  The reference raises for an empty observed box; the device
  stores (1, 1, 0, 0) and sets status bit 0.
- conv1's input (deepIM_flownet.py:33-62): images / 255, then depths / 255 (INPUT_DEPTH), then the masks (INPUT_MASK).

Tolerance rule.  u = 2^-24 is float32's unit roundoff.  Every bound below is a first-order sum of one u per float32
operation on the magnitude it rounds, and the sum is multiplied by 1 + 16 u, which covers the second-order terms of the
at most eight roundings involved (gamma_n = n u / (1 - n u)).

- Coordinates.  The device evaluates x in float32 as step = fl(2 / (W - 1)), a = fl(j step), xt = fl(-1 + a),
  xs = fl(fl(wx xt) + tx), x = fl(fl(xs + 1) (W - 1)) / 2 (the halving is exact).  With A = 2j / (W - 1):
      d_xt = u (2 A + |xt|)                         step and product, then the sum
      d_xs = |wx| d_xt + u (|wx xt| + |xs|)
      d_x  = (W - 1) / 2 (d_xs + 2 u |xs + 1|)        the +1 and the product by W - 1
  `coord_bound(w, t, N)` returns d_x per output index (d_y likewise).  The tap weights are 1 - (x - floor x) and
  1 - that: the first rounds once at magnitude <= 1 (error <= u / 2 = 2^-25), the second is exact (Sterbenz), so the
  two weights are exact for a point moved by at most 2^-25; that is added to d_x.  The float64 evaluation of the
  exact x adds 2^-50 (|x| + N).  A known-answer test holds the float32 chain to d_x for every j of every affine used.
- Continuous outputs (modes 0, 3, 4, 6; float depth; conv1's image and depth channels).  The interpolant is continuous,
  so the device's value comes from some point of the box x +- d_x, y +- d_y.  On that box the interpolant is bilinear
  on each cell it meets, so its extremes lie among the box's corners and the points where the integer grid lines inside
  it cross the box edges (at most one line per axis while d < 1/2): `sample_interval` evaluates those nine points.
  Then the float32 arithmetic: the four weight products and the product-plus-three-FMA chain round five times at
  magnitude <= M = max |tap| over the taps the box touches: widen by 5 u M.  Mode 3 (and the fused loop's images)
  also rounds each tap's image + mean (u M, M over |image + mean|) and the final - mean (u |result|); modes 4 and 6
  scale the interval by wx (or 1 / wx) and round once more (u |result|).
- Discrete outputs (modes 1, 2, 5, box-mask lanes, box indices).  Where the interval of the value being rounded or
  compared does not contain the threshold (a half-integer; k + 0.95 before round(s - 0.45), with the subtraction's own
  rounding and float32(0.45)'s error added; the float32 threshold of a box), the device must equal the reference
  exactly.  Elsewhere the pixel is ambiguous and excluded, and every test asserts the excluded share.
- Zoom factor.  c = K t in float32 is three products and two sums: each component is within gamma_3 sum_j |K_ij t_j|
  of the float64 value; c_x is their float32 quotient (one more u).  The float64 factor is evaluated over the
  resulting interval of (c_x, c_y) (each of its terms is monotone or convex in one coordinate), and the stored float32
  must lie in that range widened by 1 ulp of float32.  The empty-render fallback has no float32 step and no widening
  beyond that ulp.
- 16-bit conv1 input.  conv1's channel value is the continuous interval / 255, plus the float32 division's rounding
  (u |q|).  fp16 and bf16: the stored value is the 16-bit rounding of a float32 value in that interval, and rounding is
  monotone, so it lies between the 16-bit roundings of the ends.  bf16x3: hi + lo lies in that interval widened by one
  ulp of lo (lo is the rounding of the exact float32 residual).
"""
import numpy as np

U = 2.0 ** -24
GAMMA = 1.0 + 16 * U  # second-order cover of a first-order bound
WEIGHT_SHIFT = 2.0 ** -25  # the rounding of 1 - frac, as a move of the sample point
F32 = np.float32
THR_BIN, THR_MASK, THR_IMG, FLOW_OFFSET = float(F32(0.2)), float(F32(0.3)), float(F32(0.01)), 0.45
MAX_AMBIGUOUS = 0.01  # share of pixels a test may exclude as ambiguous


# ------------------------------------------------------------------------------------------------------------ sampler
def grid(w, t, N):
    """the exact source coordinate of output indices 0 ... N-1 along one axis (GridGenerator affine, align_corners)"""
    o = np.arange(N, dtype=np.float64)
    return ((float(w) * (-1.0 + 2.0 * o / (N - 1)) + float(t)) + 1.0) * (N - 1) / 2.0


def coord_bound(w, t, N, dw=0.0, dt=0.0):
    """d_x of the module docstring: the float32 coordinate chain's error bound per output index, plus the weights' move;
    dw, dt: how far the affine itself may be from (w, t) (the inverse affine's float32 rounding)"""
    w, t = float(w), float(t)
    A = 2.0 * np.arange(N, dtype=np.float64) / (N - 1)
    xt = -1.0 + A
    xs = w * xt + t
    d_xt = U * (2.0 * A + np.abs(xt))
    d_xs = abs(w) * d_xt + U * (np.abs(w * xt) + np.abs(xs))
    d_x = (N - 1) / 2.0 * (d_xs + 2.0 * U * np.abs(xs + 1.0))
    d_x = d_x + (N - 1) / 2.0 * (dw * np.abs(xt) + dt)
    x = (xs + 1.0) * (N - 1) / 2.0
    return d_x * GAMMA + WEIGHT_SHIFT + 2.0 ** -50 * (np.abs(x) + N)


def _taps(img, X, Y):
    """the image extended by zeros at integer points (X, Y) (broadcast); clipping far indices keeps them out of frame"""
    H, W = img.shape
    Xi = np.clip(X, -2, W + 1).astype(np.int64)
    Yi = np.clip(Y, -2, H + 1).astype(np.int64)
    ok = (Xi >= 0) & (Xi < W) & (Yi >= 0) & (Yi < H)
    return np.where(ok, img[np.clip(Yi, 0, H - 1), np.clip(Xi, 0, W - 1)], 0.0)


def sample(img, X, Y):
    """the sampler at source points X [..., 1, W'] and Y [..., H', 1] (broadcast), float64"""
    img = np.asarray(img, np.float64)
    x0, y0 = np.floor(X), np.floor(Y)
    fx, fy = X - x0, Y - y0
    top = (1.0 - fx) * _taps(img, x0, y0) + fx * _taps(img, x0 + 1, y0)
    bot = (1.0 - fx) * _taps(img, x0, y0 + 1) + fx * _taps(img, x0 + 1, y0 + 1)
    return (1.0 - fy) * top + fy * bot


def zoom(img, affine):
    """the float64 sampler on the whole plane at the affine's exact grid"""
    H, W = img.shape
    wx, wy, tx, ty = [float(v) for v in affine]
    return sample(img, grid(wx, tx, W)[None, :], grid(wy, ty, H)[:, None])


def _axis_points(c, d):
    """the three points of one axis: both ends of c +- d and the integer inside (an end when there is none)"""
    assert (d < 0.5).all(), "coordinate bound reaches half a pixel: the nine-point rule needs d < 1/2"
    lo, hi = c - d, c + d
    k = np.floor(hi)
    mid = np.where(k > lo, k, lo)
    return np.stack([lo, mid, hi])


def sample_interval(img, affine, da=(0.0, 0.0, 0.0, 0.0)):
    """[lo, hi] of the float64 sampler over each output pixel's coordinate box (nine points), and M = max |tap| over the
    taps the box touches: the continuous interval before the float32 arithmetic's widening.  da: the affine's own
    uncertainty (inv_affine_f32)"""
    img = np.asarray(img, np.float64)
    H, W = img.shape
    wx, wy, tx, ty = [float(v) for v in affine]
    x, y = grid(wx, tx, W), grid(wy, ty, H)
    px = _axis_points(x, coord_bound(wx, tx, W, da[0], da[2]))  # [3, W]
    py = _axis_points(y, coord_bound(wy, ty, H, da[1], da[3]))  # [3, H]
    vals = np.stack([sample(img, px[a][None, :], py[b][:, None]) for a in range(3) for b in range(3)])
    lo, hi = vals.min(0), vals.max(0)
    cx = np.stack([np.floor(px[0]), np.floor(px[0]) + 1, np.floor(px[2]) + 1])
    cy = np.stack([np.floor(py[0]), np.floor(py[0]) + 1, np.floor(py[2]) + 1])
    a = np.abs(img)
    M = np.max(np.stack([_taps(a, cx[p][None, :], cy[q][:, None]) for p in range(3) for q in range(3)]), axis=0)
    return lo, hi, M


def _round_half_away(v):
    return np.sign(v) * np.floor(np.abs(v) + 0.5)


def _ambiguous(lo, hi, offset):
    """the interval [lo, hi] contains a threshold k + offset of round(s - offset + 1/2) for an integer k"""
    return np.floor(hi - offset) >= np.ceil(lo - offset)


def zoom_expect(img, affine, mode, mean=0.0, wx=None, da=(0.0, 0.0, 0.0, 0.0)):
    """What zoom_gather_kernel mode `mode` must produce on one plane under `affine` (the affine actually used: the zoom
    factor, or the inverse one).  Continuous modes (0, 3, 4, 6): ("interval", lo, hi).  Discrete modes (1, 2, 5):
    ("exact", value, ambiguous), value the float64 result where the pixel is not ambiguous.  mean: mode 3's channel mean;
    wx: the zoom factor's first entry for modes 4 and 6; da: the affine's uncertainty (inv_affine_f32)."""
    img = np.asarray(img, np.float64)
    if mode == 2:
        img = (img > THR_BIN).astype(np.float64)
    mean = float(F32(mean))  # pixel_means is an mx.nd.array: float32
    if mode == 3:
        img = img + mean
    lo, hi, M = sample_interval(img, affine, da)
    slack = 5 * U * M
    if mode == 3:
        slack = slack + U * M
    lo, hi = lo - slack * GAMMA, hi + slack * GAMMA
    if mode == 3:
        lo, hi = lo - mean, hi - mean
        r = U * np.maximum(np.abs(lo), np.abs(hi))
        return "interval", lo - r, hi + r
    if mode in (4, 6):
        s = float(wx) if mode == 4 else 1.0 / float(wx)
        lo, hi = lo * s, hi * s
        r = U * np.maximum(np.abs(lo), np.abs(hi)) * GAMMA
        return "interval", lo - r, hi + r
    if mode == 0:
        return "interval", lo, hi
    if mode == 5:
        r = U * (np.maximum(np.abs(lo), np.abs(hi)) + FLOW_OFFSET) + abs(float(F32(FLOW_OFFSET)) - FLOW_OFFSET)
        lo, hi = lo - FLOW_OFFSET - r, hi - FLOW_OFFSET + r
    amb = _ambiguous(lo, hi, 0.5)
    return "exact", _round_half_away(0.5 * (lo + hi)), amb


def check_plane(got, exp, tag):
    """assert a device (or oracle) plane against zoom_expect's result; returns the ambiguous share (0 for intervals)"""
    got = np.asarray(got, np.float64)
    if exp[0] == "interval":
        lo, hi = exp[1], exp[2]
        bad = np.argwhere(~((got >= lo) & (got <= hi)))
        assert not len(bad), "%s: %d pixels outside the float64 interval; first (i, j) = %s: got %r, interval [%r, %r]" % (
            tag, len(bad), tuple(bad[0]), got[tuple(bad[0])], lo[tuple(bad[0])], hi[tuple(bad[0])])
        return 0.0
    want, amb = exp[1], exp[2]
    share = float(amb.mean())
    assert share < MAX_AMBIGUOUS, "%s: %.3g of the pixels are ambiguous" % (tag, share)
    bad = np.argwhere((got != want) & ~amb)
    assert not len(bad), "%s: %d unambiguous pixels differ; first (i, j) = %s: got %r, want %r" % (
        tag, len(bad), tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])])
    return share


# ------------------------------------------------------------------------------------------------- affine, ZoomTrans
def inv_affine(zf, H, W):
    """zoom_flow.py:35-44: (lo, hi) float64 bounds of the inverse affine before its float32 storage (the formula's few
    float64 roundings, 8 ulp of float64 each way); the device stores the float32 rounding of a value in between"""
    wx_in, wy_in, tx_in, ty_in = [float(v) for v in zf]
    cx = tx_in * 0.5 * W + 0.5 * W
    cy = ty_in * 0.5 * H + 0.5 * H
    a = np.array([1.0 / wx_in, 1.0 / wy_in, (W * 0.5 - cx) / (wx_in * W) * 2.0, (H * 0.5 - cy) / (wy_in * H) * 2.0])
    # the translation's terms are at most (2 + |t_in|) / w_in in magnitude
    scale = np.array([abs(a[0]), abs(a[1]), (2 + abs(tx_in)) / abs(wx_in), (2 + abs(ty_in)) / abs(wy_in)])
    r = 8 * 2.0 ** -53 * scale
    return a - r, a + r


def inv_affine_f32(zf, H, W):
    """(lo, hi) float32: the float32 roundings of inv_affine's ends, between which the stored inverse affine lies"""
    lo, hi = inv_affine(zf, H, W)
    return lo.astype(F32), hi.astype(F32)


def inv_affine_for_sampling(zf, H, W):
    """(affine, da): a float32 inverse affine to sample at and how far the stored one may be from it (for zoom_expect)"""
    lo, hi = inv_affine_f32(zf, H, W)
    return lo, (hi.astype(np.float64) - lo.astype(np.float64))


def zoom_trans(zf, trans, inv, scale=True):
    """ZoomTrans forward (scale=True) and backward (scale = b_zoom_grad): x, y times (inv) or over wx, z unchanged.  The
    float64 product of two float32 values is exact, and a float64 quotient rounded to float32 is the correctly rounded
    float32 quotient (53 >= 2 * 24 + 2), so the float32 result is exact: returned as float32"""
    zf = np.asarray(zf, np.float64)
    t = np.asarray(trans, np.float64).copy()
    if scale:
        w = zf[:, :1]
        t[:, :2] = t[:, :2] * w if inv else t[:, :2] / w
    return t.astype(F32)


# -------------------------------------------------------------------------------------------------------------- boxes
def box(valid):
    """inclusive (x0, x1, y0, y1) of a boolean [H, W] map, -1s when empty"""
    cols, rows = np.flatnonzero(valid.any(0)), np.flatnonzero(valid.any(1))
    if not len(cols):
        return np.full(4, -1, np.int64)
    return np.array([cols[0], cols[-1], rows[0], rows[-1]])


def mask_valid(mask, rendered):
    """ZoomMask's valid map of a [C, H, W] mask: sum_c > 0.3, the rendered mask binarised at 0.2 first.  Returns (valid,
    ambiguous): the sum of C <= 3 float32 values rounds at most twice"""
    m = np.asarray(mask, np.float64)
    if rendered:
        m = (m > THR_BIN).astype(np.float64)
    s = m.sum(0)
    err = 2 * U * np.abs(m).sum(0) * GAMMA if m.shape[0] > 1 else 0.0
    return s > THR_MASK, np.abs(s - THR_MASK) <= err


def image_valid(image, means):
    """ZoomImage's valid map of a [3, H, W] image: sum_c (image_c + mean_c) > 0.01; five float32 roundings (three tap
    sums, two adds) at magnitude <= sum_c |image_c + mean_c| each.  Returns (valid, ambiguous)"""
    a = np.asarray(image, np.float64) + np.asarray(means, F32).astype(np.float64)[:, None, None]
    s = a.sum(0)
    err = 3 * U * np.abs(a).sum(0) * GAMMA
    return s > THR_IMG, np.abs(s - THR_IMG) <= err


def box_range(valid, ambiguous):
    """(largest, smallest) boxes over every reading of the ambiguous pixels"""
    return box(valid | ambiguous), box(valid & ~ambiguous)


def box_ok(got, valid, ambiguous):
    """the device's inclusive box lies between the smallest and the largest reading (equal when nothing is ambiguous)"""
    big, small = box_range(valid, ambiguous)
    got = np.asarray(got, np.int64)
    if (big == small).all():
        return (got == big).all()
    if got[1] < 0:
        return small[1] < 0
    if small[1] < 0:
        return (got[0] >= big[0]) & (got[1] <= big[1]) & (got[2] >= big[2]) & (got[3] <= big[3])
    return bool((big[0] <= got[0] <= small[0]) and (small[1] <= got[1] <= big[1]) and (big[2] <= got[2] <= small[2])
                and (small[3] <= got[3] <= big[3]))


def observed_rectangle(ren_box, H, W):
    """data_pair.py:93-105: ones on [y0:y1, x0:x1] of the rendered box (end-exclusive), float64 [H, W]"""
    m = np.zeros((H, W))
    x0, x1, y0, y1 = [int(v) for v in ren_box]
    if x1 >= 0:
        m[y0:y1, x0:x1] = 1.0
    return m


# -------------------------------------------------------------------------------------------------------- zoom factor
def _factor(real, ren, zcx, zcy, H, W):
    """zoom_mask.py:86-95 in float64 at one zoom centre: (wx, tx, ty)"""
    left = max(zcx - ren[0], zcx - real[0])
    right = max(ren[1] - zcx, real[1] - zcx)
    up = max(zcy - ren[2], zcy - real[2])
    down = max(real[3] - zcy, ren[3] - zcy)
    crop = max(0.75 * right, 0.75 * left, up, down) * 1.4 * 2
    return crop / H, zcx / W * 2 - 1, zcy / H * 2 - 1


def zoom_factor_range(real, ren, t, K, H, W):
    """(lo, hi) float64 bounds of (wx, wy, tx, ty) over the float32 error of c = K t and c / c2 (module docstring).  None
    for an empty observed box (the reference raises)."""
    real = [float(v) for v in real]
    ren = [float(v) for v in ren]
    if real[1] < 0:
        return None
    if ren[1] < 0:
        cxr, cyr = [(real[0] + real[1]) * 0.5] * 2, [(real[2] + real[3]) * 0.5] * 2
        ren = real
    else:
        K = np.asarray(K, F32).astype(np.float64).reshape(3, 3)
        t = np.asarray(t, F32).astype(np.float64)
        c = K @ t
        e = 3 * U / (1 - 3 * U) * (np.abs(K) @ np.abs(t)) + 2.0 ** -50 * np.abs(c)
        assert c[2] - e[2] > 0, "zoom centre behind the camera"

        def quot(i):
            q = [(c[i] + a) / (c[2] + b) for a in (-e[i], e[i]) for b in (-e[2], e[2])]
            lo, hi = min(q), max(q)
            return [lo - U * abs(lo) * GAMMA, hi + U * abs(hi) * GAMMA]
        cxr, cyr = quot(0), quot(1)
    # every term of m is monotone in one coordinate; the x terms' max is convex, with its minimum where left = right
    pts_x = [cxr[0], cxr[1], min(max((min(ren[0], real[0]) + max(ren[1], real[1])) * 0.5, cxr[0]), cxr[1])]
    pts_y = [cyr[0], cyr[1], min(max((min(ren[2], real[2]) + max(ren[3], real[3])) * 0.5, cyr[0]), cyr[1])]
    w = [_factor(real, ren, x, y, H, W)[0] for x in pts_x for y in pts_y]
    lo = np.array([min(w), min(w), cxr[0] / W * 2 - 1, cyr[0] / H * 2 - 1])
    hi = np.array([max(w), max(w), cxr[1] / W * 2 - 1, cyr[1] / H * 2 - 1])
    return lo, hi


def factor_ok(got, rng):
    """the stored float32 factor lies in the range widened by 1 ulp of float32"""
    lo, hi = rng
    got = np.asarray(got, np.float64)
    ulp_lo = np.spacing(np.abs(lo).astype(F32)).astype(np.float64)
    ulp_hi = np.spacing(np.abs(hi).astype(F32)).astype(np.float64)
    return bool(((got >= lo - ulp_lo) & (got <= hi + ulp_hi)).all())


# -------------------------------------------------------------------------------------------------------- conv1 input
def conv1_lanes(net):
    """conv1's input channels (deepIM_flownet.py:33-62): (blob, channels, divisor) in order"""
    lanes = [("zio", 3, 255.0), ("zir", 3, 255.0)]
    if net == "rgbd":
        lanes += [("zdo", 1, 255.0), ("zdr", 1, 255.0)]
    if net != "image":
        lanes += [("zmo", 1, 1.0), ("zmr", 1, 1.0)]
    return lanes


def _to16(v, fmt):
    import torch
    v32 = np.asarray(v, np.float64).astype(F32)
    if fmt == "fp16":
        return v32.astype(np.float16).astype(np.float64)
    return torch.from_numpy(np.ascontiguousarray(v32)).bfloat16().double().numpy()


def scaled_interval(lo, hi, divisor):
    """a continuous interval after the float32 division by 255 (one more rounding)"""
    lo, hi = lo / divisor, hi / divisor
    return lo - U * np.abs(lo) * GAMMA, hi + U * np.abs(hi) * GAMMA


def stored16_ok(hi16, lo16, lo, hi, prec):
    """conv1's stored 16-bit value(s) against the channel's interval [lo, hi] (already / 255): a boolean map"""
    if prec in ("fp16", "bf16"):
        fmt = "fp16" if prec == "fp16" else "bf16"
        return (hi16 >= _to16(lo, fmt)) & (hi16 <= _to16(hi, fmt))
    s = hi16.astype(np.float64) + lo16.astype(np.float64)
    e = np.where(lo16 == 0, 0.0, 2.0 ** (np.floor(np.log2(np.abs(np.where(lo16 == 0, 1.0, lo16)))) - 7))
    return (s >= lo - e) & (s <= hi + e)
