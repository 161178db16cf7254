// augment.cu -- train-time augmentation of the observed inputs (lib/utils/image.py:96-155 background replacement,
// lib/utils/mask_dilate.py observed-mask dilation).  Compiled with -fmad=false: the resize coordinates are double / float
// sequences specified operation by operation.
#include <math.h>

#include "launch.cuh"

namespace dim {

// Background geometry of one photo (image.py:108-145 and resize, image.py:552-572), in float64 like the reference.
// Canvas H x W = the observed image.  The photo is cropped from its top-left corner to the canvas aspect:
//   bh >= bw: crop height = ceil(bw * H/W), width bw;  bh < bw: crop width = ceil(bh / (H/W)), height bh.
// The reference branches on whether canvas and photo are both landscape / both portrait, but its two branches slice the
// same rows and columns (a numpy slice past the end stops at the end, which is the "if bg_h_new < bg_h" test of the
// first branch), so both reduce to the min() below.
// Then resize(crop, min(H, W), max(H, W)): scale = min / crop min side, unless round(scale * crop max side) > max, then
// max / crop max side; cv2.resize(fx = fy = scale) gives cvRound(crop side * scale) destination pixels.
int bg_geometry(int H, int W, int bh, int bw, BgGeom *g) {
  const double ratio = (double)H / (double)W;
  int ch = bh, cw = bw;
  if (bh >= bw) ch = min((int)ceil((double)bw * ratio), bh);
  else cw = min((int)ceil((double)bh / ratio), bw);
  const int tmin = min(H, W), tmax = max(H, W);
  const int smin = min(ch, cw), smax = max(ch, cw);
  double s = (double)tmin / (double)smin;
  if (nearbyint(s * (double)smax) > (double)tmax) s = (double)tmax / (double)smax;  // np.round: half to even
  g->crop_h = ch; g->crop_w = cw;
  g->dst_h = (int)nearbyint((double)ch * s);  // saturate_cast<int>(double) = cvRound: half to even
  g->dst_w = (int)nearbyint((double)cw * s);
  g->scale = s;
  if (g->dst_h > H || g->dst_w > W || g->dst_h < 1 || g->dst_w < 1) {
    set_error("background %dx%d: resized crop %dx%d does not fit the %dx%d canvas", bh, bw, g->dst_h, g->dst_w, H, W);
    return 2;
  }
  // 1/scale == 2 exactly: cv2 switches INTER_LINEAR to its fast INTER_AREA path.  Where every destination pixel has a full
  // 2x2 source cell both give the same bytes (verified against cv2 4.13); with an odd crop side the last row / column
  // averages a partial cell, which this kernel does not reproduce.
  if (1.0 / s == 2.0 && (2 * g->dst_h > ch || 2 * g->dst_w > cw)) {
    set_error("background %dx%d: a crop of %dx%d at scale exactly 1/2 takes cv2's partial-cell INTER_AREA border path, "
              "which is not reproduced", bh, bw, ch, cw);
    return 2;
  }
  return 0;
}

// OpenCV 4.x cv::resize(INTER_LINEAR) on CV_8U, pinned against cv2 4.13.0 (bit for bit on random sizes and scales):
//   x: fx = (float)((dx + 0.5) * (1/scale) - 0.5); sx = floor(fx); fx -= sx; sx < 0 -> (sx, fx) = (0, 0);
//      sx >= w - 1 -> (sx, fx) = (w - 1, 0); alpha = (cvRound((1 - fx) * 2048), cvRound(fx * 2048)) (int16; may not sum
//      to 2048);  row sum T = S[sx] * alpha0 + S[sx + 1] * alpha1 (int32, exact);
//   y: the same fy / sy / beta, but only the source ROW indices are clamped to [0, h - 1] (beta keeps fy);
//   out = sat_u8((mulhi16(T0 >> 4, beta0) + mulhi16(T1 >> 4, beta1) + 2) >> 2), mulhi16(a, b) = (a * b) >> 16 -- the
//      SIMD vertical pass (VResizeLinearVec_32s8u), which cv2 4.13 also applies to the tail of each row, rather than the
//      scalar (T0 * beta0 + T1 * beta1 + 2^21) >> 22.
// The reference's requirements.txt leaves OpenCV unpinned; another version may round differently.
__device__ __forceinline__ void lin_tap(int d, double inv, int n, int clamp_weight, int &s0, int &s1, int &w0, int &w1) {
  float f = (float)__dsub_rn(__dmul_rn((double)d + 0.5, inv), 0.5);
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  if (clamp_weight) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= n - 1) { f = 0.f; s = n - 1; }
  }
  w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  w1 = __float2int_rn(__fmul_rn(f, 2048.f));
  s0 = min(max(s, 0), n - 1);
  s1 = min(max(s + 1, 0), n - 1);
}

// One thread per canvas pixel: composite = mask != 0 ? (u8) observed : (inside the resized crop ? resized photo : 0),
// image = float32(float64(composite) - mean) in RGB CHW (image.py:583-594).
__global__ void __launch_bounds__(256) replace_bg_kernel(BgLaunch L, const float *obs, const float *mask, int H, int W,
                                                         float *image, uint8_t *comp) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int bl = blockIdx.y;
  if (q >= H * W) return;
  const BgInst &in = L.inst[bl];
  const int b = L.b0 + bl;
  const size_t P = (size_t)H * W;
  const int y = q / W, x = q - y * W;
  const float *o = obs + ((size_t)b * P + q) * 3;
  int c[3];
  if (in.data == nullptr || mask[(size_t)b * P + q] != 0.f) {
#pragma unroll
    for (int k = 0; k < 3; ++k) c[k] = (int)(uint8_t)fminf(fmaxf(o[k], 0.f), 255.f);  // numpy's float -> uint8 store
  } else if (y < in.dst_h && x < in.dst_w) {
    int x0, x1, a0, a1, y0, y1, b0, b1;
    lin_tap(x, in.inv_scale, in.crop_w, 1, x0, x1, a0, a1);
    lin_tap(y, in.inv_scale, in.crop_h, 0, y0, y1, b0, b1);
    const uint8_t *r0 = in.data + (size_t)y0 * in.stride * 3, *r1 = in.data + (size_t)y1 * in.stride * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int t0 = r0[x0 * 3 + k] * a0 + r0[x1 * 3 + k] * a1;
      const int t1 = r1[x0 * 3 + k] * a0 + r1[x1 * 3 + k] * a1;
      const int v = ((((t0 >> 4) * b0) >> 16) + (((t1 >> 4) * b1) >> 16) + 2) >> 2;
      c[k] = min(max(v, 0), 255);
    }
  } else {
    c[0] = c[1] = c[2] = 0;
  }
  if (comp) {
    uint8_t *d = comp + ((size_t)b * P + q) * 3;
    d[0] = (uint8_t)c[0]; d[1] = (uint8_t)c[1]; d[2] = (uint8_t)c[2];
  }
  float *im = image + (size_t)b * 3 * P;
  im[q] = (float)((double)c[2] - L.mean[0]);
  im[P + q] = (float)((double)c[1] - L.mean[1]);
  im[2 * P + q] = (float)((double)c[0] - L.mean[2]);
}

int replace_bg_launch(dim_ctx *ctx, const BgLaunch &L, int nb, const float *obs, const float *mask, float *image,
                      uint8_t *comp, cudaStream_t st) {
  replace_bg_kernel<<<dim3(cdiv(ctx->H * ctx->W, 256), nb), 256, 0, st>>>(L, obs, mask, ctx->H, ctx->W, image, comp);
  DIM_LAUNCH_CHECK();
  return 0;
}

// mask_dilate.py:19-47.  draws[b] = direction, then the thickness of the down, up, right and left shift (<= 0: skipped).
// Every shift tests the ORIGINAL mask (a pixel gains 1 per side whose shifted source is nonzero while it is zero itself),
// so the result is orig where orig != 0 (clipped to 1 above 1, anything else left as it is) and min(gains, 1) elsewhere.
__global__ void __launch_bounds__(256) mask_dilate_kernel(const float *in, const int *draws, int H, int W, float *out) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (q >= H * W) return;
  const float *m = in + (size_t)b * H * W;
  const int y = q / W, x = q - y * W;
  const float v = m[q];
  float r;
  if (v != 0.f) {
    r = v > 1.f ? 1.f : v;
  } else {
    const int *d = draws + 5 * b;
    const int td = d[1], tu = d[2], tr = d[3], tl = d[4];
    const bool hit = (td > 0 && y >= td && m[q - td * W] != 0.f) || (tu > 0 && y + tu < H && m[q + tu * W] != 0.f) ||
                     (tr > 0 && x >= tr && m[q - tr] != 0.f) || (tl > 0 && x + tl < W && m[q + tl] != 0.f);
    r = hit ? 1.f : 0.f;
  }
  out[(size_t)b * H * W + q] = r;
}

int mask_dilate_launch(dim_ctx *ctx, const float *in, const int *draws, int B, float *out, cudaStream_t st) {
  mask_dilate_kernel<<<dim3(cdiv(ctx->H * ctx->W, 256), B), 256, 0, st>>>(in, draws, ctx->H, ctx->W, out);
  DIM_LAUNCH_CHECK();
  return 0;
}

}  // namespace dim
