// zoom.cu -- mask bbox, zoom factor and the bilinear zoom gathers (compiled with -fmad=false).
//
// Replaces the Python custom ops of deepim/operator_py/: ZoomMask (zoom_mask.py:29-112),
// ZoomImageWithFactor (zoom_image_with_factor.py:31-65), ZoomMaskWithFactor
// (zoom_mask_with_factor.py:29-64), ZoomFlow (zoom_flow.py:28-71), ZoomDepth (zoom_depth.py:24-44)
// and the MXNet GridGenerator('affine') + BilinearSampler pair they call (SURVEY 8(a) row a6):
//     x_t = -1 + j*(2/(W-1)),  x_s = wx*x_t + tx,  x = (x_s+1)*(W-1)/2,  4 taps, zero padding.
// The reference does the bbox on the host after three full-mask asnumpy() syncs and one
// GridGenerator launch per sample; here everything stays on the device.
#include <cuda_fp16.h>

#include "launch.cuh"

namespace dim {

// ------------------------------------------------------------------------------------- bbox
__global__ void bbox_init_kernel(int *bbox8, int B, int H, int W) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * 2) return;
  bbox8[4 * t + 0] = W;
  bbox8[4 * t + 1] = -1;
  bbox8[4 * t + 2] = H;
  bbox8[4 * t + 3] = -1;
}

// one block per (row, instance, which-mask).  valid = sum_c(mask) > 0.3 (zoom_mask.py:36-37), with
// each channel binarised at 0.2 first for the rendered mask (l.39-43).
// img_mode (ZoomImage, zoom_image.py:33-37): valid = sum_c(img + pixel_mean_c) > 0.01 for both images.
__global__ void __launch_bounds__(160) mask_bbox_kernel(const float *mask_real, const float *mask_ren, int C,
                                                        int H, int W, int *bbox8, int img_mode, float m0, float m1,
                                                        float m2) {
  const int i = blockIdx.x, b = blockIdx.y, which = blockIdx.z;
  const float *src = (which == 0 ? mask_real : mask_ren) + (size_t)b * C * H * W + (size_t)i * W;
  int x0 = 0x7fffffff, x1 = -1;
  for (int j4 = threadIdx.x * 4; j4 < W; j4 += blockDim.x * 4) {
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    for (int c = 0; c < C; ++c) {
      float4 v = *reinterpret_cast<const float4 *>(src + (size_t)c * H * W + j4);
      float e[4] = {v.x, v.y, v.z, v.w};
      const float mc = c == 0 ? m0 : (c == 1 ? m1 : m2);
#pragma unroll
      for (int k = 0; k < 4; ++k) s[k] += img_mode ? (e[k] + mc) : (which ? (e[k] > 0.2f ? 1.f : 0.f) : e[k]);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (s[k] > (img_mode ? 0.01f : 0.3f)) {
        x0 = min(x0, j4 + k);
        x1 = max(x1, j4 + k);
      }
  }
  x0 = __reduce_min_sync(0xffffffffu, x0);
  x1 = __reduce_max_sync(0xffffffffu, x1);
  if ((threadIdx.x & 31) == 0 && x1 >= 0) {
    int *o = bbox8 + (b * 2 + which) * 4;
    atomicMin(o + 0, x0);
    atomicMax(o + 1, x1);
    atomicMin(o + 2, i);
    atomicMax(o + 3, i);
  }
}

// zoom factor, one thread per instance (zoom_mask.py:59-103; ZoomImage's is the same code, zoom_image.py:41-86).  Mixed
// precision as the reference's numpy 1.x: c = K.t and c_x = c0/c2 in float32, everything after in float64, stored as float32.
// ren_empty_bit: status bit set where the rendered box is empty and the zoom centres on the observed box (0: none)
// cams: instance b uses the camera cams.K(b); an instance whose frame index is out of range gets status bit 3
__global__ void zoom_factor_kernel(int *bbox8, const float *src_pose, int B, int H, int W, FrameCams cams,
                                   float *zoom_factor, int *bbox_out, int *status, const int *cls_flag, int ren_empty_bit) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float k[9];
  cams.K(b, k);
  // rasteriser: bad class index (bit 1); frame index out of range (bit 3)
  const int cf = (cls_flag ? cls_flag[b] : 0) | (cams.bad(b) ? 8 : 0);
  int *bb = bbox8 + 8 * b;
  if (bb[1] < 0) bb[0] = bb[1] = bb[2] = bb[3] = -1;
  if (bb[5] < 0) bb[4] = bb[5] = bb[6] = bb[7] = -1;
  if (bbox_out)
    for (int k = 0; k < 8; ++k) bbox_out[8 * b + k] = bb[k];
  float *zf = zoom_factor + 4 * b;
  if (bb[1] < 0) {  // the reference raises (np.min of an empty array); flag it
    zf[0] = zf[1] = 1.f;
    zf[2] = zf[3] = 0.f;
    if (status) status[b] = 1 | cf;
    return;
  }
  if (status) status[b] = cf | (bb[5] < 0 ? ren_empty_bit : 0);
  const double real_x0 = bb[0], real_x1 = bb[1], real_y0 = bb[2], real_y1 = bb[3];
  const float *sp = src_pose + 12 * b;
  const float t0 = sp[3], t1 = sp[7], t2 = sp[11];
  const float c0 = (k[0] * t0 + k[1] * t1) + k[2] * t2;
  const float c1 = (k[3] * t0 + k[4] * t1) + k[5] * t2;
  const float c2 = (k[6] * t0 + k[7] * t1) + k[8] * t2;
  const float cxf = c0 / c2, cyf = c1 / c2;
  double ren_x0, ren_x1, ren_y0, ren_y1, zcx, zcy;
  if (bb[5] < 0) {  // "NO POINT VALID IN MASK rendered" (zoom_mask.py:70-77)
    ren_x0 = real_x0; ren_x1 = real_x1; ren_y0 = real_y0; ren_y1 = real_y1;
    zcx = (real_x0 + real_x1) * 0.5;
    zcy = (real_y0 + real_y1) * 0.5;
  } else {
    ren_x0 = bb[4]; ren_x1 = bb[5]; ren_y0 = bb[6]; ren_y1 = bb[7];
    zcx = (double)cxf;
    zcy = (double)cyf;
  }
  const double left = fmax(zcx - ren_x0, zcx - real_x0);
  const double right = fmax(ren_x1 - zcx, real_x1 - zcx);
  const double up = fmax(zcy - ren_y0, zcy - real_y0);
  const double down = fmax(real_y1 - zcy, ren_y1 - zcy);
  const double m = fmax(fmax(0.75 * right, 0.75 * left), fmax(up, down));
  const double crop_height = m * 1.4 * 2;
  const double wx = crop_height / (double)H;
  zf[0] = (float)wx;
  zf[1] = (float)wx;
  zf[2] = (float)(zcx / (double)W * 2.0 - 1.0);
  zf[3] = (float)(zcy / (double)H * 2.0 - 1.0);
}

// ------------------------------------------------------------------------------------ sampler
struct Tap {
  int x0, y0;
  float wx1, wy1;
};

__device__ __forceinline__ Tap src_coord(int i, int j, float wx, float wy, float tx, float ty, int H, int W,
                                         float stepx, float stepy) {
  float xt = -1.0f + (float)j * stepx;
  float yt = -1.0f + (float)i * stepy;
  float xs = wx * xt + tx;
  float ys = wy * yt + ty;
  float xr = ((xs + 1.0f) * (float)(W - 1)) / 2.0f;
  float yr = ((ys + 1.0f) * (float)(H - 1)) / 2.0f;
  float fx0 = floorf(xr), fy0 = floorf(yr);
  Tap t;
  t.x0 = fx0 < -4.0f ? -4 : (fx0 > (float)(W + 4) ? W + 4 : (int)fx0);
  t.y0 = fy0 < -4.0f ? -4 : (fy0 > (float)(H + 4) ? H + 4 : (int)fy0);
  t.wx1 = 1.0f - (xr - fx0);
  t.wy1 = 1.0f - (yr - fy0);
  return t;
}

template <int BIN>
__device__ __forceinline__ float fetch(const float *img, int H, int W, int y, int x, float add) {
  if (x < 0 || x > W - 1 || y < 0 || y > H - 1) return 0.0f;
  float v = __ldg(img + (size_t)y * W + x);
  if (BIN) v = v > 0.2f ? 1.0f : 0.0f;
  return v + add;
}

template <int BIN>
__device__ __forceinline__ float bilinear(const float *img, int H, int W, const Tap &t, float add) {
  float tl = fetch<BIN>(img, H, W, t.y0, t.x0, add);
  float tr = fetch<BIN>(img, H, W, t.y0, t.x0 + 1, add);
  float bl = fetch<BIN>(img, H, W, t.y0 + 1, t.x0, add);
  float br = fetch<BIN>(img, H, W, t.y0 + 1, t.x0 + 1, add);
  const float wx1 = t.wx1, wy1 = t.wy1, ax = 1.0f - wx1, ay = 1.0f - wy1;
  const float a = wy1 * wx1, b = wy1 * ax, c = ay * wx1, d = ay * ax;
  return fmaf(br, d, fmaf(bl, c, fmaf(tr, b, tl * a)));
}

// inverse-zoom affine (zoom_flow.py:35-44): float32 scalars with python numbers -> float64
__device__ __forceinline__ void inv_affine(const float *zf, int H, int W, float *a) {
  double wx_in = zf[0], wy_in = zf[1], tx_in = zf[2], ty_in = zf[3];
  double wx = 1.0 / wx_in, wy = 1.0 / wy_in;
  double crop_w = wx_in * (double)W, crop_h = wy_in * (double)H;
  double cx = tx_in * 0.5 * (double)W + 0.5 * (double)W;
  double cy = ty_in * 0.5 * (double)H + 0.5 * (double)H;
  a[0] = (float)wx;
  a[1] = (float)wy;
  a[2] = (float)(((double)W * 0.5 - cx) / crop_w * 2.0);
  a[3] = (float)(((double)H * 0.5 - cy) / crop_h * 2.0);
}

// MODE 0 plain | 1 round | 2 binarise(>0.2) then round | 3 (img+mean) sample - mean |
//      4 sample * wx | 5 round(sample - 0.45) | 6 sample / wx
struct ZoomParams {
  const float *src;
  float *dst;
  const float *zoom_factor;  // [B,4]
  int C, H, W, inv;
  float param[4];  // per-channel mean for MODE 3
  float stepx, stepy;
};

template <int MODE>
__global__ void __launch_bounds__(256) zoom_gather_kernel(ZoomParams p) {
  __shared__ float aff[4];
  const int b = blockIdx.y;
  if (threadIdx.x == 0) {
    const float *zf = p.zoom_factor + 4 * b;
    if (p.inv) {
      inv_affine(zf, p.H, p.W, aff);
    } else {
      aff[0] = zf[0]; aff[1] = zf[1]; aff[2] = zf[2]; aff[3] = zf[3];
    }
  }
  __syncthreads();
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= p.H * p.W) return;
  const int i = q / p.W, j = q % p.W;
  const Tap t = src_coord(i, j, aff[0], aff[1], aff[2], aff[3], p.H, p.W, p.stepx, p.stepy);
  const float wxf = p.zoom_factor[4 * b];
  const size_t P = (size_t)p.H * p.W;
  for (int c = 0; c < p.C; ++c) {
    const float *img = p.src + ((size_t)b * p.C + c) * P;
    float v;
    if (MODE == 1) v = roundf(bilinear<0>(img, p.H, p.W, t, 0.f));
    else if (MODE == 2) v = roundf(bilinear<1>(img, p.H, p.W, t, 0.f));
    else if (MODE == 3) v = bilinear<0>(img, p.H, p.W, t, p.param[c]) - p.param[c];
    else if (MODE == 4) v = bilinear<0>(img, p.H, p.W, t, 0.f) * wxf;
    else if (MODE == 5) v = roundf(bilinear<0>(img, p.H, p.W, t, 0.f) - 0.45f);
    else if (MODE == 6) v = bilinear<0>(img, p.H, p.W, t, 0.f) / wxf;
    else v = bilinear<0>(img, p.H, p.W, t, 0.f);
    p.dst[((size_t)b * p.C + c) * P + q] = v;
  }
}

int zoom_gather_launch(dim_ctx *ctx, int mode, const float *src, float *dst, const float *zoom_factor, int B, int C,
                       int inv, const float *param, cudaStream_t st) {
  ZoomParams p;
  p.src = src; p.dst = dst; p.zoom_factor = zoom_factor; p.C = C; p.H = ctx->H; p.W = ctx->W; p.inv = inv;
  for (int k = 0; k < 4; ++k) p.param[k] = (param && k < C) ? param[k] : 0.f;
  p.stepx = (float)(2.0 / (double)(ctx->W - 1));
  p.stepy = (float)(2.0 / (double)(ctx->H - 1));
  dim3 grid(cdiv(ctx->H * ctx->W, 256), B);
  switch (mode) {
    case 0: zoom_gather_kernel<0><<<grid, 256, 0, st>>>(p); break;
    case 1: zoom_gather_kernel<1><<<grid, 256, 0, st>>>(p); break;
    case 2: zoom_gather_kernel<2><<<grid, 256, 0, st>>>(p); break;
    case 3: zoom_gather_kernel<3><<<grid, 256, 0, st>>>(p); break;
    case 4: zoom_gather_kernel<4><<<grid, 256, 0, st>>>(p); break;
    case 5: zoom_gather_kernel<5><<<grid, 256, 0, st>>>(p); break;
    case 6: zoom_gather_kernel<6><<<grid, 256, 0, st>>>(p); break;
    default: set_error("zoom_gather: bad mode"); return 2;
  }
  DIM_LAUNCH_CHECK();
  return 0;
}

int zoom_factor_launch(dim_ctx *ctx, const float *mask_real, const float *mask_ren, int C, const float *src_pose,
                       int B, const float *K9, float *zoom_factor, int *bbox_out, int *status, cudaStream_t st,
                       const float *img_means) {
  DIM_REQUIRE((ctx->W & 3) == 0, "width must be a multiple of 4");
  bbox_init_kernel<<<cdiv(2 * B, 128), 128, 0, st>>>(ctx->bbox8, B, ctx->H, ctx->W);
  DIM_LAUNCH_CHECK();
  mask_bbox_kernel<<<dim3(ctx->H, B, 2), 160, 0, st>>>(mask_real, mask_ren, C, ctx->H, ctx->W, ctx->bbox8,
                                                       img_means ? 1 : 0, img_means ? img_means[0] : 0.f,
                                                       img_means ? img_means[1] : 0.f, img_means ? img_means[2] : 0.f);
  DIM_LAUNCH_CHECK();
  zoom_factor_kernel<<<cdiv(B, 64), 64, 0, st>>>(ctx->bbox8, src_pose, B, ctx->H, ctx->W, frame_cams(K9), zoom_factor,
                                                  bbox_out, status, nullptr, 0);
  DIM_LAUNCH_CHECK();
  return 0;
}

// zoom factor when both boxes are already known (fused loop: the rendered box comes from the
// rasteriser, the observed box is the end-exclusive rectangle of it, data_pair.py:93-105)
__global__ void zoom_factor_from_ren_kernel(const int *bbox_ren, int *bbox8, int B) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int x0 = bbox_ren[4 * b], x1 = bbox_ren[4 * b + 1], y0 = bbox_ren[4 * b + 2], y1 = bbox_ren[4 * b + 3];
  int *bb = bbox8 + 8 * b;
  bb[4] = x0; bb[5] = x1; bb[6] = y0; bb[7] = y1;
  // rectangle [y0:y1, x0:x1] is empty when the mask is a single row/column (or empty)
  if (x1 < 0 || x1 - 1 < x0 || y1 - 1 < y0) {
    bb[0] = bb[1] = bb[2] = bb[3] = -1;
  } else {
    bb[0] = x0; bb[1] = x1 - 1; bb[2] = y0; bb[3] = y1 - 1;
  }
}

int zoom_factor_from_ren_launch(dim_ctx *ctx, const int *bbox_ren, const float *src_pose, int B, const FrameCams &cams,
                                float *zoom_factor, int *bbox_out, int *status, cudaStream_t st) {
  zoom_factor_from_ren_kernel<<<cdiv(B, 64), 64, 0, st>>>(bbox_ren, ctx->bbox8, B);
  DIM_LAUNCH_CHECK();
  zoom_factor_kernel<<<cdiv(B, 64), 64, 0, st>>>(ctx->bbox8, src_pose, B, ctx->H, ctx->W, cams, zoom_factor, bbox_out, status,
                                                  ctx->cls_flag, 0);
  DIM_LAUNCH_CHECK();
  return 0;
}

// Image-only network (ZoomImage, zoom_image.py:33-37): the observed box of the fused loop, valid = sum_c(image + mean) > 0.01
// over obs4's colours (which hold image + mean), the float32 sum of mask_bbox_kernel's img_mode in the same channel order.
// Once per dim_refine call: the observed image does not change over the iterations.  One block per (row, frame): with
// a frame map each frame's box is reduced once, however many instances observe it.
__global__ void __launch_bounds__(160) obs_colour_box_kernel(const float4 *obs4, int H, int W, int *bbox_obs) {
  const int i = blockIdx.x, b = blockIdx.y;
  const float4 *src = obs4 + ((size_t)b * H + i) * W;
  int x0 = 0x7fffffff, x1 = -1;
  for (int j = threadIdx.x; j < W; j += blockDim.x) {
    const float4 v = src[j];
    if (((v.x + v.y) + v.z) > 0.01f) {
      x0 = min(x0, j);
      x1 = max(x1, j);
    }
  }
  x0 = __reduce_min_sync(0xffffffffu, x0);
  x1 = __reduce_max_sync(0xffffffffu, x1);
  if ((threadIdx.x & 31) == 0 && x1 >= 0) {
    int *o = bbox_obs + 4 * b;
    atomicMin(o + 0, x0);
    atomicMax(o + 1, x1);
    atomicMin(o + 2, i);
    atomicMax(o + 3, i);
  }
}

__global__ void box4_init_kernel(int *box, int B, int H, int W) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  box[4 * b + 0] = W;
  box[4 * b + 1] = -1;
  box[4 * b + 2] = H;
  box[4 * b + 3] = -1;
}

int obs_colour_box_launch(dim_ctx *ctx, const float4 *obs4, int F, int *bbox_obs, cudaStream_t st) {
  box4_init_kernel<<<cdiv(F, 64), 64, 0, st>>>(bbox_obs, F, ctx->H, ctx->W);
  DIM_LAUNCH_CHECK();
  obs_colour_box_kernel<<<dim3(ctx->H, F), 160, 0, st>>>(obs4, ctx->H, ctx->W, bbox_obs);
  DIM_LAUNCH_CHECK();
  return 0;
}

// zoom factor of the image-only loop: the observed box from obs_colour_box_kernel, the rendered one from the rasteriser's
// colour-valid bbox (raster.cu COLOUR_BOX), then ZoomImage's arithmetic -- zoom_factor_kernel, with the observed-centre
// fallback for an empty render flagged as status bit 2 (the reference prints "NO POINT VALID IN rendered" and goes on); an
// empty observed image is bit 0 with the (1,1,0,0) factor (the reference raises).
// bbox_obs holds one box per frame; the instance's observed box is gathered here from its frame (cams.frame).
__global__ void boxes_to_bbox8_kernel(const int *bbox_obs, const int *bbox_ren, int *bbox8, int B, FrameCams cams) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int f = cams.frame(b);
  for (int k = 0; k < 4; ++k) {
    bbox8[8 * b + k] = bbox_obs[4 * f + k];
    bbox8[8 * b + 4 + k] = bbox_ren[4 * b + k];
  }
}

int zoom_factor_from_boxes_launch(dim_ctx *ctx, const int *bbox_obs, const int *bbox_ren, const float *src_pose, int B,
                                  const FrameCams &cams, float *zoom_factor, int *bbox_out, int *status, cudaStream_t st) {
  boxes_to_bbox8_kernel<<<cdiv(B, 64), 64, 0, st>>>(bbox_obs, bbox_ren, ctx->bbox8, B, cams);
  DIM_LAUNCH_CHECK();
  zoom_factor_kernel<<<cdiv(B, 64), 64, 0, st>>>(ctx->bbox8, src_pose, B, ctx->H, ctx->W, cams, zoom_factor, bbox_out, status,
                                                  ctx->cls_flag, 4);
  DIM_LAUNCH_CHECK();
  return 0;
}

// mask_observed := 1 on [y0:y1, x0:x1] END-EXCLUSIVE (lib/pair_matching/data_pair.py:93-105)
__global__ void __launch_bounds__(256) box_mask_kernel(const int *bbox, int H, int W, float *mask) {
  const int b = blockIdx.y;
  const int q4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (q4 >= H * W) return;
  const int i = q4 / W, j = q4 % W;
  const int x0 = bbox[4 * b], x1 = bbox[4 * b + 1], y0 = bbox[4 * b + 2], y1 = bbox[4 * b + 3];
  float v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = (x1 >= 0 && i >= y0 && i < y1 && j + k >= x0 && j + k < x1) ? 1.f : 0.f;
  *reinterpret_cast<float4 *>(mask + (size_t)b * H * W + q4) = make_float4(v[0], v[1], v[2], v[3]);
}

int box_mask_launch(dim_ctx *ctx, const int *bbox, int B, float *mask, cudaStream_t st) {
  box_mask_kernel<<<dim3(cdiv(ctx->H * ctx->W / 4, 256), B), 256, 0, st>>>(bbox, ctx->H, ctx->W, mask);
  DIM_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------- fused zoom -> NHWC8
// One thread per 2x2 quad of output pixels: samples the 6 image planes (with the +mean / -mean dance of
// zoom_image_with_factor.py:44-62), the rendered mask and the analytic observed box mask with the
// same taps, applies the graph's /255 (deepIM_flownet.py:53-60) and writes the 8-channel pixels as
// bf16 / fp16 (16 B each) straight into conv1's zero-bordered, space-to-depth input buffer; `lo` (optional) receives the
// bf16 residual for the bf16x3 precision mode.
// The two source images already hold (image + mean) -- the sampler's first step, done once by their producers with the
// same float32 addition -- so a tap costs no arithmetic before its weight.
struct FusedZoomParams {
  const float4 *obs4;   // [F,H,W,4] observed frames (RGB - mean) + mean, w unused (RGB-D network: w = depth_observed)
  const int32_t *frame_idx;  // [B] frame of each instance (FrameCams::frame); nullptr: frame b
  int n_frames;
  const float4 *ren4;   // [B,H,W,4] rendered (RGB - mean) + mean, w = mask_rendered (0/1) (RGB-D network: w = depth)
  const int *bbox8;     // observed box = bb[0..3] (inclusive)
  const int *vbox;      // [B,4] x0,x1,y0,y1: ren4 is only valid inside this box (rasteriser), background outside; nullable
  float bg[3];          // background of the rendered image + mean: (float)(0.0 - mean) + (float)mean
  const float *zoom_factor;
  int H, W, Hs, Ws, pad;  // conv1 input is space-to-depth: [B,Hs,Ws,(ph,pw,c)=32]
  float mean[3];
  float stepx, stepy;
  __nv_bfloat16 *hi, *lo;
};

__device__ __forceinline__ uint32_t pack2_f16(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t *>(&h);
}

// One axis of the sampler (mx.sym.GridGenerator affine + BilinearSampler, same float32 sequence as src_coord): the two
// taps c0, c0 + 1 of output coordinate `o`, their weights with zero padding folded in (an out-of-frame tap gets weight 0
// and an arbitrary in-bounds address: it contributes exactly +0, the sampler's "value 0"), whether each tap lies in the
// rendered image's valid box [v0, v1] and in the observed box [m0, m1].
struct AxisTap {
  int a0, a1;      // clamped tap coordinates (in frame)
  float w0, w1;    // tap weights, 0 outside the frame
  bool r0, r1;     // tap in frame and inside the rendered-valid box
  bool m0, m1;     // tap inside the observed box (out-of-frame taps carry weight 0, so the frame test is not needed)
};
__device__ __forceinline__ AxisTap axis_tap(int o, float w, float t, int N, float step, int v0, int v1, int m0, int m1) {
  const float ct = -1.0f + (float)o * step;
  const float cs = w * ct + t;
  const float cr = ((cs + 1.0f) * (float)(N - 1)) / 2.0f;
  const float f0 = floorf(cr);
  const int c0 = f0 < -4.0f ? -4 : (f0 > (float)(N + 4) ? N + 4 : (int)f0);
  const float wa = 1.0f - (cr - f0), wb = 1.0f - wa;
  const bool ok0 = c0 >= 0 && c0 <= N - 1, ok1 = c0 + 1 >= 0 && c0 + 1 <= N - 1;
  AxisTap a;
  a.a0 = ok0 ? c0 : 0;
  a.a1 = ok1 ? c0 + 1 : 0;
  a.w0 = ok0 ? wa : 0.f;
  a.w1 = ok1 ? wb : 0.f;
  a.r0 = ok0 && c0 >= v0 && c0 <= v1;
  a.r1 = ok1 && c0 + 1 >= v0 && c0 + 1 <= v1;
  a.m0 = c0 >= m0 && c0 <= m1;
  a.m1 = c0 + 1 >= m0 && c0 + 1 <= m1;
  return a;
}

// eight channel values -> one 16-byte chunk (bf16 / fp16), `l` the bf16 residuals (bf16x3)
template <bool LO, bool F16>
__device__ __forceinline__ void pack_chunk(const float *v, uint4 &h, uint4 &l) {
  if (F16) {  // |v| <= 1 (depth: metres / 255): always in range
    h = make_uint4(pack2_f16(v[0], v[1]), pack2_f16(v[2], v[3]), pack2_f16(v[4], v[5]), pack2_f16(v[6], v[7]));
  } else {
    uint32_t hh[4], ll[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const __nv_bfloat16 h0 = __float2bfloat16_rn(v[2 * c]), h1 = __float2bfloat16_rn(v[2 * c + 1]);
      hh[c] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
      if (LO) {
        const __nv_bfloat16 l0 = __float2bfloat16_rn(v[2 * c] - __bfloat162float(h0));
        const __nv_bfloat16 l1 = __float2bfloat16_rn(v[2 * c + 1] - __bfloat162float(h1));
        ll[c] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
      }
    }
    h = make_uint4(hh[0], hh[1], hh[2], hh[3]);
    if (LO) l = make_uint4(ll[0], ll[1], ll[2], ll[3]);
  }
}

// DEPTH (RGB-D network, deepIM_flownet.py:35-43): the channels are image_observed/255, image_rendered/255,
// depth_observed/255, depth_rendered/255, mask_observed, mask_rendered in two chunks (channels 0-7, then 8-9 and zeros).
// The depths ride in the w lanes: obs4.w = depth_observed, ren4.w = the render's depth (0 = background, so the rendered
// mask depth > 0.2 of tester.py:440 is the same binarisation at 0.2 as for the 0/1 mask).  ZoomDepth (zoom_depth.py:24-44)
// is the plain bilinear sample, zero outside the frame: the image taps with no mean.
// MASK = false (image-only network, INPUT_MASK: False, deepIM_flownet.py:53-62): channels 6 and 7 are exact zeros -- conv1's
// weight pack carries zero columns there -- and neither the box mask nor the ren4.w taps are computed.
template <bool LO, bool F16, bool DEPTH = false, bool MASK = true>
__device__ __forceinline__ void zoom_fused_pixel(const FusedZoomParams &p, const float4 *__restrict__ ob,
                                                 const float4 *__restrict__ rn, const AxisTap &x, const AxisTap &y,
                                                 uint4 (&h)[DEPTH ? 2 : 1], uint4 (&l)[DEPTH ? 2 : 1]) {
  const int W = p.W;
  const int y0 = y.a0 * W, y1 = y.a1 * W;
  const float4 O00 = __ldg(ob + (y0 + x.a0)), O01 = __ldg(ob + (y0 + x.a1));
  const float4 O10 = __ldg(ob + (y1 + x.a0)), O11 = __ldg(ob + (y1 + x.a1));
  // rendered taps: outside the rasteriser's vertex box the image is background by construction (and ren4 is not written there)
  const float4 bg4 = make_float4(p.bg[0], p.bg[1], p.bg[2], 0.f);
  const float4 R00 = (y.r0 && x.r0) ? __ldg(rn + (y0 + x.a0)) : bg4;
  const float4 R01 = (y.r0 && x.r1) ? __ldg(rn + (y0 + x.a1)) : bg4;
  const float4 R10 = (y.r1 && x.r0) ? __ldg(rn + (y1 + x.a0)) : bg4;
  const float4 R11 = (y.r1 && x.r1) ? __ldg(rn + (y1 + x.a1)) : bg4;
  const float wa = y.w0 * x.w0, wb = y.w0 * x.w1, wc = y.w1 * x.w0, wd = y.w1 * x.w1;
  constexpr int MO = DEPTH ? 8 : 6;  // channel of mask_observed; mask_rendered follows
  float v[DEPTH ? 16 : 8];
  // (img + mean) sampled with zero padding, then - mean, then the graph's /255.  The IEEE division is spelled out as
  // q = x * (1/255); q += (x - q * 255) * (1/255) with two fused multiply-adds: the correctly rounded quotient for every
  // |x| < 2^10 (exhaustively compared with x / 255.0f on 2e7 samples + all integer texels), at 3 instructions instead of ~10
  const float rcp255 = 1.0f / 255.0f;
  auto img = [&](float tl, float tr, float bl, float br, float m) -> float {
    const float s = fmaf(br, wd, fmaf(bl, wc, fmaf(tr, wb, tl * wa))) - m;
    const float q = s * rcp255;
    return fmaf(fmaf(-q, 255.0f, s), rcp255, q);
  };
  v[0] = img(O00.x, O01.x, O10.x, O11.x, p.mean[0]);
  v[1] = img(O00.y, O01.y, O10.y, O11.y, p.mean[1]);
  v[2] = img(O00.z, O01.z, O10.z, O11.z, p.mean[2]);
  v[3] = img(R00.x, R01.x, R10.x, R11.x, p.mean[0]);
  v[4] = img(R00.y, R01.y, R10.y, R11.y, p.mean[1]);
  v[5] = img(R00.z, R01.z, R10.z, R11.z, p.mean[2]);
  if constexpr (DEPTH) {
    v[6] = img(O00.w, O01.w, O10.w, O11.w, 0.f);
    v[7] = img(R00.w, R01.w, R10.w, R11.w, 0.f);
#pragma unroll
    for (int c = 10; c < 16; ++c) v[c] = 0.f;
  }
  if constexpr (!MASK) {
    v[MO] = v[MO + 1] = 0.f;
  } else {
    {  // observed mask = rectangle (an empty box has m0 > m1 on both axes)
      const float tl = (y.m0 && x.m0) ? 1.f : 0.f, tr = (y.m0 && x.m1) ? 1.f : 0.f;
      const float bl = (y.m1 && x.m0) ? 1.f : 0.f, br = (y.m1 && x.m1) ? 1.f : 0.f;
      v[MO] = roundf(fmaf(br, wd, fmaf(bl, wc, fmaf(tr, wb, tl * wa))));
    }
    {  // rendered mask, binarised at 0.2 (zoom_mask.py:39-41)
      const float tl = R00.w > 0.2f ? 1.f : 0.f, tr = R01.w > 0.2f ? 1.f : 0.f;
      const float bl = R10.w > 0.2f ? 1.f : 0.f, br = R11.w > 0.2f ? 1.f : 0.f;
      v[MO + 1] = roundf(fmaf(br, wd, fmaf(bl, wc, fmaf(tr, wb, tl * wa))));
    }
  }
  pack_chunk<LO, F16>(v, h[0], l[0]);
  if constexpr (DEPTH) pack_chunk<LO, F16>(v + 8, h[1], l[1]);
}

// one thread per space-to-depth pixel = a 2x2 quad of output pixels = the four 16-byte channel chunks
// of conv1's strip layout (consecutive threads write consecutive 16 B of each chunk plane); border
// slots are rewritten with zeros.  Sources are the pixel-interleaved float4 images, so each tap is one 16-byte load
// per image; the column taps of the quad's two columns and the row taps of its two rows are computed once each.
// DEPTH: the RGB-D network's input, two chunk planes per quad slot: [B*Hs rows][8 planes = (slot, half)][Ws cols][8 ch]
// Instance b's observed taps come from frame frame(b) of obs4 (dim_refine's frame map), its rendered taps from ren4[b].
template <bool LO, bool F16, bool DEPTH = false, bool MASK = true>
__global__ void __launch_bounds__(128, 8) zoom_fused_nhwc8_kernel(FusedZoomParams p) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= p.Hs * p.Ws) return;
  const int sr = q / p.Ws, sc = q - sr * p.Ws;
  const float4 z = __ldg(reinterpret_cast<const float4 *>(p.zoom_factor) + b);
  int4 bb = make_int4(1, 0, 1, 0);  // observed box (inclusive); empty: m0 > m1
  if (MASK) bb = __ldg(reinterpret_cast<const int4 *>(p.bbox8) + 2 * b);
  if (bb.y < 0) { bb.x = 1; bb.y = 0; bb.z = 1; bb.w = 0; }
  int4 vb = make_int4(0, p.W, 0, p.H);
  if (p.vbox) vb = __ldg(reinterpret_cast<const int4 *>(p.vbox) + b);
  const int i0 = 2 * sr - p.pad, j0 = 2 * sc - p.pad;
  AxisTap xt[2], yt[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    xt[k] = axis_tap(j0 + k, z.x, z.z, p.W, p.stepx, vb.x, vb.y, bb.x, bb.y);
    yt[k] = axis_tap(i0 + k, z.y, z.w, p.H, p.stepy, vb.z, vb.w, bb.z, bb.w);
  }
  const size_t P = (size_t)p.H * p.W;
  const FrameCams fc{p.frame_idx, nullptr, p.n_frames, {}};
  const float4 *ob = p.obs4 + (size_t)fc.frame(b) * P, *rn = p.ren4 + (size_t)b * P;
  // conv1 strip layout: [B*Hs rows][4 chunks (= quad slot)][Ws cols][8 ch] (DEPTH: 2 chunks per slot)
  constexpr int NC = DEPTH ? 2 : 1;
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    const int i = i0 + (s >> 1), j = j0 + (s & 1);
    uint4 h[NC], l[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) h[c] = l[c] = make_uint4(0u, 0u, 0u, 0u);  // zero bits are the same in both formats
    if (i >= 0 && i < p.H && j >= 0 && j < p.W) zoom_fused_pixel<LO, F16, DEPTH, MASK>(p, ob, rn, xt[s & 1], yt[s >> 1], h, l);
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const size_t o = ((((size_t)b * p.Hs + sr) * 4 * NC + s * NC + c) * p.Ws + sc) * 8;
      *reinterpret_cast<uint4 *>(p.hi + o) = h[c];
      if (LO) *reinterpret_cast<uint4 *>(p.lo + o) = l[c];
    }
  }
}

int zoom_fused_launch(dim_ctx *ctx, const float4 *obs4, const float4 *ren4, const float *zoom_factor,
                      const float *means_rgb, int B, int Hs, int Ws, int pad, __nv_bfloat16 *hi, __nv_bfloat16 *lo,
                      cudaStream_t st, int f16, const double *means_d, bool depth, bool mask, const FrameCams &cams) {
  FusedZoomParams p;
  p.obs4 = obs4; p.ren4 = ren4;
  // the frame map only: the kernel runs at its 64-register bound, and the whole FrameCams in its parameters makes it spill
  p.frame_idx = cams.frame_idx; p.n_frames = cams.n_frames;
  p.bbox8 = ctx->bbox8; p.zoom_factor = zoom_factor;
  p.vbox = means_d ? ctx->vbox : nullptr;  // means_d given: ren4 comes from the fused loop's box-only render
  for (int c = 0; c < 3; ++c) p.bg[c] = (means_d ? (float)(0.0 - means_d[c]) : 0.f) + means_rgb[c];
  p.H = ctx->H; p.W = ctx->W; p.Hs = Hs; p.Ws = Ws; p.pad = pad;
  for (int c = 0; c < 3; ++c) p.mean[c] = means_rgb[c];
  p.stepx = (float)(2.0 / (double)(ctx->W - 1));
  p.stepy = (float)(2.0 / (double)(ctx->H - 1));
  p.hi = hi; p.lo = lo;
  dim3 grid(cdiv(Hs * Ws, 128), B);
  DIM_REQUIRE(mask || !depth, "zoom_fused: the image-only network has no depth input");
  if (!mask) {
    if (f16) zoom_fused_nhwc8_kernel<false, true, false, false><<<grid, 128, 0, st>>>(p);
    else if (lo) zoom_fused_nhwc8_kernel<true, false, false, false><<<grid, 128, 0, st>>>(p);
    else zoom_fused_nhwc8_kernel<false, false, false, false><<<grid, 128, 0, st>>>(p);
  } else if (depth) {
    if (f16) zoom_fused_nhwc8_kernel<false, true, true><<<grid, 128, 0, st>>>(p);
    else if (lo) zoom_fused_nhwc8_kernel<true, false, true><<<grid, 128, 0, st>>>(p);
    else zoom_fused_nhwc8_kernel<false, false, true><<<grid, 128, 0, st>>>(p);
  } else if (f16) {
    zoom_fused_nhwc8_kernel<false, true><<<grid, 128, 0, st>>>(p);  // zero bits are the same in both formats
  } else if (lo) {
    zoom_fused_nhwc8_kernel<true, false><<<grid, 128, 0, st>>>(p);
  } else {
    zoom_fused_nhwc8_kernel<false, false><<<grid, 128, 0, st>>>(p);
  }
  DIM_LAUNCH_CHECK();
  return 0;
}

// RGB-D network: the observed depth into the w lanes of obs4 (constant over the iterations, like the image).  Device f32
// depth in metres, or the loader's uint16 file values converted as lib/utils/image.py:203,218 does: float32(u16) /
// float32(DEPTH_FACTOR) (a numpy float32 array divided by a Python float stays float32; IEEE division).
__global__ void __launch_bounds__(256) obs4_depth_kernel(float4 *obs4, int P, const float *depth, const uint16_t *depth_u16,
                                                         float factor) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= P) return;
  const size_t o = (size_t)b * P + q;
  reinterpret_cast<float *>(obs4 + o)[3] = depth ? depth[o] : __fdiv_rn((float)depth_u16[o], factor);
}
int obs4_depth_launch(dim_ctx *ctx, float4 *obs4, int B, const float *depth, const uint16_t *depth_u16, float factor,
                      cudaStream_t st) {
  const int P = ctx->H * ctx->W;
  obs4_depth_kernel<<<dim3(cdiv(P, 256), B), 256, 0, st>>>(obs4, P, depth, depth_u16, factor);
  DIM_LAUNCH_CHECK();
  return 0;
}

// NCHW f32 (3 planes, image - mean) -> pixel-interleaved float4 (x,y,z = plane + mean: the sampler's first step, w = 0):
// once per dim_refine call
__global__ void __launch_bounds__(256) pack_obs4_kernel(const float *img, int P, float4 *out, float m0, float m1, float m2) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= P) return;
  const float *s = img + (size_t)b * 3 * P;
  out[(size_t)b * P + q] = make_float4(s[q] + m0, s[P + q] + m1, s[2 * (size_t)P + q] + m2, 0.f);
}
int pack_obs4_launch(dim_ctx *ctx, const float *img, int B, float4 *out, const double *means, cudaStream_t st) {
  const int P = ctx->H * ctx->W;
  pack_obs4_kernel<<<dim3(cdiv(P, 256), B), 256, 0, st>>>(img, P, out, (float)means[0], (float)means[1], (float)means[2]);
  DIM_LAUNCH_CHECK();
  return 0;
}

// NCHW float32 zoomed blobs -> conv1 NHWC8 bf16 input (used by dim_net_fwd on the op surface); mo = mr = nullptr: the
// image-only network, whose channels 6-7 are zeros
__global__ void __launch_bounds__(256) pack_nhwc8_kernel(const float *io, const float *ir, const float *mo,
                                                         const float *mr, int H, int W, int Hs, int Ws, int pad,
                                                         __nv_bfloat16 *hi, __nv_bfloat16 *lo, int f16) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= H * W) return;
  const size_t P = (size_t)H * W;
  float v[8];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    v[c] = io[((size_t)b * 3 + c) * P + q] / 255.0f;
    v[3 + c] = ir[((size_t)b * 3 + c) * P + q] / 255.0f;
  }
  v[6] = mo ? mo[(size_t)b * P + q] : 0.f;
  v[7] = mr ? mr[(size_t)b * P + q] : 0.f;
  __align__(16) __nv_bfloat16 h[8];
  __align__(16) __nv_bfloat16 l[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    if (f16) {
      reinterpret_cast<__half *>(h)[c] = __float2half_rn(v[c]);
    } else {
      h[c] = __float2bfloat16_rn(v[c]);
      l[c] = __float2bfloat16_rn(v[c] - __bfloat162float(h[c]));
    }
  }
  const int oi = q / W + pad, oj = q % W + pad;
  const size_t o = ((((size_t)b * Hs + (oi >> 1)) * 4 + ((oi & 1) * 2 + (oj & 1))) * Ws + (oj >> 1)) * 8;
  *reinterpret_cast<uint4 *>(hi + o) = *reinterpret_cast<const uint4 *>(h);
  if (lo) *reinterpret_cast<uint4 *>(lo + o) = *reinterpret_cast<const uint4 *>(l);
}

int pack_nhwc8_launch(dim_ctx *ctx, const float *io, const float *ir, const float *mo, const float *mr, int B,
                      int Hs, int Ws, int pad, __nv_bfloat16 *hi, __nv_bfloat16 *lo, cudaStream_t st, int f16) {
  pack_nhwc8_kernel<<<dim3(cdiv(ctx->H * ctx->W, 256), B), 256, 0, st>>>(io, ir, mo, mr, ctx->H, ctx->W, Hs, Ws, pad,
                                                                         hi, f16 ? nullptr : lo, f16);
  DIM_LAUNCH_CHECK();
  return 0;
}

// NCHW float32 zoomed blobs + zoomed depths -> the RGB-D network's conv1 input (dim_net_fwd, training step): channels
// io/255, ir/255, do/255, dr/255, mo, mr in two 8-channel chunks per space-to-depth phase
__global__ void __launch_bounds__(256) pack_nhwc10_kernel(const float *io, const float *ir, const float *dobs,
                                                          const float *dren, const float *mo, const float *mr, int H, int W,
                                                          int Hs, int Ws, int pad, __nv_bfloat16 *hi, __nv_bfloat16 *lo,
                                                          int f16) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= H * W) return;
  const size_t P = (size_t)H * W;
  float v[16];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    v[c] = io[((size_t)b * 3 + c) * P + q] / 255.0f;
    v[3 + c] = ir[((size_t)b * 3 + c) * P + q] / 255.0f;
  }
  v[6] = dobs[(size_t)b * P + q] / 255.0f;
  v[7] = dren[(size_t)b * P + q] / 255.0f;
  v[8] = mo[(size_t)b * P + q];
  v[9] = mr[(size_t)b * P + q];
#pragma unroll
  for (int c = 10; c < 16; ++c) v[c] = 0.f;
  const int oi = q / W + pad, oj = q % W + pad;
  const int slot = (oi & 1) * 2 + (oj & 1);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    __align__(16) __nv_bfloat16 h[8];
    __align__(16) __nv_bfloat16 l[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float x = v[8 * half + c];
      if (f16) {
        reinterpret_cast<__half *>(h)[c] = __float2half_rn(x);
      } else {
        h[c] = __float2bfloat16_rn(x);
        l[c] = __float2bfloat16_rn(x - __bfloat162float(h[c]));
      }
    }
    const size_t o = ((((size_t)b * Hs + (oi >> 1)) * 8 + slot * 2 + half) * Ws + (oj >> 1)) * 8;
    *reinterpret_cast<uint4 *>(hi + o) = *reinterpret_cast<const uint4 *>(h);
    if (lo) *reinterpret_cast<uint4 *>(lo + o) = *reinterpret_cast<const uint4 *>(l);
  }
}

int pack_nhwc10_launch(dim_ctx *ctx, const float *io, const float *ir, const float *dobs, const float *dren, const float *mo,
                       const float *mr, int B, int Hs, int Ws, int pad, __nv_bfloat16 *hi, __nv_bfloat16 *lo, cudaStream_t st,
                       int f16) {
  pack_nhwc10_kernel<<<dim3(cdiv(ctx->H * ctx->W, 256), B), 256, 0, st>>>(io, ir, dobs, dren, mo, mr, ctx->H, ctx->W, Hs, Ws,
                                                                          pad, hi, f16 ? nullptr : lo, f16);
  DIM_LAUNCH_CHECK();
  return 0;
}

// GroupPicker (deepim/operator_py/group_picker.py:22-60): out[b] = in[b, g*cg:(g+1)*cg] with g = group_idx[b];
// backward scatters the gradient into the picked group and zero elsewhere.  n = elements per channel (H*W).
__global__ void __launch_bounds__(256) group_pick_kernel(const float *in, const float *group_idx, int B, int Ctot, int groups,
                                                         size_t n, float *out, int backward) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int cg = Ctot / groups;
  if (!backward) {
    if (i >= (size_t)B * cg * n) return;
    const int b = (int)(i / ((size_t)cg * n));
    const size_t r = i - (size_t)b * cg * n;
    const int g = (int)group_idx[b];
    // the reference asserts 0 <= g < group_num (group_picker.py:35); on the device an out-of-range index picks nothing
    out[i] = (g >= 0 && g < groups) ? in[((size_t)b * Ctot + (size_t)g * cg) * n + r] : 0.f;
  } else {
    if (i >= (size_t)B * Ctot * n) return;
    const int b = (int)(i / ((size_t)Ctot * n));
    const size_t r = i - (size_t)b * Ctot * n;
    const int c = (int)(r / n), g = (int)group_idx[b];
    out[i] = (g >= 0 && g < groups && c / cg == g) ? in[((size_t)b * cg + (c - g * cg)) * n + (r - (size_t)c * n)] : 0.f;
  }
}
int group_pick_launch(const float *in, const float *group_idx, int B, int Ctot, int groups, size_t n, float *out, int backward,
                      cudaStream_t st) {
  const size_t total = (size_t)B * (backward ? Ctot : Ctot / groups) * n;
  group_pick_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(in, group_idx, B, Ctot, groups, n, out, backward);
  DIM_LAUNCH_CHECK();
  return 0;
}

}  // namespace dim
