// train.cu -- the training step of the refiner network on the device (SURVEY 8 row a10, config C4):
// train-only decoder + heads + losses (deepim/symbols/deepIM_flownet.py:121-365), the backward pass of
// the whole graph, and the MXNet-SGD update (deepim/train.py:296-304; one update per inner iteration,
// deepim/core/module.py:1131-1137).
//
//   tensor-core work (wgmma + TMA):
//     forward   encoder convs (net.cu), deconv5 / deconv4 as 4 parity sub-convolutions (2x2 taps, stride-2 store)
//     dgrad     stride-1 layers: flipped-kernel convolution of dZ; stride-2 layers: 4 parity sub-convolutions;
//               deconvolutions: a stride-2 4x4 convolution of the (cropped) output gradient
//               -- all through conv_igemm_persistent_kernel<EPI = 1>, whose epilogue fuses "+ skip gradient" and
//               the LeakyReLU backward mask (sign of the stored activation) and stores bf16 dZ of the layer below
//     wgrad     conv_wgrad_kernel (MN-major operands, pixel index = contraction) + deterministic slice reduction
//   CUDA-core work: the 2-/1-channel flow / mask heads (Convolution1/2/3, mask_conv3, upsample_flow*), the fixed
//     bilinear 32x32 s16 upsampling + losses, fc6/fc7/rot/trans backward, bias gradients, SGD, weight repacking.
//
// Mixed precision: bf16 activations and activation gradients, fp32 accumulation, fp32 master weights /
// momentum / gradients (the flat parameter vector uses the MXNet layouts, order = param table below, so that the
// gradient all-reduce and checkpoints see the reference's tensors).
// Precision of the step (dim_train_set_precision): DIM_PREC_BF16 (default) as above, or DIM_PREC_BF16X3, in which every
// bf16 activation, activation gradient and operand pack is a hi / lo pair (x = hi + lo, ~16 significant bits): the
// tensor-core kernels run their SPLIT3 form (hi*hi + lo*hi + hi*lo) and the CUDA-core kernels below, templated on S3,
// read hi + lo and store pairs.  Their S3 = false instantiations are the bf16 step.
#include <string.h>

#include <algorithm>

#include "conv_wgrad.cuh"
#include "launch.cuh"
#include "net_state.cuh"

namespace dim {

// ------------------------------------------------------------------------------------ parameters
enum { PK_CONV = 0, PK_FC = 1, PK_DECONV = 2, PK_FROZEN = 3 };
struct ParamSpec {
  const char *name;
  int kind, d0, d1, k;  // conv (Cout,Cin,k,k) / fc (out,in) / deconv (Cin,Cout,k,k) / frozen (C,1,k,k)
};
static const ParamSpec kParams[24] = {
    {"flow_conv1", PK_CONV, 64, 8, 7},   {"conv2", PK_CONV, 128, 64, 5},    {"conv3", PK_CONV, 256, 128, 5},
    {"conv3_1", PK_CONV, 256, 256, 3},   {"conv4", PK_CONV, 512, 256, 3},   {"conv4_1", PK_CONV, 512, 512, 3},
    {"conv5", PK_CONV, 512, 512, 3},     {"conv5_1", PK_CONV, 512, 512, 3}, {"conv6", PK_CONV, 1024, 512, 3},
    {"conv6_1", PK_CONV, 1024, 1024, 3}, {"fc6", PK_FC, 256, 81920, 1},     {"fc7", PK_FC, 256, 256, 1},
    {"rot", PK_FC, 4, 256, 1},           {"trans", PK_FC, 3, 256, 1},
    {"Convolution1", PK_CONV, 2, 1024, 3}, {"deconv5", PK_DECONV, 1024, 512, 4}, {"upsample_flow6to5", PK_DECONV, 2, 2, 4},
    {"Convolution2", PK_CONV, 2, 1026, 3}, {"deconv4", PK_DECONV, 1026, 256, 4}, {"upsample_flow5to4", PK_DECONV, 2, 2, 4},
    {"Convolution3", PK_CONV, 2, 770, 3},  {"mask_conv3", PK_CONV, 1, 770, 3},
    {"upsampling", PK_FROZEN, 2, 1, 32},   {"mask_upsampling", PK_FROZEN, 1, 1, 32}};
enum { P_FC6 = 10, P_FC7 = 11, P_ROT = 12, P_TRANS = 13, P_CONV1D = 14, P_DECONV5 = 15, P_UP65 = 16, P_CONV2D = 17,
       P_DECONV4 = 18, P_UP54 = 19, P_CONV3D = 20, P_MASK3 = 21, P_UPS = 22, P_MUPS = 23 };

struct ParamOff { size_t w, b, wn, bn; };

// bf16 NHWC buffer with border; lo: its bf16x3 lo half (same layout), allocated by the first switch to that precision
struct Buf {
  __nv_bfloat16 *p = nullptr, *lo = nullptr;
  int H = 0, W = 0, Hp = 0, Wp = 0, py = 0, px = 0, C = 0;  // valid extent, allocated extent, border, channels
  size_t per_image() const { return (size_t)Hp * Wp * C; }
};

struct TrainMaps {
  // generic-kernel parameter blocks, one per launch
  ConvKParams deconv5_fwd[4], deconv4_fwd[4], deconv5_dgrad, deconv4_dgrad;
  LayerGeom g_deconv5_fwd[4], g_deconv4_fwd[4], g_deconv5_dgrad, g_deconv4_dgrad;
  ConvKParams dgrad[10][4];
  LayerGeom g_dgrad[10][4];
  int n_dgrad[10];
  WgradParams wg[10], wg_deconv5, wg_deconv4;
  int wg_bn[10], wg_bn_d5, wg_bn_d4;
};

struct TrainState {
  ParamOff off[24];
  size_t n_params = 0;
  float *master = nullptr, *mom = nullptr;
  Buf act10b, cat2, cat3, dcat2, dcat3, dA10p, gz[10], s2d32;
  Buf s2d64;         // RGB-D network: conv1's input as NHWC-64 (weight gradient operand)
  float *flow6 = nullptr, *flow5 = nullptr, *flow4 = nullptr, *mask4 = nullptr;
  float *dflow6 = nullptr, *dflow5 = nullptr, *dflow4 = nullptr, *dmask4 = nullptr;
  float *dfull = nullptr;        // [B][3][H][W] gradient wrt the full-resolution flow (2) / mask logit (1)
  float *loss_part = nullptr;    // [3][LOSS_BLOCKS]
  float *h6 = nullptr, *h7 = nullptr, *rot_raw = nullptr, *ztrans = nullptr, *rot_n = nullptr, *trans_est = nullptr;
  float *pts_est = nullptr, *dpts = nullptr, *drot_n = nullptr, *dtrans = nullptr, *drot = nullptr, *dh7 = nullptr, *dh6 = nullptr;
  float *bias_part = nullptr;    // [<= BIAS_CHUNKS][1088]
  float *thin_part = nullptr;    // [THIN_CHUNKS][2][1026*9]
  float *thin_w[4] = {};         // Convolution1/2/3, mask_conv3 as [tap][co][ci]
  float *wg_partial = nullptr;
  size_t wg_partial_elems = 0;
  // bf16 operand packs
  __nv_bfloat16 *dg_pack[10][4] = {};  // data-gradient kernels of encoder layers 1..9 (per parity class)
  __nv_bfloat16 *d5_fwd[4] = {}, *d4_fwd[4] = {}, *d5_dg = nullptr, *d4_dg = nullptr;
  // bf16x3 step (dim_train_set_precision): the lo halves of the packs above, allocated with the buffers' lo halves by the
  // first switch (fc6's lo pack is the inference one, NetState::fc6_w_lo)
  __nv_bfloat16 *dg_pack_lo[10][4] = {};
  __nv_bfloat16 *d5_fwd_lo[4] = {}, *d4_fwd_lo[4] = {}, *d5_dg_lo = nullptr, *d4_dg_lo = nullptr;
  bool s3 = false;        // the step runs in DIM_PREC_BF16X3
  bool lo_alloc = false;  // the lo halves exist
  std::map<int, TrainMaps> maps;  // per batch size (+ kS3MapKey for the bf16x3 launch descriptors)
  int max_points = 0;
  // internal streams: [0..2] run parity classes 1..3 next to class 0 on the caller's stream; [3] runs the weight / bias
  // gradients next to the data-gradient chain (both only read the dZ buffers)
  cudaStream_t side[4] = {};
  cudaEvent_t ev_phase[9] = {};  // phase boundaries of the last step on the caller's stream (dim_train_debug_phases)
  cudaEvent_t ev_fork = nullptr, ev_cls[3] = {}, ev_side = nullptr, ev_repack = nullptr;
};

static constexpr int LOSS_BLOCKS = 1024;
static constexpr int THIN_CHUNKS = 256;
static constexpr int BIAS_CHUNKS = 256;  // upper bound; the launch uses min(256, npix / 64) chunks
static constexpr int kS3MapKey = 1 << 20;

// ---------------------------------------------------------------------------------- small kernels
// a bf16 value of the step: hi, plus lo in bf16x3 (hi + lo is exact in fp32)
template <bool S3>
__device__ __forceinline__ float ld_pair(const __nv_bfloat16 *hi, const __nv_bfloat16 *lo, size_t i) {
  return S3 ? __bfloat162float(hi[i]) + __bfloat162float(lo[i]) : __bfloat162float(hi[i]);
}
// ... and its store: hi = bf16(v), in bf16x3 also lo = bf16(v - hi)
template <bool S3>
__device__ __forceinline__ void st_pair(__nv_bfloat16 *hi, __nv_bfloat16 *lo, size_t i, float v) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[i] = h;
  if (S3) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}

template <bool S3>
__global__ void __launch_bounds__(256) strip_to_nhwc32_kernel(const __nv_bfloat16 *src, const __nv_bfloat16 *src_lo, __nv_bfloat16 *dst,
                                                              __nv_bfloat16 *dst_lo, size_t n_chunks, int Ws) {
  // src [(b*Hs + r)][4][Ws][8] -> dst [(b*Hs + r)][Ws][32]; one 16-byte chunk per thread
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_chunks) return;
  const int col = (int)(i % Ws);
  const int chunk = (int)((i / Ws) % 4);
  const size_t row = i / ((size_t)Ws * 4);
  *reinterpret_cast<uint4 *>(dst + ((row * Ws + col) * 32 + chunk * 8)) = *reinterpret_cast<const uint4 *>(src + i * 8);
  if (S3) *reinterpret_cast<uint4 *>(dst_lo + ((row * Ws + col) * 32 + chunk * 8)) = *reinterpret_cast<const uint4 *>(src_lo + i * 8);
}

// RGB-D conv1 input: src [(b*Hs + r)][8][Ws][8] -> dst [(b*Hs + r)][Ws][64] (channel = phase*16 + c); one 16-byte chunk per thread
template <bool S3>
__global__ void __launch_bounds__(256) strip_to_nhwc64_kernel(const __nv_bfloat16 *src, const __nv_bfloat16 *src_lo, __nv_bfloat16 *dst,
                                                              __nv_bfloat16 *dst_lo, size_t n_chunks, int Ws) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_chunks) return;
  const int col = (int)(i % Ws);
  const int chunk = (int)((i / Ws) % 8);
  const size_t row = i / ((size_t)Ws * 8);
  *reinterpret_cast<uint4 *>(dst + ((row * Ws + col) * 64 + chunk * 8)) = *reinterpret_cast<const uint4 *>(src + i * 8);
  if (S3) *reinterpret_cast<uint4 *>(dst_lo + ((row * Ws + col) * 64 + chunk * 8)) = *reinterpret_cast<const uint4 *>(src_lo + i * 8);
}

// copy channels [0,C) of an NHWC buffer's valid region into another buffer (different border / channel stride)
template <bool S3>
__global__ void __launch_bounds__(256) copy_interior_kernel(const __nv_bfloat16 *src, const __nv_bfloat16 *src_lo, int sHp, int sWp, int spy,
                                                            int spx, int sC, __nv_bfloat16 *dst, __nv_bfloat16 *dst_lo, int dHp, int dWp,
                                                            int dpy, int dpx, int dC, int dcoff, int B, int H, int W, int C) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int c8n = C / 8;
  if (i >= (size_t)B * H * W * c8n) return;
  const int c8 = (int)(i % c8n);
  const int x = (int)((i / c8n) % W), y = (int)((i / ((size_t)c8n * W)) % H), b = (int)(i / ((size_t)c8n * W * H));
  const size_t si = (((size_t)b * sHp + y + spy) * sWp + x + spx) * sC + c8 * 8;
  const size_t di = (((size_t)b * dHp + y + dpy) * dWp + x + dpx) * dC + dcoff + c8 * 8;
  *reinterpret_cast<uint4 *>(dst + di) = *reinterpret_cast<const uint4 *>(src + si);
  if (S3) *reinterpret_cast<uint4 *>(dst_lo + di) = *reinterpret_cast<const uint4 *>(src_lo + si);
}

// g[c] *= (a[c] > 0 ? 1 : slope) over channels [coff, coff+C) of the valid region (LeakyReLU backward in place).  bf16x3: g is a
// pair; the activation's hi half alone decides the mask (hi + lo has the sign of hi, see store_pair_generic)
template <bool S3>
__global__ void __launch_bounds__(256) lrelu_mask_inplace_kernel(__nv_bfloat16 *g, __nv_bfloat16 *g_lo, const __nv_bfloat16 *a, int Hp,
                                                                 int Wp, int py, int px, int cs, int coff, int B, int H, int W, int C,
                                                                 float slope) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int c8n = C / 8;
  if (i >= (size_t)B * H * W * c8n) return;
  const int c8 = (int)(i % c8n);
  const int x = (int)((i / c8n) % W), y = (int)((i / ((size_t)c8n * W)) % H), b = (int)(i / ((size_t)c8n * W * H));
  const size_t o = (((size_t)b * Hp + y + py) * Wp + x + px) * cs + coff + c8 * 8;
  __align__(16) __nv_bfloat16 gv[8];
  __align__(16) __nv_bfloat16 gl[8];
  __align__(16) __nv_bfloat16 av[8];
  *reinterpret_cast<uint4 *>(gv) = *reinterpret_cast<const uint4 *>(g + o);
  if (S3) *reinterpret_cast<uint4 *>(gl) = *reinterpret_cast<const uint4 *>(g_lo + o);
  *reinterpret_cast<uint4 *>(av) = *reinterpret_cast<const uint4 *>(a + o);
#pragma unroll
  for (int e = 0; e < 8; ++e)
    if (!(__bfloat162float(av[e]) > 0.f)) st_pair<S3>(gv, gl, e, ld_pair<S3>(gv, gl, e) * slope);
  *reinterpret_cast<uint4 *>(g + o) = *reinterpret_cast<const uint4 *>(gv);
  if (S3) *reinterpret_cast<uint4 *>(g_lo + o) = *reinterpret_cast<const uint4 *>(gl);
}

// ---- thin 3x3 / pad 1 convolutions with <= 2 output channels (Convolution1/2/3, mask_conv3): CUDA cores
// forward: one 128-thread block per output pixel; the 4 warps split the input channels (warp w takes ci = w*32 + lane,
// + 128, ...) so the dependent-FMA chain per lane is 4x shorter than with one warp per pixel; fixed-order combine
template <int CO, bool S3>
__global__ void __launch_bounds__(128) thin_conv_fwd_kernel(const __nv_bfloat16 *x, const __nv_bfloat16 *x_lo, int Hp, int Wp, int cs,
                                                            int Cin, int B, int H, int W, const float *w, const float *bias, float *out) {
  __shared__ float red[4][CO];
  const int pix = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int xx = pix % W, yy = (pix / W) % H, b = pix / (W * H);
  float acc[CO];
#pragma unroll
  for (int co = 0; co < CO; ++co) acc[co] = 0.f;
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      const size_t px = (((size_t)b * Hp + yy + ky) * Wp + xx + kx) * cs;  // border 1 == pad 1
      for (int ci = threadIdx.x; ci < Cin; ci += 128) {
        const float v = ld_pair<S3>(x, x_lo, px + ci);
#pragma unroll
        for (int co = 0; co < CO; ++co) acc[co] = fmaf(v, w[((ky * 3 + kx) * CO + co) * Cin + ci], acc[co]);  // w = [tap][co][ci]
      }
    }
#pragma unroll
  for (int co = 0; co < CO; ++co) {
    float v = acc[co];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[warp][co] = v;
  }
  __syncthreads();
  if (threadIdx.x < CO) out[(size_t)pix * CO + threadIdx.x] = (((red[0][threadIdx.x] + red[1][threadIdx.x]) + red[2][threadIdx.x]) + red[3][threadIdx.x]) + bias[threadIdx.x];
}

// weight gradient, stage 1: thread (ci, tap) x pixel chunk blockIdx.y -> part[chunk][co][ci*9 + tap]
template <int CO, bool S3>
__global__ void __launch_bounds__(256) thin_conv_wgrad_kernel(const __nv_bfloat16 *x, const __nv_bfloat16 *x_lo, int Hp, int Wp, int cs,
                                                              int Cin, int B, int H, int W, const float *dy, float *part) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Cin * 9) return;
  const int ci = i % Cin, tap = i / Cin, ky = tap / 3, kx = tap % 3;
  const int npix = B * H * W, per = (npix + gridDim.y - 1) / gridDim.y;
  const int p0 = blockIdx.y * per, p1 = min(npix, p0 + per);
  float acc[CO];
#pragma unroll
  for (int co = 0; co < CO; ++co) acc[co] = 0.f;
  int xx = p0 % W, yy = (p0 / W) % H, b = p0 / (W * H);
  for (int p = p0; p < p1; ++p) {
    const float v = ld_pair<S3>(x, x_lo, (((size_t)b * Hp + yy + ky) * Wp + xx + kx) * cs + ci);
    const float *d = dy + (size_t)p * CO;
#pragma unroll
    for (int co = 0; co < CO; ++co) acc[co] = fmaf(v, d[co], acc[co]);
    if (++xx == W) { xx = 0; if (++yy == H) { yy = 0; ++b; } }
  }
#pragma unroll
  for (int co = 0; co < CO; ++co) part[((size_t)blockIdx.y * CO + co) * Cin * 9 + i] = acc[co];
}
// stage 2: fixed-order sum over the chunks, MXNet layout (co, ci, ky, kx); bias gradient by the last block
template <int CO>
__global__ void __launch_bounds__(256) thin_conv_wgrad_final_kernel(const float *part, int chunks, int Cin, const float *dy, int npix,
                                                                    float *dw, float *db) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < CO * Cin * 9) {
    const int co = i / (Cin * 9), r = i % (Cin * 9), ci = r % Cin, tap = r / Cin;
    float a = 0.f;
    for (int c = 0; c < chunks; ++c) a += part[((size_t)c * CO + co) * Cin * 9 + r];
    dw[(size_t)(co * Cin + ci) * 9 + tap] = a;
  }
  if (blockIdx.x == gridDim.x - 1) {
    __shared__ float red[256];
    for (int co = 0; co < CO; ++co) {
      float a = 0.f;
      for (int p = threadIdx.x; p < npix; p += 256) a += dy[(size_t)p * CO + co];
      red[threadIdx.x] = a;
      __syncthreads();
      for (int s = 128; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
      }
      if (threadIdx.x == 0) db[co] = red[0];
      __syncthreads();
    }
  }
}

// data gradient: one thread per (pixel, ci); writes (accumulate = 0) or adds to a bf16 NHWC buffer with border 1
template <int CO, bool S3>
__global__ void __launch_bounds__(256) thin_conv_dgrad_kernel(const float *dy, const float *w, int Cin, int B, int H, int W,
                                                              __nv_bfloat16 *dx, __nv_bfloat16 *dx_lo, int Hp, int Wp, int py, int px,
                                                              int cs, int c_write, int accumulate) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * H * W * c_write) return;
  const int ci = (int)(i % c_write);
  const int xx = (int)((i / c_write) % W), yy = (int)((i / ((size_t)c_write * W)) % H), b = (int)(i / ((size_t)c_write * W * H));
  float acc = 0.f;
  if (ci < Cin)
    for (int ky = 0; ky < 3; ++ky) {
      const int oy = yy + 1 - ky;
      if (oy < 0 || oy >= H) continue;
      for (int kx = 0; kx < 3; ++kx) {
        const int ox = xx + 1 - kx;
        if (ox < 0 || ox >= W) continue;
        const float *d = dy + ((size_t)(b * H + oy) * W + ox) * CO;
#pragma unroll
        for (int co = 0; co < CO; ++co) acc = fmaf(d[co], w[((ky * 3 + kx) * CO + co) * Cin + ci], acc);  // w = [tap][co][ci]
      }
    }
  const size_t o = (((size_t)b * Hp + yy + py) * Wp + xx + px) * cs + ci;
  if (accumulate) acc += ld_pair<S3>(dx, dx_lo, o);
  st_pair<S3>(dx, dx_lo, o, acc);
}

// ---- thin 2 -> 2 deconvolution k4 s2 + Crop(offset 1) (upsample_flow6to5 / 5to4)
template <bool S3>
__global__ void __launch_bounds__(256) thin_deconv_fwd_kernel(const float *in, int B, int Hi, int Wi, const float *w, const float *bias,
                                                              __nv_bfloat16 *out, __nv_bfloat16 *out_lo, int Hp, int Wp, int py, int px,
                                                              int cs, int coff, int Ho, int Wo) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * Ho * Wo * 2) return;
  const int co = i & 1, ox = (i >> 1) % Wo, oy = ((i >> 1) / Wo) % Ho, b = (i >> 1) / (Wo * Ho);
  float acc = bias[co];
  for (int ky = 0; ky < 4; ++ky) {
    const int t = oy + 1 - ky;  // full-resolution row oy+1 = 2*iy + ky
    if (t < 0 || (t & 1) || (t >> 1) >= Hi) continue;
    for (int kx = 0; kx < 4; ++kx) {
      const int u = ox + 1 - kx;
      if (u < 0 || (u & 1) || (u >> 1) >= Wi) continue;
      const float *p = in + ((size_t)(b * Hi + (t >> 1)) * Wi + (u >> 1)) * 2;
      acc = fmaf(p[0], w[((0 * 2 + co) * 4 + ky) * 4 + kx], acc);
      acc = fmaf(p[1], w[((1 * 2 + co) * 4 + ky) * 4 + kx], acc);
    }
  }
  st_pair<S3>(out, out_lo, (((size_t)b * Hp + oy + py) * Wp + ox + px) * cs + coff + co, acc);
}

// backward of the thin deconvolution: din (one thread per input pixel x ci)
template <bool S3>
__device__ __forceinline__ float thin_dY(const __nv_bfloat16 *dout, const __nv_bfloat16 *dout_lo, int Hp, int Wp, int py, int px, int cs,
                                         int coff, int Ho, int Wo, int b, int oy, int ox, int co) {
  if (oy < 0 || oy >= Ho || ox < 0 || ox >= Wo) return 0.f;
  return ld_pair<S3>(dout, dout_lo, (((size_t)b * Hp + oy + py) * Wp + ox + px) * cs + coff + co);
}
template <bool S3>
__global__ void __launch_bounds__(256) thin_deconv_bwd_kernel(const float *in, int B, int Hi, int Wi, const float *w,
                                                              const __nv_bfloat16 *dout, const __nv_bfloat16 *dout_lo, int Hp, int Wp,
                                                              int py, int px, int cs, int coff, int Ho, int Wo, float *din) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * Hi * Wi * 2) return;
  const int ci = i & 1, ix = (i >> 1) % Wi, iy = ((i >> 1) / Wi) % Hi, b = (i >> 1) / (Wi * Hi);
  float acc = 0.f;
  for (int ky = 0; ky < 4; ++ky)
    for (int kx = 0; kx < 4; ++kx)
      for (int co = 0; co < 2; ++co)
        acc = fmaf(thin_dY<S3>(dout, dout_lo, Hp, Wp, py, px, cs, coff, Ho, Wo, b, 2 * iy + ky - 1, 2 * ix + kx - 1, co),
                   w[((ci * 2 + co) * 4 + ky) * 4 + kx], acc);
  din[i] = acc;
}
// dw (64 values) and db (2 values): one block per output, threads stride over the pixels, fixed-order tree reduction
template <bool S3>
__global__ void __launch_bounds__(256) thin_deconv_wgrad_kernel(const float *in, int B, int Hi, int Wi, const __nv_bfloat16 *dout,
                                                                const __nv_bfloat16 *dout_lo, int Hp, int Wp, int py, int px, int cs,
                                                                int coff, int Ho, int Wo, float *dw, float *db) {
  __shared__ float red[256];
  const int t = blockIdx.x;  // 0..63: dw[((ci*2+co)*4+ky)*4+kx], 64..65: db[co]
  float acc = 0.f;
  if (t < 64) {
    const int kx = t & 3, ky = (t >> 2) & 3, co = (t >> 4) & 1, ci = t >> 5;
    for (int p = threadIdx.x; p < B * Hi * Wi; p += 256) {
      const int ix = p % Wi, iy = (p / Wi) % Hi, b = p / (Wi * Hi);
      acc = fmaf(in[(size_t)p * 2 + ci], thin_dY<S3>(dout, dout_lo, Hp, Wp, py, px, cs, coff, Ho, Wo, b, 2 * iy + ky - 1, 2 * ix + kx - 1, co),
                 acc);
    }
  } else {
    const int co = t - 64;
    for (int p = threadIdx.x; p < B * Ho * Wo; p += 256) {
      const int ox = p % Wo, oy = (p / Wo) % Ho, b = p / (Wo * Ho);
      acc += thin_dY<S3>(dout, dout_lo, Hp, Wp, py, px, cs, coff, Ho, Wo, b, oy, ox, co);
    }
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) { if (t < 64) dw[t] = red[0]; else db[t - 64] = red[0]; }
}

// ---- full-resolution heads: fixed bilinear Deconvolution k32 s16 (+ Crop offset 8), flow loss, mask loss
// (deepIM_flownet.py:184-208, 329-349).  One thread per output pixel; every output pixel has <= 2x2 sources.
// Writes flow_est (= flow_est_crop * NORMALIZE_FLOW), mask_prob, per-pixel gradients and loss partial sums.
__global__ void __launch_bounds__(256) fullres_loss_kernel(const float *flow4, const float *mask4, int h4, int w4, const float *wf,
                                                           const float *wm, const float *zflow, const float *zfw,
                                                           const float *mask_gt, int B, int H, int W, float norm_flow,
                                                           float gs_flow, float gs_mask, float *flow_est, float *mask_prob,
                                                           float *dfull, float *loss_part) {
  __shared__ float red[2][256];
  const size_t P = (size_t)H * W;
  float lf = 0.f, lm = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)B * P; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W), y = (int)((i / W) % H), b = (int)(i / P);
    const int Y = y + 8, X = x + 8;  // position in the un-cropped (in-1)*16+32 output
    float v[3] = {0.f, 0.f, 0.f};
    for (int iy = Y / 16 - 1; iy <= Y / 16; ++iy) {
      if (iy < 0 || iy >= h4) continue;
      const int ky = Y - 16 * iy;
      for (int ix = X / 16 - 1; ix <= X / 16; ++ix) {
        if (ix < 0 || ix >= w4) continue;
        const int kx = X - 16 * ix;
        const size_t s = (size_t)(b * h4 + iy) * w4 + ix;
        v[0] = fmaf(flow4[s * 2], wf[ky * 32 + kx], v[0]);
        v[1] = fmaf(flow4[s * 2 + 1], wf[1024 + ky * 32 + kx], v[1]);
        v[2] = fmaf(mask4[s], wm[ky * 32 + kx], v[2]);
      }
    }
    const size_t q = (size_t)y * W + x;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      if (zflow) {
        const float wgt = zfw[((size_t)b * 2 + c) * P + q];
        const float d = v[c] - zflow[((size_t)b * 2 + c) * P + q] / norm_flow;
        lf += wgt * d * d;
        dfull[((size_t)b * 3 + c) * P + q] = gs_flow * 2.f * wgt * d;
      }
      if (flow_est) flow_est[((size_t)b * 2 + c) * P + q] = v[c] * norm_flow;
    }
    const float pr = 1.f / (1.f + __expf(-v[2]));
    if (mask_gt) {
      const float lab = mask_gt[(size_t)b * P + q];
      // BCE with logits: max(x,0) - x*y + log(1 + exp(-|x|))
      lm += fmaxf(v[2], 0.f) - v[2] * lab + log1pf(__expf(-fabsf(v[2])));
      dfull[((size_t)b * 3 + 2) * P + q] = gs_mask * (pr - lab);
    }
    if (mask_prob) mask_prob[(size_t)b * P + q] = pr;
  }
  red[0][threadIdx.x] = lf;
  red[1][threadIdx.x] = lm;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) {
      red[0][threadIdx.x] += red[0][threadIdx.x + s];
      red[1][threadIdx.x] += red[1][threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    loss_part[blockIdx.x] = red[0][0];
    loss_part[LOSS_BLOCKS + blockIdx.x] = red[1][0];
  }
}

// gradient of the bilinear upsampling: d low-res (b, iy, ix, c) = sum over its 32x32 footprint; one warp per output
__global__ void __launch_bounds__(256) upsample_bwd_kernel(const float *dfull, const float *wf, const float *wm, int B, int H, int W,
                                                           int h4, int w4, float *dflow4, float *dmask4) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * h4 * w4 * 3) return;
  const int c = warp % 3, ix = (warp / 3) % w4, iy = (warp / (3 * w4)) % h4, b = warp / (3 * w4 * h4);
  const float *wk = c < 2 ? wf + c * 1024 : wm;
  const size_t P = (size_t)H * W;
  float acc = 0.f;
  for (int ky = 0; ky < 32; ++ky) {
    const int y = 16 * iy + ky - 8, x = 16 * ix + lane - 8;
    if (y < 0 || y >= H || x < 0 || x >= W) continue;
    acc = fmaf(dfull[((size_t)b * 3 + c) * P + (size_t)y * W + x], wk[ky * 32 + lane], acc);
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    const size_t s = (size_t)(b * h4 + iy) * w4 + ix;
    if (c < 2) dflow4[s * 2 + c] = acc; else dmask4[s] = acc;
  }
}

// ---- pose heads: L2Normalization, invZoomTrans, point-matching loss gradient (deepIM_flownet.py:217-316)
__global__ void pose_head_fwd_kernel(const float *rot_raw, const float *ztrans, const float *zoom_factor, int B, float *rot_n,
                                     float *trans_est) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float *r = rot_raw + 4 * b;
  const float n = sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3] + 1e-10f);
  for (int k = 0; k < 4; ++k) rot_n[4 * b + k] = r[k] / n;
  const float wx = zoom_factor[4 * b];
  trans_est[3 * b] = ztrans[3 * b] * wx;
  trans_est[3 * b + 1] = ztrans[3 * b + 1] * wx;
  trans_est[3 * b + 2] = ztrans[3 * b + 2];
}

__global__ void __launch_bounds__(256) pm_loss_kernel(const float *pts_est, const float *pts_obs, const float *pw, size_t n, float norm,
                                                      float gs, float *dpts, float *loss_part) {
  __shared__ float red[256];
  float l = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float d = (pts_est[i] - pts_obs[i]) / norm;
    l += pw[i] * fabsf(d);
    dpts[i] = gs * pw[i] * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) / norm;
  }
  red[threadIdx.x] = l;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss_part[2 * LOSS_BLOCKS + blockIdx.x] = red[0];
}

// one block of 256 threads: fixed-order tree reduction of the per-block partial sums (float64)
__global__ void __launch_bounds__(256) loss_final_kernel(const float *loss_part, int nb_full, int nb_pm, float gs_flow, float gs_pm,
                                                         float gs_mask, float *losses /*flow_sum, pm_sum, mask_bce_sum, objective*/) {
  __shared__ double red[3][256];
  double f = 0, m = 0, p = 0;
  for (int i = threadIdx.x; i < nb_full; i += 256) { f += loss_part[i]; m += loss_part[LOSS_BLOCKS + i]; }
  for (int i = threadIdx.x; i < nb_pm; i += 256) p += loss_part[2 * LOSS_BLOCKS + i];
  red[0][threadIdx.x] = f; red[1][threadIdx.x] = m; red[2][threadIdx.x] = p;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s)
      for (int k = 0; k < 3; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    f = red[0][0]; m = red[1][0]; p = red[2][0];
    losses[0] = (float)f; losses[1] = (float)p; losses[2] = (float)m;
    losses[3] = (float)(gs_flow * f + gs_pm * p + gs_mask * m);
  }
}

// backward of L2Normalization (d rot_raw) ; ZoomTrans backward with b_zoom_grad=False is the identity
__global__ void pose_head_bwd_kernel(const float *rot_raw, const float *rot_n, const float *drot_n, int B, float *drot) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float *r = rot_raw + 4 * b;
  const float n = sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3] + 1e-10f);
  float dot = 0.f;
  for (int k = 0; k < 4; ++k) dot += rot_n[4 * b + k] * drot_n[4 * b + k];
  for (int k = 0; k < 4; ++k) drot[4 * b + k] = (drot_n[4 * b + k] - rot_n[4 * b + k] * dot) / n;
}

// fc7 / rot / trans backward: block per instance -> dh7, dh6 (pre-activation gradients)
__global__ void __launch_bounds__(256) fc_heads_bwd_kernel(const float *drot, const float *dztrans, const float *rot_w,
                                                           const float *trans_w, const float *fc7_w /*(out,in)*/, const float *h6,
                                                           const float *h7, float *dh7, float *dh6) {
  __shared__ float g7[256];
  const int b = blockIdx.x, j = threadIdx.x;
  float a = 0.f;
  for (int k = 0; k < 4; ++k) a = fmaf(drot[4 * b + k], rot_w[k * 256 + j], a);
  for (int k = 0; k < 3; ++k) a = fmaf(dztrans[3 * b + k], trans_w[k * 256 + j], a);
  if (!(h7[b * 256 + j] > 0.f)) a *= 0.1f;
  g7[j] = a;
  dh7[b * 256 + j] = a;
  __syncthreads();
  float c = 0.f;
  for (int o = 0; o < 256; ++o) c = fmaf(g7[o], fc7_w[o * 256 + j], c);
  if (!(h6[b * 256 + j] > 0.f)) c *= 0.1f;
  dh6[b * 256 + j] = c;
}

// dW[o][k] = sum_b dy[b][o] * x[b][k], db[o] = sum_b dy[b][o]  (small fully-connected layers)
__global__ void __launch_bounds__(256) fc_wgrad_kernel(const float *dy, const float *x, int B, int O, int K, float *dw, float *db) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < O * K) {
    const int o = i / K, k = i % K;
    float a = 0.f;
    for (int b = 0; b < B; ++b) a = fmaf(dy[b * O + o], x[b * K + k], a);
    dw[i] = a;
  }
  if (i < O) {
    float a = 0.f;
    for (int b = 0; b < B; ++b) a += dy[b * O + i];
    db[i] = a;
  }
}

// fc6 weight gradient; the flat vector keeps fc6_weight as (256, h*10+w, c) -- the NHWC order of ReLU10 -- so both the
// activation reads and the gradient writes are coalesced (the host API permutes to MXNet's (256, c*80+hw) on load / get)
template <bool S3>
__global__ void __launch_bounds__(256) fc6_wgrad_kernel(const float *dh6, const __nv_bfloat16 *a10, const __nv_bfloat16 *a10_lo, int B,
                                                        float *dw) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // over 81920 / 2 pairs of k
  if (i >= 81920 / 2) return;
  float2 a[16];
#pragma unroll
  for (int b = 0; b < 16; ++b)
    if (b < B) {
      a[b] = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(a10 + (size_t)b * 81920 + 2 * i));
      if (S3) {
        const float2 l = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(a10_lo + (size_t)b * 81920 + 2 * i));
        a[b].x += l.x;
        a[b].y += l.y;
      }
    }
  for (int o = blockIdx.y * 32; o < blockIdx.y * 32 + 32; ++o) {
    float2 acc = make_float2(0.f, 0.f);
#pragma unroll
    for (int b = 0; b < 16; ++b)
      if (b < B) { const float d = dh6[b * 256 + o]; acc.x = fmaf(d, a[b].x, acc.x); acc.y = fmaf(d, a[b].y, acc.y); }
    *reinterpret_cast<float2 *>(dw + (size_t)o * 81920 + 2 * i) = acc;
  }
}
// fc6 data gradient, added to the bf16 partial gradient of ReLU10 ([B][80][1024]).  Block = 64 consecutive k (2 per lane),
// warp w streams output rows o in [32w, 32w+32) of the packed bf16 weight matrix; the 8 partial sums per (b, k) are
// combined through shared memory in fixed order.  bf16x3: the weights are w_hi + w_lo and dA is a pair.
template <bool S3>
__global__ void __launch_bounds__(256) fc6_dgrad_kernel(const float *dh6, const __nv_bfloat16 *w_hi /*[256][81920] packed*/,
                                                        const __nv_bfloat16 *w_lo, int B, __nv_bfloat16 *dA, __nv_bfloat16 *dA_lo) {
  __shared__ float red[8][16][64];
  __shared__ float dh[16][256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = blockIdx.x * 64 + 2 * lane;
  for (int i = threadIdx.x; i < 16 * 256; i += 256) dh[i >> 8][i & 255] = (i >> 8) < B ? dh6[i] : 0.f;
  __syncthreads();
  float2 acc[16];
#pragma unroll
  for (int b = 0; b < 16; ++b) acc[b] = make_float2(0.f, 0.f);
#pragma unroll 4
  for (int o = warp * 32; o < warp * 32 + 32; ++o) {
    float2 w = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(w_hi + (size_t)o * 81920 + k0));
    if (S3) {
      const float2 l = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(w_lo + (size_t)o * 81920 + k0));
      w.x += l.x;
      w.y += l.y;
    }
#pragma unroll
    for (int b = 0; b < 16; ++b) {
      const float d = dh[b][o];
      acc[b].x = fmaf(d, w.x, acc[b].x);
      acc[b].y = fmaf(d, w.y, acc[b].y);
    }
  }
#pragma unroll
  for (int b = 0; b < 16; ++b) {
    red[warp][b][2 * lane] = acc[b].x;
    red[warp][b][2 * lane + 1] = acc[b].y;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < B * 64; i += 256) {
    const int b = i >> 6, kk = i & 63;
    float s = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < 8; ++w8) s += red[w8][b][kk];
    const size_t o = (size_t)b * 81920 + blockIdx.x * 64 + kk;
    st_pair<S3>(dA, dA_lo, o, ld_pair<S3>(dA, dA_lo, o) + s);
  }
}

// bias gradient = per-channel sum over all pixels of a bf16 NHWC buffer (zero border included), two stages
template <bool S3>
__global__ void __launch_bounds__(256) bias_partial_kernel(const __nv_bfloat16 *g, const __nv_bfloat16 *g_lo, size_t npix, int cs, int coff,
                                                           int C, float *part) {
  const int c = blockIdx.x * 64 + (threadIdx.x & 63), lanep = threadIdx.x >> 6, chunk = blockIdx.y;
  __shared__ float red[4][64];
  const size_t per = (npix + gridDim.y - 1) / gridDim.y;
  const size_t p0 = (size_t)chunk * per, p1 = p0 + per < npix ? p0 + per : npix;
  float a = 0.f;
  if (c < C)
    for (size_t p = p0 + lanep; p < p1; p += 4) a += ld_pair<S3>(g, g_lo, p * cs + coff + c);
  red[lanep][threadIdx.x & 63] = a;
  __syncthreads();
  if (threadIdx.x < 64 && c < C)
    part[(size_t)chunk * 1088 + c] = (red[0][threadIdx.x] + red[1][threadIdx.x]) + (red[2][threadIdx.x] + red[3][threadIdx.x]);
}
__global__ void bias_final_kernel(const float *part, int chunks, int C, float *db) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a = 0.f;
  for (int k = 0; k < chunks; ++k) a += part[(size_t)k * 1088 + c];
  db[c] = a;
}

// MXNet SGD with momentum (train.py:296-304): mom = m*mom - lr*(rescale*g + wd*w); w += mom
// One launch over the flat vector: seg_end[s] = end offset of segment s (weight, bias, weight, bias, ...; 44 segments
// cover the 22 trainable tensors), even segments are weights (weight decay applies), odd ones biases (wd_mult = 0).
struct SgdSegs { unsigned long long end[44]; };
__global__ void __launch_bounds__(256) sgd_kernel(float *w, float *mom, const float *g, size_t n, const __grid_constant__ SgdSegs segs,
                                                  float lr, float momentum, float wd, float rescale) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int lo = 0, hi = 43;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (i < segs.end[mid]) hi = mid; else lo = mid + 1;
  }
  const float wdv = (lo & 1) ? 0.f : wd;
  const float m = momentum * mom[i] - lr * (rescale * g[i] + wdv * w[i]);
  mom[i] = m;
  w[i] += m;
}

// ---- weight repacking (fp32 master, MXNet layouts -> bf16 operand packs); the inference network's packs are net.cu's
// (net_pack_weights).  The packs are permutations of (Cout, Cin, k, k); a thread-per-destination gather reads the master
// with a k*k-float stride (every 4-byte read in its own sector).  The tiled kernels below read k*k-float rows (contiguous)
// into shared memory and write 64 consecutive bf16 per (tap, class): both sides coalesced.
//
// data-gradient packs of ALL parity classes of one layer: class (ry, rx) is [Cin][Ty][Tx][Cout] with ky = ry + s*(Ty-1-ty).
// block = (ci, 64 output channels): reads 64 rows of k*k floats, writes 64 consecutive bf16 per (class, tap)
// lo[c] = nullptr: no lo half (bf16 step); otherwise the bf16x3 residual pack of class c
struct DgradPackDst { __nv_bfloat16 *p[4], *lo[4]; };
__global__ void __launch_bounds__(256) pack_dgrad_kernel(const float *w, int Cout, int Cin, int k, int s, DgradPackDst dst) {
  __shared__ float tile[64 * 25];
  const int ci = blockIdx.x, co0 = blockIdx.y * 64, kk = k * k;
  for (int i = threadIdx.x; i < 64 * kk; i += 256) {
    const int col = i / kk, e = i - col * kk;
    tile[i] = w[((size_t)(co0 + col) * Cin + ci) * kk + e];
  }
  __syncthreads();
  const int ncls = s == 2 ? 4 : 1;
  for (int c = 0; c < ncls; ++c) {
    const int ry = c >> 1, rx = c & 1;
    const int Ty = s == 2 ? (k - ry + 1) / 2 : k, Tx = s == 2 ? (k - rx + 1) / 2 : k;
    for (int i = threadIdx.x; i < Ty * Tx * 64; i += 256) {
      const int tt = i >> 6, col = i & 63;
      const int ky = ry + s * (Ty - 1 - tt / Tx), kx = rx + s * (Tx - 1 - tt % Tx);
      store_split(dst.p[c], dst.lo[c], ((size_t)ci * Ty * Tx + tt) * Cout + co0 + col, tile[col * kk + ky * k + kx]);
    }
  }
}
// deconvolution forward, all 4 parity classes: class (ry, rx) is [Cout][2][2][Cin_eff], ky = ry + 2*(1 - ty); W (Cin,Cout,4,4).
// block = (co, 64 input channels)
__global__ void __launch_bounds__(256) pack_deconv_fwd_kernel(const float *w, int Cin, int Cout, int Cin_eff, DgradPackDst dst) {
  __shared__ float tile[64 * 16];
  const int co = blockIdx.x, c0 = blockIdx.y * 64;
  for (int i = threadIdx.x; i < 64 * 16; i += 256) {
    const int cl = i >> 4, e = i & 15;
    tile[i] = (c0 + cl < Cin) ? w[((size_t)(c0 + cl) * Cout + co) * 16 + e] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 4 * 4 * 64; i += 256) {
    const int cl = i & 63, t = (i >> 6) & 3, c = i >> 8;
    const int ky = (c >> 1) + 2 * (1 - t / 2), kx = (c & 1) + 2 * (1 - t % 2);
    if (c0 + cl < Cin_eff) store_split(dst.p[c], dst.lo[c], ((size_t)co * 4 + t) * Cin_eff + c0 + cl, tile[cl * 16 + ky * 4 + kx]);
  }
}
// deconvolution data gradient = stride-2 4x4 convolution: [Cin_eff][4][4][Cout]; block = one ci: Cout*16 contiguous floats in
__global__ void __launch_bounds__(256) pack_deconv_dgrad_kernel(const float *w, int Cin, int Cout, int Cin_eff, __nv_bfloat16 *dst,
                                                                __nv_bfloat16 *dst_lo) {
  extern __shared__ float dtile[];  // [Cout][17] (padded: the transposed read below would otherwise hit 2 banks)
  const int ci = blockIdx.x;
  for (int i = threadIdx.x; i < Cout * 16; i += 256) dtile[(i >> 4) * 17 + (i & 15)] = ci < Cin ? w[(size_t)ci * Cout * 16 + i] : 0.f;
  __syncthreads();
  for (int i = threadIdx.x; i < Cout * 16; i += 256) {
    const int co = i % Cout, tap = i / Cout;
    store_split(dst, dst_lo, ((size_t)ci * 16 + tap) * Cout + co, dtile[co * 17 + tap]);
  }
}
// thin-conv weights (CO, Cin, 3, 3) -> [tap][co][ci] fp32 so that lanes striding over ci read consecutive words
__global__ void __launch_bounds__(256) pack_thin_kernel(const float *w, int CO, int Cin, float *wt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= CO * Cin * 9) return;
  const int ci = i % Cin, co = (i / Cin) % CO, tap = i / (Cin * CO);
  wt[i] = w[((size_t)(co * Cin + ci)) * 9 + tap];
}

// ------------------------------------------------------------------------------------ host side
static size_t param_numel(const ParamSpec &s) { return (size_t)s.d0 * s.d1 * s.k * s.k; }
// the table entry of the RGB, the RGB-D or the image-only network: they differ only in flow_conv1's input channels (8 / 10 / 6)
static ParamSpec param_spec(int i, bool input_depth, bool input_mask = true) {
  ParamSpec s = kParams[i];
  if (i == 0 && input_depth) s.d1 = 10;
  if (i == 0 && !input_mask) s.d1 = 6;
  return s;
}
static size_t bias_numel(const ParamSpec &s) {
  if (s.kind == PK_FROZEN) return 0;
  return s.kind == PK_DECONV ? s.d1 : s.d0;
}

static int alloc_buf(dim_ctx *ctx, Buf &b, int B, int H, int W, int C, int border, bool even) {
  b.H = H; b.W = W; b.C = C; b.py = b.px = border;
  b.Hp = H + 2 * border; b.Wp = W + 2 * border;
  if (even) { b.Hp += b.Hp & 1; b.Wp += b.Wp & 1; }
  return dev_alloc(ctx, &b.p, b.per_image() * B, true);
}

static TrainState *&train_of(dim_ctx *ctx) {
  static std::map<dim_ctx *, TrainState *> table;  // contexts are created/destroyed from one host thread at a time
  return table[ctx];
}

int train_create(dim_ctx *ctx, int max_points) {
  NetState *ns = ctx->net;
  DIM_REQUIRE(ns && ns->net_ok, "dim_train_create: needs a 480x640 context");
  DIM_REQUIRE(train_of(ctx) == nullptr, "dim_train_create: already created");
  DIM_REQUIRE(ctx->max_batch <= 16, "dim_train_create: max_batch must be <= 16");
  TrainState *ts = new TrainState();
  train_of(ctx) = ts;
  ts->max_points = max_points;
  size_t off = 0;
  for (int i = 0; i < 24; ++i) {
    ts->off[i].w = off; ts->off[i].wn = param_numel(param_spec(i, ns->input_depth, ns->input_mask)); off += ts->off[i].wn;
    ts->off[i].b = off; ts->off[i].bn = bias_numel(kParams[i]); off += ts->off[i].bn;
  }
  ts->n_params = off;
  const int B = ctx->max_batch;
  int rc = 0;
  rc |= dev_alloc(ctx, &ts->master, off, true);
  rc |= dev_alloc(ctx, &ts->mom, off, true);
  const LayerGeom *g = ns->g;
  rc |= alloc_buf(ctx, ts->act10b, B, g[9].Ho, g[9].Wo, 1024, 1, false);
  rc |= alloc_buf(ctx, ts->cat2, B, g[7].Ho, g[7].Wo, 1088, 1, true);
  rc |= alloc_buf(ctx, ts->cat3, B, g[5].Ho, g[5].Wo, 832, 1, true);
  rc |= alloc_buf(ctx, ts->dcat2, B, g[7].Ho, g[7].Wo, 1088, 1, true);
  rc |= alloc_buf(ctx, ts->dcat3, B, g[5].Ho, g[5].Wo, 832, 1, true);
  rc |= alloc_buf(ctx, ts->dA10p, B, g[9].Ho, g[9].Wo, 1024, 0, false);
  for (int i = 0; i < 10; ++i) rc |= alloc_buf(ctx, ts->gz[i], B, g[i].Ho, g[i].Wo, g[i].Cout, 1, false);
  if (ns->input_depth) rc |= alloc_buf(ctx, ts->s2d64, B, g[0].rows, g[0].cols, 64, 0, false);
  else rc |= alloc_buf(ctx, ts->s2d32, B, g[0].rows, g[0].cols, 32, 0, false);
  const size_t n6 = (size_t)B * g[9].Ho * g[9].Wo, n5 = (size_t)B * g[7].Ho * g[7].Wo, n4 = (size_t)B * g[5].Ho * g[5].Wo;
  rc |= dev_alloc(ctx, &ts->flow6, n6 * 2, true); rc |= dev_alloc(ctx, &ts->dflow6, n6 * 2, true);
  rc |= dev_alloc(ctx, &ts->flow5, n5 * 2, true); rc |= dev_alloc(ctx, &ts->dflow5, n5 * 2, true);
  rc |= dev_alloc(ctx, &ts->flow4, n4 * 2, true); rc |= dev_alloc(ctx, &ts->dflow4, n4 * 2, true);
  rc |= dev_alloc(ctx, &ts->mask4, n4, true);     rc |= dev_alloc(ctx, &ts->dmask4, n4, true);
  rc |= dev_alloc(ctx, &ts->dfull, (size_t)B * 3 * ctx->H * ctx->W, true);
  rc |= dev_alloc(ctx, &ts->loss_part, (size_t)3 * LOSS_BLOCKS, true);
  rc |= dev_alloc(ctx, &ts->h6, (size_t)B * 256, true); rc |= dev_alloc(ctx, &ts->h7, (size_t)B * 256, true);
  rc |= dev_alloc(ctx, &ts->dh6, (size_t)B * 256, true); rc |= dev_alloc(ctx, &ts->dh7, (size_t)B * 256, true);
  rc |= dev_alloc(ctx, &ts->rot_raw, (size_t)B * 4, true); rc |= dev_alloc(ctx, &ts->ztrans, (size_t)B * 3, true);
  rc |= dev_alloc(ctx, &ts->rot_n, (size_t)B * 4, true); rc |= dev_alloc(ctx, &ts->trans_est, (size_t)B * 3, true);
  rc |= dev_alloc(ctx, &ts->drot_n, (size_t)B * 4, true); rc |= dev_alloc(ctx, &ts->dtrans, (size_t)B * 3, true);
  rc |= dev_alloc(ctx, &ts->drot, (size_t)B * 4, true);
  rc |= dev_alloc(ctx, &ts->pts_est, (size_t)B * 3 * max_points, true);
  rc |= dev_alloc(ctx, &ts->dpts, (size_t)B * 3 * max_points, true);
  rc |= dev_alloc(ctx, &ts->bias_part, (size_t)BIAS_CHUNKS * 1088, true);
  rc |= dev_alloc(ctx, &ts->thin_part, (size_t)THIN_CHUNKS * 2 * 1026 * 9, true);
  for (int i = 0; i < 4; ++i) rc |= dev_alloc(ctx, &ts->thin_w[i], (size_t)2 * 1026 * 9, true);
  // operand packs
  for (int i = 1; i < 10; ++i) {
    const LayerSpec &s = kLayers[i];
    const int ncls = s.stride == 2 ? 4 : 1;
    for (int c = 0; c < ncls; ++c) rc |= dev_alloc(ctx, &ts->dg_pack[i][c], (size_t)s.Cin * s.k * s.k * s.Cout, true);  // upper bound per class
  }
  for (int c = 0; c < 4; ++c) {
    rc |= dev_alloc(ctx, &ts->d5_fwd[c], (size_t)512 * 4 * 1024, true);
    rc |= dev_alloc(ctx, &ts->d4_fwd[c], (size_t)256 * 4 * 1088, true);
  }
  rc |= dev_alloc(ctx, &ts->d5_dg, (size_t)1024 * 16 * 512, true);
  rc |= dev_alloc(ctx, &ts->d4_dg, (size_t)1088 * 16 * 256, true);
  ts->wg_partial_elems = (size_t)24 << 20;  // 96 MB of fp32 partial tiles (largest layer: 9 taps x 1024 x 1024 = 9.4 M)
  rc |= dev_alloc(ctx, &ts->wg_partial, ts->wg_partial_elems, false);
  ns->save_h6 = ts->h6;
  ns->save_h7 = ts->h7;
  for (int i = 0; i < 4; ++i) DIM_CHECK(cudaStreamCreateWithFlags(&ts->side[i], cudaStreamNonBlocking));
  DIM_CHECK(cudaEventCreateWithFlags(&ts->ev_fork, cudaEventDisableTiming));
  DIM_CHECK(cudaEventCreateWithFlags(&ts->ev_side, cudaEventDisableTiming));
  DIM_CHECK(cudaEventCreateWithFlags(&ts->ev_repack, cudaEventDisableTiming));
  for (int i = 0; i < 3; ++i) DIM_CHECK(cudaEventCreateWithFlags(&ts->ev_cls[i], cudaEventDisableTiming));
  for (int i = 0; i < 9; ++i) DIM_CHECK(cudaEventCreate(&ts->ev_phase[i]));
  if (rc) {  // an allocation failed: leave no half-built state behind (the buffers themselves are owned by ctx)
    set_error("dim_train_create: device allocation failed (%d)", rc);
    train_destroy(ctx);
    return 12;
  }
  return 0;
}

void train_destroy(dim_ctx *ctx) {
  TrainState *&ts = train_of(ctx);
  if (ts) {
    for (int i = 0; i < 4; ++i) if (ts->side[i]) cudaStreamDestroy(ts->side[i]);
    if (ts->ev_fork) cudaEventDestroy(ts->ev_fork);
    if (ts->ev_side) cudaEventDestroy(ts->ev_side);
    if (ts->ev_repack) { ctx->net->repack_done = nullptr; cudaEventDestroy(ts->ev_repack); }
    for (int i = 0; i < 3; ++i) if (ts->ev_cls[i]) cudaEventDestroy(ts->ev_cls[i]);
    for (int i = 0; i < 9; ++i) if (ts->ev_phase[i]) cudaEventDestroy(ts->ev_phase[i]);
  }
  delete ts;
  ts = nullptr;
}

#define LAUNCH1D(kernel, n, st, ...)                                              \
  do {                                                                            \
    const size_t _n = (size_t)(n);                                                \
    if (_n) kernel<<<(unsigned)((_n + 255) / 256), 256, 0, st>>>(__VA_ARGS__);    \
    DIM_LAUNCH_CHECK();                                                           \
  } while (0)

// the master's conv1 ... conv6_1, fc6 and fc7 weights in net_pack_weights' order
static void master_weights(const TrainState *ts, const float *w[12]) {
  for (int i = 0; i < 12; ++i) w[i] = ts->master + ts->off[i].w;
}

// refresh every bf16 operand pack (and the fp32 head parameters of the inference net) from the master weights
// with_lo = false skips the bf16 'lo' halves (only the bf16x3 modes read them); they are then marked stale and refreshed
// lazily by train_refresh_lo() the next time the bf16x3 inference mode runs, or by the switch of the step to bf16x3.  The
// fp16 packs of DIM_PREC_FP16 are marked stale too: only that inference mode reads them, and train_refresh_f16() packs them
// from the master when it next runs
static int repack_all(dim_ctx *ctx, cudaStream_t st, bool with_lo) {
  TrainState *ts = train_of(ctx);
  const float *M = ts->master;
  const float *w[12];
  master_weights(ts, w);
  if (int rc = net_pack_weights(ctx, w, st, PACK_HI | (with_lo ? PACK_LO : 0u))) return rc;
  // the training packs' lo halves exist once the step has run in bf16x3 (nullptr before)
  auto L = [with_lo](__nv_bfloat16 *lo) { return with_lo ? lo : nullptr; };
  for (int i = 1; i < 10; ++i) {
    const LayerSpec &s = kLayers[i];
    DgradPackDst d{{ts->dg_pack[i][0], ts->dg_pack[i][1], ts->dg_pack[i][2], ts->dg_pack[i][3]},
                   {L(ts->dg_pack_lo[i][0]), L(ts->dg_pack_lo[i][1]), L(ts->dg_pack_lo[i][2]), L(ts->dg_pack_lo[i][3])}};
    pack_dgrad_kernel<<<dim3(s.Cin, s.Cout / 64), 256, 0, st>>>(M + ts->off[i].w, s.Cout, s.Cin, s.k, s.stride, d);
    DIM_LAUNCH_CHECK();
  }
  {
    DgradPackDst d5{{ts->d5_fwd[0], ts->d5_fwd[1], ts->d5_fwd[2], ts->d5_fwd[3]},
                    {L(ts->d5_fwd_lo[0]), L(ts->d5_fwd_lo[1]), L(ts->d5_fwd_lo[2]), L(ts->d5_fwd_lo[3])}};
    DgradPackDst d4{{ts->d4_fwd[0], ts->d4_fwd[1], ts->d4_fwd[2], ts->d4_fwd[3]},
                    {L(ts->d4_fwd_lo[0]), L(ts->d4_fwd_lo[1]), L(ts->d4_fwd_lo[2]), L(ts->d4_fwd_lo[3])}};
    pack_deconv_fwd_kernel<<<dim3(512, 1024 / 64), 256, 0, st>>>(M + ts->off[P_DECONV5].w, 1024, 512, 1024, d5);
    DIM_LAUNCH_CHECK();
    pack_deconv_fwd_kernel<<<dim3(256, 1088 / 64), 256, 0, st>>>(M + ts->off[P_DECONV4].w, 1026, 256, 1088, d4);
    DIM_LAUNCH_CHECK();
  }
  LAUNCH1D(pack_thin_kernel, 2 * 1024 * 9, st, M + ts->off[P_CONV1D].w, 2, 1024, ts->thin_w[0]);
  LAUNCH1D(pack_thin_kernel, 2 * 1026 * 9, st, M + ts->off[P_CONV2D].w, 2, 1026, ts->thin_w[1]);
  LAUNCH1D(pack_thin_kernel, 2 * 770 * 9, st, M + ts->off[P_CONV3D].w, 2, 770, ts->thin_w[2]);
  LAUNCH1D(pack_thin_kernel, 1 * 770 * 9, st, M + ts->off[P_MASK3].w, 1, 770, ts->thin_w[3]);
  pack_deconv_dgrad_kernel<<<1024, 256, 512 * 17 * 4, st>>>(M + ts->off[P_DECONV5].w, 1024, 512, 1024, ts->d5_dg, L(ts->d5_dg_lo));
  DIM_LAUNCH_CHECK();
  pack_deconv_dgrad_kernel<<<1088, 256, 256 * 17 * 4, st>>>(M + ts->off[P_DECONV4].w, 1026, 256, 1088, ts->d4_dg, L(ts->d4_dg_lo));
  DIM_LAUNCH_CHECK();
  return 0;
}

int train_load_params(dim_ctx *ctx, const float *flat_host, size_t n, cudaStream_t st) {
  TrainState *ts = train_of(ctx);
  NetState *ns = ctx->net;
  DIM_REQUIRE(ts != nullptr, "dim_train_load_params: dim_train_create has not been called");
  DIM_REQUIRE(n == ts->n_params, "dim_train_load_params: wrong parameter count");
  if (int rc = net_alloc_weights(ctx)) return rc;
  DIM_CHECK(cudaMemcpyAsync(ts->master, flat_host, n * sizeof(float), cudaMemcpyHostToDevice, st));
  DIM_CHECK(cudaMemsetAsync(ts->mom, 0, n * sizeof(float), st));
  // fp32 parameters that the kernels read as they are (biases, rot / trans heads) now alias the master vector, so an
  // update needs no copy for them; cached launch descriptors hold the old pointers -> rebuild them lazily
  ns->train_aliased = true;
  for (int i = 0; i < 10; ++i) ns->bias[i] = ts->master + ts->off[i].b;
  ns->fc6_b = ts->master + ts->off[P_FC6].b; ns->fc7_b = ts->master + ts->off[P_FC7].b;
  ns->rot_w = ts->master + ts->off[P_ROT].w; ns->rot_b = ts->master + ts->off[P_ROT].b;
  ns->trans_w = ts->master + ts->off[P_TRANS].w; ns->trans_b = ts->master + ts->off[P_TRANS].b;
  ns->maps.clear();
  ns->loaded = true;
  return repack_all(ctx, st, true);
}

// the per-batch-size launch descriptors are rebuilt on the next step (they hold the weight-gradient K-slice counts chosen
// for dim_ctx::num_sms); host-side parameter blocks only, so kernels already enqueued are unaffected
void train_drop_maps(dim_ctx *ctx) {
  if (TrainState *ts = train_of(ctx)) ts->maps.clear();
}

// a lazy refresh on the caller's stream st read the master: the next update's SGD must wait for it as for its own repack
static int refreshed_on(dim_ctx *ctx, TrainState *ts, cudaStream_t st) {
  DIM_CHECK(cudaEventRecord(ts->ev_repack, st));
  ctx->net->repack_done = ts->ev_repack;
  return 0;
}

// called by net_forward before a bf16x3 pass when the training step left the lo halves stale
int train_refresh_lo(dim_ctx *ctx, cudaStream_t st) {
  TrainState *ts = train_of(ctx);
  if (ts == nullptr) return 0;
  if (int rc = repack_all(ctx, st, true)) return rc;
  return refreshed_on(ctx, ts, st);
}

// called by net_forward before an fp16 pass after an update: the fp16 packs from the master, rounded once as dim_net_load
// rounds them, so a training context and an inference context loaded with its weights run the same fp16 network
int train_refresh_f16(dim_ctx *ctx, cudaStream_t st) {
  TrainState *ts = train_of(ctx);
  if (ts == nullptr) return 0;
  const float *w[12];
  master_weights(ts, w);
  if (int rc = net_pack_weights(ctx, w, st, PACK_F16)) return rc;
  return refreshed_on(ctx, ts, st);
}

// the lo halves of the step's bf16 buffers and of its operand packs (bf16x3); zero-filled, so borders and padding channels
// start (and stay) zero in both halves
static int alloc_lo(dim_ctx *ctx, TrainState *ts) {
  const int B = ctx->max_batch;
  int rc = 0;
  Buf *bufs[] = {&ts->act10b, &ts->cat2, &ts->cat3, &ts->dcat2, &ts->dcat3, &ts->dA10p, ctx->net->input_depth ? &ts->s2d64 : &ts->s2d32};
  for (Buf *b : bufs) rc |= dev_alloc(ctx, &b->lo, b->per_image() * B, true);
  for (int i = 0; i < 10; ++i) rc |= dev_alloc(ctx, &ts->gz[i].lo, ts->gz[i].per_image() * B, true);
  for (int i = 1; i < 10; ++i) {
    const LayerSpec &s = kLayers[i];
    for (int c = 0; c < (s.stride == 2 ? 4 : 1); ++c) {
      const int Ty = s.stride == 2 ? (s.k - (c >> 1) + 1) / 2 : s.k, Tx = s.stride == 2 ? (s.k - (c & 1) + 1) / 2 : s.k;
      rc |= dev_alloc(ctx, &ts->dg_pack_lo[i][c], (size_t)s.Cin * Ty * Tx * s.Cout, true);  // exact class size
    }
  }
  for (int c = 0; c < 4; ++c) {
    rc |= dev_alloc(ctx, &ts->d5_fwd_lo[c], (size_t)512 * 4 * 1024, true);
    rc |= dev_alloc(ctx, &ts->d4_fwd_lo[c], (size_t)256 * 4 * 1088, true);
  }
  rc |= dev_alloc(ctx, &ts->d5_dg_lo, (size_t)1024 * 16 * 512, true);
  rc |= dev_alloc(ctx, &ts->d4_dg_lo, (size_t)1088 * 16 * 256, true);
  if (rc) {
    set_error("dim_train_set_precision: device allocation failed (%d)", rc);
    return 12;
  }
  ts->lo_alloc = true;
  return 0;
}

int train_set_precision(dim_ctx *ctx, int precision) {
  TrainState *ts = train_of(ctx);
  DIM_REQUIRE(ts != nullptr, "dim_train_set_precision: call dim_train_create first");
  DIM_REQUIRE(precision == DIM_PREC_BF16 || precision == DIM_PREC_BF16X3,
              "dim_train_set_precision: the training step runs in DIM_PREC_BF16 or DIM_PREC_BF16X3");
  const bool s3 = precision == DIM_PREC_BF16X3;
  if (s3 == ts->s3) return 0;
  if (s3) {
    // not on the hot path: wait for every stream of the context, allocate once, then bring every lo half up to the master
    // weights (updates made in bf16 left them stale)
    DIM_CHECK(cudaDeviceSynchronize());
    if (!ts->lo_alloc)
      if (int rc = alloc_lo(ctx, ts)) return rc;
    if (ctx->net->loaded && ctx->net->train_aliased) {
      if (int rc = repack_all(ctx, ts->side[3], true)) return rc;
      DIM_CHECK(cudaStreamSynchronize(ts->side[3]));
    }
  }
  ts->s3 = s3;
  return 0;
}

int train_get_precision(dim_ctx *ctx, int *precision) {
  TrainState *ts = train_of(ctx);
  DIM_REQUIRE(ts != nullptr, "dim_train_get_precision: call dim_train_create first");
  *precision = ts->s3 ? DIM_PREC_BF16X3 : DIM_PREC_BF16;
  return 0;
}

int train_get_params(dim_ctx *ctx, float *flat_host, size_t n, int which, cudaStream_t st) {
  TrainState *ts = train_of(ctx);
  DIM_REQUIRE(ts != nullptr && n == ts->n_params, "dim_train_get_params: bad state or size");
  DIM_CHECK(cudaMemcpyAsync(flat_host, which ? ts->mom : ts->master, n * sizeof(float), cudaMemcpyDeviceToHost, st));
  DIM_CHECK(cudaStreamSynchronize(st));
  return 0;
}

size_t train_param_count(dim_ctx *ctx) { TrainState *ts = train_of(ctx); return ts ? ts->n_params : 0; }
int train_param_info(int idx, const char **name, long long *w_numel, long long *b_numel, bool input_depth, bool input_mask) {
  if (idx < 0 || idx >= 24) return 1;
  const ParamSpec s = param_spec(idx, input_depth, input_mask);
  *name = s.name; *w_numel = (long long)param_numel(s); *b_numel = (long long)bias_numel(s);
  return 0;
}

// ------------------------------------------------------------------------ generic conv launches
static void pick_tile(int W, int rows_total, int cap, int &BW, int &BH, int max_bw = 1 << 30, int max_bh = 1 << 30) {
  // power-of-two BW x BH = cap rectangle with the least padding; prefer TMA boxes inside the tensor extents
  for (int pass = 0; pass < 2; ++pass) {
    long best = -1;
    for (int bw = 1; bw <= cap; bw <<= 1) {
      const int bh = cap / bw;
      if (pass == 0 && (bw > max_bw || bh > max_bh)) continue;
      const long cost = (long)cdiv(W, bw) * bw * cdiv(rows_total, bh) * bh;
      if (best < 0 || cost < best || (cost == best && bw > BW)) { best = cost; BW = bw; BH = bh; }
    }
    if (best >= 0) return;
  }
}

template <int BN, int ST, bool S3 = false>
static int launch_generic(const ConvKParams &kp, int total_tiles, int n_tiles, int cap, cudaStream_t st) {
  using S = ConvSmem2<BN, ST, S3, 1>;
  static bool attr_set = false;
  if (!attr_set) {
    DIM_CHECK(cudaFuncSetAttribute(conv_igemm_persistent_kernel<BN, ST, S3, false, 1>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    attr_set = true;
  }
  const int grid = total_tiles < cap ? total_tiles : cap;
  conv_igemm_persistent_kernel<BN, ST, S3, false, 1><<<grid, 384, S::TOTAL, st>>>(kp, total_tiles, n_tiles);
  DIM_LAUNCH_CHECK();
  return 0;
}

// one CTA per SM with the deepest ring that fits (STAGES x stage bytes <= 192 KB; bf16x3 stages hold hi and lo operands)
static int run_generic(dim_ctx *ctx, const ConvKParams &kp, const LayerGeom &g, int B, cudaStream_t st, bool s3) {
  const int n_tiles = cdiv(g.Cout, g.BLOCK_N);
  const int total = cdiv(B * g.Hq, g.BH) * g.n_col_tiles * n_tiles;
  const int sms = ctx->num_sms;
  if (s3) {
    if (g.BLOCK_N == 256) return launch_generic<256, 2, true>(kp, total, n_tiles, sms, st);
    if (g.BLOCK_N == 128) return launch_generic<128, 3, true>(kp, total, n_tiles, sms, st);
    return launch_generic<64, 4, true>(kp, total, n_tiles, sms, st);
  }
  if (g.BLOCK_N == 256) return launch_generic<256, 4>(kp, total, n_tiles, sms, st);
  if (g.BLOCK_N == 128) return launch_generic<128, 6>(kp, total, n_tiles, sms, st);
  return launch_generic<64, 8>(kp, total, n_tiles, sms, st);
}

// Describe one launch of the generic kernel.
//   in      : bf16 NHWC input buffer (border included), channels [in_coff, in_coff + K_ch) are the K range
//   stride2 : read through the 4 parity views (k4 s2 convolution), else stride-1 taps with (off_r, off_c)
//   w, w_lo : [N][KH*KW][K_ch] bf16 pack and its lo half
//   out     : output buffer; virtual pixel (oh, ow) -> interior (oh*sy + oy, ow*sx + ox)
//   s3      : bf16x3 (SPLIT3): also the lo maps of the input and the weights, the lo halves of out and addend
static int make_generic(ConvKParams &kp, LayerGeom &g, int B, const Buf &in, int in_coff, int K_ch, bool stride2, int KH, int KW,
                        int off_r, int off_c, int Ho, int Wo, const __nv_bfloat16 *w, const __nv_bfloat16 *w_lo, int N,
                        const float *bias, float slope, const Buf &out, int out_coff, int sy, int sx, int oy, int ox,
                        const Buf *addend, int add_coff, const Buf *mask, int mask_coff, int mask_climit, bool s3) {
  memset(&kp, 0, sizeof(kp));
  memset(&g, 0, sizeof(g));
  g.Cout = N; g.KH = KH; g.KW = KW; g.BLOCK_K = 64;
  g.BLOCK_N = (N % 256 == 0) ? 256 : ((N % 128 == 0) ? 128 : 64);
  g.Hq = stride2 ? in.Hp / 2 : in.Hp;
  pick_tile(Wo, B * g.Hq, 128, g.BW, g.BH, stride2 ? in.Wp / 2 : in.Wp, B * g.Hq);
  g.n_col_tiles = cdiv(Wo, g.BW);
  g.kblocks = KH * KW * (K_ch / 64);
  const uint32_t box[3] = {64u, (uint32_t)g.BW, (uint32_t)g.BH};
  for (int lo = 0; lo < (s3 ? 2 : 1); ++lo) {
    __nv_bfloat16 *base = lo ? in.lo : in.p;
    CUtensorMap *a_map = lo ? kp.a_lo_map : kp.a_map;
    if (!stride2) {
      const uint64_t dims[3] = {(uint64_t)K_ch, (uint64_t)in.Wp, (uint64_t)B * in.Hp};
      const uint64_t str[2] = {(uint64_t)in.C * 2, (uint64_t)in.Wp * in.C * 2};
      if (int rc = encode_map(&a_map[0], base + in_coff, 3, dims, str, box, 64)) return rc;
      a_map[1] = a_map[2] = a_map[3] = a_map[0];
    } else {
      for (int ph = 0; ph < 2; ++ph)
        for (int pw = 0; pw < 2; ++pw) {
          const uint64_t dims[3] = {(uint64_t)K_ch, (uint64_t)in.Wp / 2, (uint64_t)B * in.Hp / 2};
          const uint64_t str[2] = {(uint64_t)2 * in.C * 2, (uint64_t)2 * in.Wp * in.C * 2};
          if (int rc = encode_map(&a_map[(ph << 1) | pw], base + ((size_t)ph * in.Wp + pw) * in.C + in_coff, 3, dims, str, box, 64))
            return rc;
        }
    }
    const uint64_t Ktot = (uint64_t)KH * KW * K_ch;
    const uint64_t dims[2] = {Ktot, (uint64_t)N};
    const uint64_t str[1] = {Ktot * 2};
    const uint32_t boxw[2] = {64u, (uint32_t)g.BLOCK_N};
    if (int rc = encode_map(lo ? &kp.b_lo_map : &kp.b_map, const_cast<__nv_bfloat16 *>(lo ? w_lo : w), 2, dims, str, boxw, 64)) return rc;
  }
  kp.KH = KH; kp.KW = KW; kp.stride = stride2 ? 2 : 1; kp.cchunks = K_ch / 64;
  kp.BW = g.BW; kp.BH = g.BH; kp.n_col_tiles = g.n_col_tiles;
  kp.Hq = g.Hq; kp.Ho = Ho; kp.Wo = Wo; kp.Bn = B;
  kp.out_Hp = out.Hp; kp.out_Wp = out.Wp; kp.out_py = out.py; kp.out_px = out.px; kp.Cout = N;
  kp.kblocks = g.kblocks;
  kp.slope = slope; kp.bias = bias; kp.out_hi = out.p; kp.out_lo = s3 ? out.lo : nullptr;
  kp.in_off_r = off_r; kp.in_off_c = off_c;
  kp.out_sy = sy; kp.out_sx = sx; kp.out_oy = oy; kp.out_ox = ox; kp.out_H = out.H; kp.out_W = out.W;
  kp.out_cs = out.C; kp.out_coff = out_coff;
  if (addend) kp.addend = {addend->p, addend->Hp, addend->Wp, addend->py, addend->px, addend->C, add_coff, s3 ? addend->lo : nullptr};
  if (mask) kp.mask = {mask->p, mask->Hp, mask->Wp, mask->py, mask->px, mask->C, mask_coff, nullptr};  // hi decides the sign
  kp.mask_climit = mask_climit;
  return 0;
}

// ------------------------------------------------------------------------------ wgrad launches
template <int BN, int ST, bool S3 = false>
static int launch_wgrad(const WgradParams &p, cudaStream_t st) {
  using S = WgradSmem<BN, ST, S3>;
  static bool attr_set = false;
  if (!attr_set) {
    DIM_CHECK(cudaFuncSetAttribute(conv_wgrad_kernel<BN, ST, S3>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    attr_set = true;
  }
  const int grid = p.KH * p.KW * p.m_tiles * p.n_tiles * p.kslices;
  conv_wgrad_kernel<BN, ST, S3><<<grid, 384, S::TOTAL, st>>>(p);
  DIM_LAUNCH_CHECK();
  return 0;
}

static int encode_map4(CUtensorMap *m, __nv_bfloat16 *base, uint64_t C, uint64_t cols, uint64_t rows, uint64_t B, uint64_t pix_stride,
                       uint64_t row_stride, uint64_t img_stride, uint32_t boxc, uint32_t bw, uint32_t bh) {
  const uint64_t dims[4] = {C, cols, rows, B};
  const uint64_t str[3] = {pix_stride * 2, row_stride * 2, img_stride * 2};
  const uint32_t box[4] = {boxc, bw, bh, 1};
  return encode_map(m, base, 4, dims, str, box, boxc == 32 ? 32 : 64);
}

// Z: M-side buffer (channels [z_coff, z_coff+M)), iterated over its valid H x W region; A: N-side buffer, read at
// (y*s + kh, x*s + kw) in ITS bordered coordinates (+ a_off); bf16x3 (ts->s3): also the maps of both lo halves
static int make_wgrad(TrainState *ts, WgradParams &p, int &BN, int B, const Buf &Z, int z_coff, int M, int H, int W, const Buf &A,
                      int a_coff, int N, int stride, int KH, int KW, int a_off_r, int a_off_c, int sms) {
  memset(&p, 0, sizeof(p));
  BN = N >= 256 ? 256 : (N >= 128 ? 128 : (N >= 64 ? 64 : 32));
  p.KH = KH; p.KW = KW; p.stride = stride;
  pick_tile(W, H, 64, p.BW, p.BH, std::min(Z.Wp, stride == 2 ? A.Wp / 2 : A.Wp), std::min(Z.Hp, stride == 2 ? A.Hp / 2 : A.Hp));
  p.rects_x = cdiv(W, p.BW); p.rects_y = cdiv(H, p.BH); p.Bn = B;
  p.z_off_r = Z.py; p.z_off_c = Z.px; p.a_off_r = a_off_r; p.a_off_c = a_off_c;
  p.m_tiles = cdiv(M, 128); p.n_tiles = cdiv(N, BN);
  p.kb_total = B * p.rects_x * p.rects_y;
  const int tiles = KH * KW * p.m_tiles * p.n_tiles;
  // K slices: one CTA per SM is resident (~192 KB ring), so pick the slice count whose CTA total fills whole waves of `sms`
  // best (e.g. 25 tiles: 11 slices = 275 CTAs = 2 waves at 93 %, where 12 slices = 300 CTAs would need a third wave)
  const size_t per_slice = (size_t)KH * KW * p.m_tiles * 128 * p.n_tiles * BN;
  int ks = 1;
  double best = -1.0;
  for (int c = 1; c <= 24 && c <= (p.kb_total + 1) / 2 && per_slice * c <= ts->wg_partial_elems; ++c) {
    const int ctas = tiles * c;
    if (c > 1 && ctas > 2 * sms) break;  // at most two waves: more slices only add fp32 partial traffic
    const double eff = (double)ctas / ((double)cdiv(ctas, sms) * sms) - 0.004 * c + (ctas >= sms ? 0.0 : -0.5);
    if (eff > best + 1e-12) { best = eff; ks = c; }
  }
  DIM_REQUIRE(per_slice * ks <= ts->wg_partial_elems, "wgrad workspace too small");
  p.kb_per_slice = cdiv(p.kb_total, ks);
  p.kslices = cdiv(p.kb_total, p.kb_per_slice);
  p.partial = ts->wg_partial;
  const uint32_t boxc = BN >= 64 ? 64 : 32;
  for (int lo = 0; lo < (ts->s3 ? 2 : 1); ++lo) {
    __nv_bfloat16 *zb = lo ? Z.lo : Z.p, *ab = lo ? A.lo : A.p;
    CUtensorMap *a_map = lo ? p.a_lo_map : p.a_map;
    if (int rc = encode_map4(lo ? &p.z_lo_map : &p.z_map, zb + z_coff, M, Z.Wp, Z.Hp, B, Z.C, (uint64_t)Z.Wp * Z.C,
                             (uint64_t)Z.Hp * Z.Wp * Z.C, 64, p.BW, p.BH))
      return rc;
    if (stride == 1) {
      if (int rc = encode_map4(&a_map[0], ab + a_coff, N, A.Wp, A.Hp, B, A.C, (uint64_t)A.Wp * A.C, (uint64_t)A.Hp * A.Wp * A.C, boxc,
                               p.BW, p.BH))
        return rc;
      a_map[1] = a_map[2] = a_map[3] = a_map[0];
    } else {
      for (int ph = 0; ph < 2; ++ph)
        for (int pw = 0; pw < 2; ++pw)
          if (int rc = encode_map4(&a_map[(ph << 1) | pw], ab + ((size_t)ph * A.Wp + pw) * A.C + a_coff, N, A.Wp / 2, A.Hp / 2, B,
                                   (uint64_t)2 * A.C, (uint64_t)2 * A.Wp * A.C, (uint64_t)A.Hp * A.Wp * A.C, boxc, p.BW, p.BH))
            return rc;
    }
  }
  return 0;
}

static int run_wgrad(const WgradParams &p, int BN, bool s3, int kind, int D0, int D1, int k, float *grad, cudaStream_t st) {
  int rc;
  // one CTA per SM, ring depth = what fits in ~192 KB of shared memory (bf16x3: a stage holds the hi and the lo operands)
  if (s3) {
    if (BN == 256) rc = launch_wgrad<256, 2, true>(p, st);
    else if (BN == 128) rc = launch_wgrad<128, 3, true>(p, st);
    else if (BN == 64) rc = launch_wgrad<64, 4, true>(p, st);
    else rc = launch_wgrad<32, 5, true>(p, st);
  } else if (BN == 256) rc = launch_wgrad<256, 4>(p, st);
  else if (BN == 128) rc = launch_wgrad<128, 6>(p, st);
  else if (BN == 64) rc = launch_wgrad<64, 8>(p, st);
  else rc = launch_wgrad<32, 8>(p, st);
  if (rc) return rc;
  const size_t total = (size_t)p.KH * p.KW * p.m_tiles * 128 * p.n_tiles * BN;
  wgrad_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(p.partial, p.kslices, p.KH * p.KW, p.m_tiles * 128,
                                                                        p.n_tiles * BN, kind, D0, D1, k, grad);
  DIM_LAUNCH_CHECK();
  return 0;
}

// conv1: one GEMM per filter row (conv1_wgrad_kernel); p was built by make_wgrad for the 16-tap form, only the slicing differs
template <int ST, bool S3>
static int launch_wgrad_conv1(const WgradParams &p, cudaStream_t st) {
  using S = Conv1WgradSmem<ST, S3>;
  static bool attr_set = false;
  if (!attr_set) {
    DIM_CHECK(cudaFuncSetAttribute(conv1_wgrad_kernel<ST, S3>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    attr_set = true;
  }
  conv1_wgrad_kernel<ST, S3><<<4 * p.kslices, 384, S::TOTAL, st>>>(p);
  DIM_LAUNCH_CHECK();
  return 0;
}
// conv1_wgrad_kernel's K slicing of the batch's pixel blocks: cdiv(2 sms, 4) slices of 4 filter-row CTAs each
static WgradParams conv1_slicing(const dim_ctx *ctx, const WgradParams &p16) {
  WgradParams p = p16;
  int ks = cdiv(2 * ctx->num_sms, 4);
  if (ks > p.kb_total / 2) ks = p.kb_total / 2;
  if (ks < 1) ks = 1;
  p.kb_per_slice = cdiv(p.kb_total, ks);
  p.kslices = cdiv(p.kb_total, p.kb_per_slice);
  return p;
}
static int run_wgrad_conv1(dim_ctx *ctx, TrainState *ts, const WgradParams &p16, float *grad, cudaStream_t st) {
  const WgradParams p = conv1_slicing(ctx, p16);
  DIM_REQUIRE((size_t)p.kslices * 4 * 128 * 64 <= ts->wg_partial_elems, "wgrad workspace too small");
  if (int rc = ts->s3 ? launch_wgrad_conv1<4, true>(p, st) : launch_wgrad_conv1<8, false>(p, st)) return rc;
  const size_t total = (size_t)4 * 128 * 64;
  // the image-only network's gradient is (64, 6, 7, 7): D1 = 6 drops the rows of the zero mask lanes
  wgrad_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(p.partial, p.kslices, 4, 128, 64, WG_CONV1_ROW, 64,
                                                                       ctx->net->input_mask ? 8 : 6, 7, grad);
  DIM_LAUNCH_CHECK();
  return 0;
}

static int bias_grad(TrainState *ts, const Buf &g, int B, int coff, int C, float *db, cudaStream_t st) {
  const size_t npix = (size_t)B * g.Hp * g.Wp;
  int chunks = (int)(npix / 64);
  chunks = chunks < 1 ? 1 : (chunks > BIAS_CHUNKS ? BIAS_CHUNKS : chunks);
  (ts->s3 ? bias_partial_kernel<true> : bias_partial_kernel<false>)<<<dim3(cdiv(C, 64), chunks), 256, 0, st>>>(g.p, g.lo, npix, g.C, coff,
                                                                                                            C, ts->bias_part);
  DIM_LAUNCH_CHECK();
  bias_final_kernel<<<cdiv(C, 256), 256, 0, st>>>(ts->bias_part, chunks, C, db);
  DIM_LAUNCH_CHECK();
  return 0;
}

template <int CO>
static int thin_wgrad(TrainState *ts, const Buf &x, int Cin, int B, int H, int W, const float *dy, float *dw, float *db, cudaStream_t st) {
  const int npix = B * H * W;
  int chunks = npix / 32;
  chunks = chunks < 1 ? 1 : (chunks > THIN_CHUNKS ? THIN_CHUNKS : chunks);
  (ts->s3 ? thin_conv_wgrad_kernel<CO, true> : thin_conv_wgrad_kernel<CO, false>)<<<dim3(cdiv(Cin * 9, 256), chunks), 256, 0, st>>>(
      x.p, x.lo, x.Hp, x.Wp, x.C, Cin, B, H, W, dy, ts->thin_part);
  DIM_LAUNCH_CHECK();
  thin_conv_wgrad_final_kernel<CO><<<cdiv(CO * Cin * 9, 256) + 1, 256, 0, st>>>(ts->thin_part, chunks, Cin, dy, npix, dw, db);
  DIM_LAUNCH_CHECK();
  return 0;
}

static int thin_deconv_bwd(const float *in, int B, int Hi, int Wi, const float *w, const Buf &dout, int coff, int Ho, int Wo, float *din,
                           float *dw, float *db, cudaStream_t st, cudaStream_t sw, TrainState *ts) {
  (ts->s3 ? thin_deconv_bwd_kernel<true> : thin_deconv_bwd_kernel<false>)<<<cdiv(B * Hi * Wi * 2, 256), 256, 0, st>>>(
      in, B, Hi, Wi, w, dout.p, dout.lo, dout.Hp, dout.Wp, dout.py, dout.px, dout.C, coff, Ho, Wo, din);
  DIM_LAUNCH_CHECK();
  DIM_CHECK(cudaEventRecord(ts->ev_fork, st));  // dout is final on st; the weight gradient is off the critical path
  DIM_CHECK(cudaStreamWaitEvent(sw, ts->ev_fork, 0));
  (ts->s3 ? thin_deconv_wgrad_kernel<true> : thin_deconv_wgrad_kernel<false>)<<<66, 256, 0, sw>>>(
      in, B, Hi, Wi, dout.p, dout.lo, dout.Hp, dout.Wp, dout.py, dout.px, dout.C, coff, Ho, Wo, dw, db);
  DIM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------ per-batch-size maps
static Buf act_buf(const NetState *ns, int i) {  // act[i] as a Buf (input of encoder layer i; 10 = ReLU10, no border)
  Buf b;
  if (i < 10) {
    const LayerGeom &g = ns->g[i];
    b.p = ns->act_hi[i]; b.lo = ns->act_lo[i]; b.Hp = g.rows; b.Wp = g.cols; b.py = g.py; b.px = g.px; b.C = g.Cbuf; b.H = g.Hin; b.W = g.Win;
  } else {
    const LayerGeom &g = ns->g[9];
    b.p = ns->act_hi[10]; b.lo = ns->act_lo[10]; b.Hp = g.Ho; b.Wp = g.Wo; b.py = b.px = 0; b.C = g.Cout; b.H = g.Ho; b.W = g.Wo;
  }
  return b;
}

static int build_train_maps(dim_ctx *ctx, int B, TrainMaps &tm) {
  NetState *ns = ctx->net;
  TrainState *ts = train_of(ctx);
  const float *M = ts->master;
  const int sms = ctx->num_sms;
  const bool s3 = ts->s3;
  // decoder forward: 4 parity classes each; output pixel = 2q + r - 1 (Crop offset 1)
  for (int c = 0; c < 4; ++c) {
    const int ry = c >> 1, rx = c & 1;
    if (int rc = make_generic(tm.deconv5_fwd[c], tm.g_deconv5_fwd[c], B, ts->act10b, 0, 1024, false, 2, 2, 0, 0, ts->act10b.H + 1,
                              ts->act10b.W + 1, ts->d5_fwd[c], ts->d5_fwd_lo[c], 512, M + ts->off[P_DECONV5].b, 0.1f, ts->cat2, 512, 2, 2,
                              ry - 1, rx - 1, nullptr, 0, nullptr, 0, 0, s3))
      return rc;
    if (int rc = make_generic(tm.deconv4_fwd[c], tm.g_deconv4_fwd[c], B, ts->cat2, 0, 1088, false, 2, 2, 0, 0, ts->cat2.H + 1,
                              ts->cat2.W + 1, ts->d4_fwd[c], ts->d4_fwd_lo[c], 256, M + ts->off[P_DECONV4].b, 0.1f, ts->cat3, 512, 2, 2,
                              ry - 1, rx - 1, nullptr, 0, nullptr, 0, 0, s3))
      return rc;
  }
  // decoder data gradients (stride-2 4x4 convolutions of the bordered output-gradient canvases)
  {
    const Buf a10 = act_buf(ns, 10);
    if (int rc = make_generic(tm.deconv5_dgrad, tm.g_deconv5_dgrad, B, ts->dcat2, 512, 512, true, 4, 4, 0, 0, ts->act10b.H, ts->act10b.W,
                              ts->d5_dg, ts->d5_dg_lo, 1024, nullptr, 0.1f, ts->gz[9], 0, 1, 1, 0, 0, &ts->dA10p, 0, &a10, 0, 1024, s3))
      return rc;
    if (int rc = make_generic(tm.deconv4_dgrad, tm.g_deconv4_dgrad, B, ts->dcat3, 512, 256, true, 4, 4, 0, 0, ts->cat2.H, ts->cat2.W,
                              ts->d4_dg, ts->d4_dg_lo, 1088, nullptr, 1.0f, ts->dcat2, 0, 1, 1, 0, 0, nullptr, 0, nullptr, 0, 0, s3))
      return rc;
  }
  // encoder data gradients, layers 9..1 -> gz[i-1]
  for (int i = 1; i < 10; ++i) {
    const LayerSpec &s = kLayers[i];
    const LayerGeom &lg = ns->g[i];
    const Buf ai = act_buf(ns, i);
    const Buf *addend = (i == 8) ? &ts->dcat2 : ((i == 6) ? &ts->dcat3 : nullptr);
    tm.n_dgrad[i] = s.stride == 2 ? 4 : 1;
    for (int c = 0; c < tm.n_dgrad[i]; ++c) {
      const int ry = c >> 1, rx = c & 1;
      int Ty, Tx, offr, offc, oy, ox, sy, Jy, Jx;
      if (s.stride == 2) {
        Ty = (s.k - ry + 1) / 2; Tx = (s.k - rx + 1) / 2;
        const int qy = (s.pad - ry + 1) >> 1, qx = (s.pad - rx + 1) >> 1;
        offr = qy + 2 - Ty; offc = qx + 2 - Tx;
        oy = 2 * qy + ry - s.pad; ox = 2 * qx + rx - s.pad;
        sy = 2;
        Jy = cdiv(lg.Hin - oy, 2); Jx = cdiv(lg.Win - ox, 2);
      } else {
        Ty = Tx = s.k; offr = offc = 0; oy = ox = 0; sy = 1; Jy = lg.Hin; Jx = lg.Win;
      }
      if (int rc = make_generic(tm.dgrad[i][c], tm.g_dgrad[i][c], B, ts->gz[i], 0, s.Cout, false, Ty, Tx, offr, offc, Jy, Jx,
                                ts->dg_pack[i][c], ts->dg_pack_lo[i][c], s.Cin, nullptr, 0.1f, ts->gz[i - 1], 0, sy, sy, oy, ox, addend, 0,
                                &ai, 0, s.Cin, s3))
        return rc;
    }
  }
  // weight gradients
  for (int i = 0; i < 10; ++i) {
    const LayerSpec &s = kLayers[i];
    if (i == 0 && ns->input_depth) {  // generic kernel over the 16 taps of the NHWC-64 copy (SW128 boxes), WG_CONV1_RGBD reduce
      if (int rc = make_wgrad(ts, tm.wg[0], tm.wg_bn[0], B, ts->gz[0], 0, 64, ns->g[0].Ho, ns->g[0].Wo, ts->s2d64, 0, 64, 1, 4, 4, 0, 0, sms))
        return rc;
    } else if (i == 0) {
      if (int rc = make_wgrad(ts, tm.wg[0], tm.wg_bn[0], B, ts->gz[0], 0, 64, ns->g[0].Ho, ns->g[0].Wo, ts->s2d32, 0, 32, 1, 4, 4, 0, 0, sms))
        return rc;
    } else {
      const Buf ai = act_buf(ns, i);
      if (int rc = make_wgrad(ts, tm.wg[i], tm.wg_bn[i], B, ts->gz[i], 0, s.Cout, ns->g[i].Ho, ns->g[i].Wo, ai, 0, s.Cin, s.stride, s.k,
                              s.k, 0, 0, sms))
        return rc;
    }
  }
  if (int rc = make_wgrad(ts, tm.wg_deconv5, tm.wg_bn_d5, B, ts->act10b, 0, 1024, ts->act10b.H, ts->act10b.W, ts->dcat2, 512, 512, 2, 4, 4, 0, 0, sms))
    return rc;
  if (int rc = make_wgrad(ts, tm.wg_deconv4, tm.wg_bn_d4, B, ts->cat2, 0, 1088, ts->cat2.H, ts->cat2.W, ts->dcat3, 512, 256, 2, 4, 4, 0, 0, sms))
    return rc;
  return 0;
}

static int copy_interior(const Buf &src, Buf &dst, int dcoff, int B, int C, cudaStream_t st, bool s3) {
  const size_t n = (size_t)B * src.H * src.W * (C / 8);
  (s3 ? copy_interior_kernel<true> : copy_interior_kernel<false>)<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
      src.p, src.lo, src.Hp, src.Wp, src.py, src.px, src.C, dst.p, dst.lo, dst.Hp, dst.Wp, dst.py, dst.px, dst.C, dcoff, B, src.H, src.W, C);
  DIM_LAUNCH_CHECK();
  return 0;
}

// the parity classes of one layer write disjoint pixels: class 0 on the caller's stream, 1..3 on internal streams
static int run_classes(dim_ctx *ctx, TrainState *ts, const ConvKParams *kp, const LayerGeom *g, int n, int B, cudaStream_t st) {
  // classes that fill the machine on their own gain nothing from running side by side: keep them on one stream
  const int tiles0 = cdiv(B * g[0].Hq, g[0].BH) * g[0].n_col_tiles * cdiv(g[0].Cout, g[0].BLOCK_N);
  if (n == 1 || tiles0 >= ctx->num_sms) {
    for (int c = 0; c < n; ++c)
      if (int rc = run_generic(ctx, kp[c], g[c], B, st, ts->s3)) return rc;
    return 0;
  }
  DIM_CHECK(cudaEventRecord(ts->ev_fork, st));
  for (int c = 1; c < n; ++c) {
    DIM_CHECK(cudaStreamWaitEvent(ts->side[c - 1], ts->ev_fork, 0));
    if (int rc = run_generic(ctx, kp[c], g[c], B, ts->side[c - 1], ts->s3)) return rc;
    DIM_CHECK(cudaEventRecord(ts->ev_cls[c - 1], ts->side[c - 1]));
  }
  if (int rc = run_generic(ctx, kp[0], g[0], B, st, ts->s3)) return rc;
  for (int c = 1; c < n; ++c) DIM_CHECK(cudaStreamWaitEvent(st, ts->ev_cls[c - 1], 0));
  return 0;
}
// everything enqueued on `st` so far becomes visible to the weight-gradient stream
static int fork_side(TrainState *ts, cudaStream_t st) {
  DIM_CHECK(cudaEventRecord(ts->ev_fork, st));
  DIM_CHECK(cudaStreamWaitEvent(ts->side[3], ts->ev_fork, 0));
  return 0;
}

// ------------------------------------------------------------------------------------ the step
static int record_buckets(const TrainIO &io, int lo_inclusive, int hi_exclusive, cudaStream_t s) {
  for (int k = 0; k < io.n_buckets; ++k)
    if (io.bucket_first_tensor[k] >= lo_inclusive && io.bucket_first_tensor[k] < hi_exclusive)
      DIM_CHECK(cudaEventRecord((cudaEvent_t)io.bucket_events[k], s));
  return 0;
}

// test hook: the K slicing of the 12 weight gradients (flow_conv1, conv2 ... conv6_1, deconv5, deconv4) of a B-image step at
// the current SM count and precision; out36[3 g ...] = slices, pixel blocks per slice (the K range one fp32 accumulator sums,
// 64 pixels a block), pixel blocks in all
int train_debug_wgrad_slices(dim_ctx *ctx, int B, int *out36) {
  TrainState *ts = train_of(ctx);
  DIM_REQUIRE(ts != nullptr && ctx->net->loaded, "dim_train_debug_wgrad_slices: call dim_train_create / dim_train_load_params first");
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch, "dim_train_debug_wgrad_slices: bad batch size");
  const int key = B + (ts->s3 ? kS3MapKey : 0);
  auto it = ts->maps.find(key);
  if (it == ts->maps.end()) {
    TrainMaps tm;
    if (int rc = build_train_maps(ctx, B, tm)) return rc;
    it = ts->maps.emplace(key, tm).first;
  }
  const TrainMaps &tm = it->second;
  for (int g = 0; g < 12; ++g) {
    WgradParams p = g < 10 ? tm.wg[g] : (g == 10 ? tm.wg_deconv5 : tm.wg_deconv4);
    if (g == 0 && !ctx->net->input_depth) p = conv1_slicing(ctx, p);
    out36[3 * g] = p.kslices; out36[3 * g + 1] = p.kb_per_slice; out36[3 * g + 2] = p.kb_total;
  }
  return 0;
}

int train_forward_backward(dim_ctx *ctx, const TrainIO &io, cudaStream_t st) {
  NetState *ns = ctx->net;
  TrainState *ts = train_of(ctx);
  DIM_REQUIRE(ts != nullptr && ns->loaded, "dim_train_forward_backward: call dim_train_create / dim_train_load_params first");
  const int B = io.B, H = ctx->H, W = ctx->W;
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch && io.N >= 0 && io.N <= ts->max_points, "dim_train_forward_backward: bad batch / point count");
  const bool labels = io.zflow && io.zfw && io.zmask_gt && io.src_pose && io.pc_model && io.pc_weights && io.pc_observed && io.N >= 1;
  DIM_REQUIRE(labels || io.grads == nullptr, "dim_train_forward_backward: the backward pass needs every label");
  DIM_REQUIRE(labels || (!io.zflow && !io.zfw && !io.zmask_gt && !io.pc_model), "dim_train_forward_backward: pass all labels or none");
  const bool s3 = ts->s3;
  const int key = B + (s3 ? kS3MapKey : 0);
  auto it = ts->maps.find(key);
  if (it == ts->maps.end()) {
    TrainMaps tm;
    if (int rc = build_train_maps(ctx, B, tm)) return rc;
    it = ts->maps.emplace(key, tm).first;
  }
  const TrainMaps &tm = it->second;
  const float *M = ts->master;
  float *G = io.grads;
  const LayerGeom *g = ns->g;
  const int h6 = g[9].Ho, w6 = g[9].Wo, h5 = g[7].Ho, w5 = g[7].Wo, h4 = g[5].Ho, w4 = g[5].Wo;
  const dim_train_config &cfg = ctx->cfg;
  const float gs_flow = cfg.lw_flow / (float)(H * W), gs_mask = cfg.lw_mask / (float)(H * W), gs_pm = cfg.lw_pm / cfg.num_3d_sample;
  const float *Tm = cfg.trans_means, *Tsd = cfg.trans_stds;

  // ---------------- forward
  DimNvtxRange r_fwd("dim_train forward + losses");
  DIM_CHECK(cudaEventRecord(ts->ev_phase[0], st));
  DIM_REQUIRE((io.zdo && io.zdr) == ns->input_depth && (io.zdo == nullptr) == (io.zdr == nullptr),
              "dim_train_forward_backward: the RGB-D network takes both zoomed depths, the RGB network none");
  if (ns->input_depth) {
    if (int rc = pack_nhwc10_launch(ctx, io.zio, io.zir, io.zdo, io.zdr, io.zmo, io.zmr, B, g[0].rows, g[0].cols, g[0].py, ns->act_hi[0],
                                    s3 ? ns->act_lo[0] : nullptr, st, 0))
      return rc;
  } else if (int rc = pack_nhwc8_launch(ctx, io.zio, io.zir, ns->input_mask ? io.zmo : nullptr, ns->input_mask ? io.zmr : nullptr,
                                        B, g[0].rows, g[0].cols, g[0].py, ns->act_hi[0],
                                        s3 ? ns->act_lo[0] : nullptr, st, 0)) {
    return rc;
  }
  if (int rc = net_forward(ctx, B, s3 ? DIM_PREC_BF16X3 : DIM_PREC_BF16, nullptr, ts->rot_raw, ts->ztrans, nullptr, st, nullptr)) return rc;
  DIM_CHECK(cudaEventRecord(ts->ev_phase[1], st));
  const Buf a10 = act_buf(ns, 10), a8 = act_buf(ns, 8), a6 = act_buf(ns, 6);
  auto thin_fwd2 = s3 ? thin_conv_fwd_kernel<2, true> : thin_conv_fwd_kernel<2, false>;
  auto thin_fwd1 = s3 ? thin_conv_fwd_kernel<1, true> : thin_conv_fwd_kernel<1, false>;
  auto thin_deconv_fwd = s3 ? thin_deconv_fwd_kernel<true> : thin_deconv_fwd_kernel<false>;
  if (int rc = copy_interior(a10, ts->act10b, 0, B, 1024, st, s3)) return rc;
  thin_fwd2<<<B * h6 * w6, 128, 0, st>>>(ts->act10b.p, ts->act10b.lo, ts->act10b.Hp, ts->act10b.Wp, 1024, 1024, B, h6, w6, ts->thin_w[0],
                                         M + ts->off[P_CONV1D].b, ts->flow6);
  DIM_LAUNCH_CHECK();
  if (int rc = run_classes(ctx, ts, tm.deconv5_fwd, tm.g_deconv5_fwd, 4, B, st)) return rc;
  if (int rc = copy_interior(a8, ts->cat2, 0, B, 512, st, s3)) return rc;
  LAUNCH1D(thin_deconv_fwd, (size_t)B * h5 * w5 * 2, st, ts->flow6, B, h6, w6, M + ts->off[P_UP65].w, M + ts->off[P_UP65].b,
           ts->cat2.p, ts->cat2.lo, ts->cat2.Hp, ts->cat2.Wp, 1, 1, 1088, 1024, h5, w5);
  thin_fwd2<<<B * h5 * w5, 128, 0, st>>>(ts->cat2.p, ts->cat2.lo, ts->cat2.Hp, ts->cat2.Wp, 1088, 1026, B, h5, w5, ts->thin_w[1],
                                         M + ts->off[P_CONV2D].b, ts->flow5);
  DIM_LAUNCH_CHECK();
  if (int rc = run_classes(ctx, ts, tm.deconv4_fwd, tm.g_deconv4_fwd, 4, B, st)) return rc;
  if (int rc = copy_interior(a6, ts->cat3, 0, B, 512, st, s3)) return rc;
  LAUNCH1D(thin_deconv_fwd, (size_t)B * h4 * w4 * 2, st, ts->flow5, B, h5, w5, M + ts->off[P_UP54].w, M + ts->off[P_UP54].b,
           ts->cat3.p, ts->cat3.lo, ts->cat3.Hp, ts->cat3.Wp, 1, 1, 832, 768, h4, w4);
  thin_fwd2<<<B * h4 * w4, 128, 0, st>>>(ts->cat3.p, ts->cat3.lo, ts->cat3.Hp, ts->cat3.Wp, 832, 770, B, h4, w4, ts->thin_w[2],
                                         M + ts->off[P_CONV3D].b, ts->flow4);
  DIM_LAUNCH_CHECK();
  thin_fwd1<<<B * h4 * w4, 128, 0, st>>>(ts->cat3.p, ts->cat3.lo, ts->cat3.Hp, ts->cat3.Wp, 832, 770, B, h4, w4, ts->thin_w[3],
                                         M + ts->off[P_MASK3].b, ts->mask4);
  DIM_LAUNCH_CHECK();
  DIM_CHECK(cudaEventRecord(ts->ev_phase[2], st));
  fullres_loss_kernel<<<LOSS_BLOCKS, 256, 0, st>>>(ts->flow4, ts->mask4, h4, w4, M + ts->off[P_UPS].w, M + ts->off[P_MUPS].w, io.zflow,
                                                   io.zfw, io.zmask_gt, B, H, W, cfg.normalize_flow, gs_flow, gs_mask, io.flow_est, io.mask_prob,
                                                   ts->dfull, ts->loss_part);
  DIM_LAUNCH_CHECK();
  pose_head_fwd_kernel<<<1, 32, 0, st>>>(ts->rot_raw, ts->ztrans, io.zoom_factor, B, ts->rot_n, ts->trans_est);
  DIM_LAUNCH_CHECK();
  const int pm_blocks = 64;
  if (io.pc_model) {
    if (int rc = transform3d_fwd_launch(io.pc_model, ts->rot_n, ts->trans_est, io.src_pose, B, io.N, Tm, Tsd, cfg.rot_coord, ts->pts_est, st)) return rc;
    pm_loss_kernel<<<pm_blocks, 256, 0, st>>>(ts->pts_est, io.pc_observed, io.pc_weights, (size_t)B * 3 * io.N, cfg.normalize_3d_point, gs_pm, ts->dpts, ts->loss_part);
    DIM_LAUNCH_CHECK();
  }
  if (io.losses) {
    loss_final_kernel<<<1, 256, 0, st>>>(ts->loss_part, LOSS_BLOCKS, io.pc_model ? pm_blocks : 0, gs_flow, gs_pm, gs_mask, io.losses);
    DIM_LAUNCH_CHECK();
  }
  if (io.rot_raw) DIM_CHECK(cudaMemcpyAsync(io.rot_raw, ts->rot_raw, (size_t)B * 16, cudaMemcpyDeviceToDevice, st));
  if (io.rot_est_norm) DIM_CHECK(cudaMemcpyAsync(io.rot_est_norm, ts->rot_n, (size_t)B * 16, cudaMemcpyDeviceToDevice, st));
  if (io.trans_est) DIM_CHECK(cudaMemcpyAsync(io.trans_est, ts->trans_est, (size_t)B * 12, cudaMemcpyDeviceToDevice, st));
  DIM_CHECK(cudaEventRecord(ts->ev_phase[3], st));
  r_fwd.end();
  if (G == nullptr) return 0;  // forward only (non-FAST_TEST outputs)

  // ---------------- backward
  DimNvtxRange r_bwd("dim_train backward");
  DIM_CHECK(cudaMemsetAsync(G + ts->off[P_UPS].w, 0, (ts->off[P_UPS].wn + ts->off[P_MUPS].wn) * sizeof(float), st));  // frozen (lr_mult 0)
  // pose heads
  if (int rc = transform3d_bwd_launch(ts->dpts, io.pc_model, ts->rot_n, ts->trans_est, io.src_pose, B, io.N, Tm, Tsd, cfg.rot_coord, ts->drot_n, ts->dtrans, st)) return rc;
  pose_head_bwd_kernel<<<1, 32, 0, st>>>(ts->rot_raw, ts->rot_n, ts->drot_n, B, ts->drot);
  DIM_LAUNCH_CHECK();
  fc_heads_bwd_kernel<<<B, 256, 0, st>>>(ts->drot, ts->dtrans, M + ts->off[P_ROT].w, M + ts->off[P_TRANS].w, M + ts->off[P_FC7].w, ts->h6,
                                         ts->h7, ts->dh7, ts->dh6);
  DIM_LAUNCH_CHECK();
  // every weight gradient runs on the internal stream sw, next to the data-gradient chain on st
  cudaStream_t sw = ts->side[3];
  if (int rc = fork_side(ts, st)) return rc;
  LAUNCH1D(fc_wgrad_kernel, 4 * 256, sw, ts->drot, ts->h7, B, 4, 256, G + ts->off[P_ROT].w, G + ts->off[P_ROT].b);
  LAUNCH1D(fc_wgrad_kernel, 3 * 256, sw, ts->dtrans, ts->h7, B, 3, 256, G + ts->off[P_TRANS].w, G + ts->off[P_TRANS].b);
  LAUNCH1D(fc_wgrad_kernel, 256 * 256, sw, ts->dh7, ts->h6, B, 256, 256, G + ts->off[P_FC7].w, G + ts->off[P_FC7].b);
  (s3 ? fc6_wgrad_kernel<true> : fc6_wgrad_kernel<false>)<<<dim3(81920 / 2 / 256, 8), 256, 0, sw>>>(ts->dh6, ns->act_hi[10], ns->act_lo[10],
                                                                                                     B, G + ts->off[P_FC6].w);
  DIM_LAUNCH_CHECK();
  LAUNCH1D(fc_wgrad_kernel, 256, sw, ts->dh6, ts->h6 /*unused for K=0*/, B, 256, 0, G + ts->off[P_FC6].w /*no write*/, G + ts->off[P_FC6].b);
  DIM_CHECK(cudaEventRecord(ts->ev_phase[4], st));
  // full-resolution heads -> 1/16 maps
  LAUNCH1D(upsample_bwd_kernel, (size_t)B * h4 * w4 * 3 * 32, st, ts->dfull, M + ts->off[P_UPS].w, M + ts->off[P_MUPS].w, B, H, W, h4, w4,
           ts->dflow4, ts->dmask4);
  // Convolution3 / mask_conv3
  if (int rc = fork_side(ts, st)) return rc;
  if (int rc = thin_wgrad<2>(ts, ts->cat3, 770, B, h4, w4, ts->dflow4, G + ts->off[P_CONV3D].w, G + ts->off[P_CONV3D].b, sw)) return rc;
  if (int rc = thin_wgrad<1>(ts, ts->cat3, 770, B, h4, w4, ts->dmask4, G + ts->off[P_MASK3].w, G + ts->off[P_MASK3].b, sw)) return rc;
  auto thin_dgrad2 = s3 ? thin_conv_dgrad_kernel<2, true> : thin_conv_dgrad_kernel<2, false>;
  auto thin_dgrad1 = s3 ? thin_conv_dgrad_kernel<1, true> : thin_conv_dgrad_kernel<1, false>;
  auto lrelu_mask_inplace = s3 ? lrelu_mask_inplace_kernel<true> : lrelu_mask_inplace_kernel<false>;
  LAUNCH1D(thin_dgrad2, (size_t)B * h4 * w4 * 832, st, ts->dflow4, ts->thin_w[2], 770, B, h4, w4, ts->dcat3.p, ts->dcat3.lo,
           ts->dcat3.Hp, ts->dcat3.Wp, 1, 1, 832, 832, 0);
  LAUNCH1D(thin_dgrad1, (size_t)B * h4 * w4 * 832, st, ts->dmask4, ts->thin_w[3], 770, B, h4, w4, ts->dcat3.p, ts->dcat3.lo,
           ts->dcat3.Hp, ts->dcat3.Wp, 1, 1, 832, 832, 1);
  // upsample_flow5to4
  if (int rc = thin_deconv_bwd(ts->flow5, B, h5, w5, M + ts->off[P_UP54].w, ts->dcat3, 768, h4, w4, ts->dflow5, G + ts->off[P_UP54].w,
                               G + ts->off[P_UP54].b, st, sw, ts))
    return rc;
  // deconv4: LeakyReLU backward on its slice, bias, weight and data gradients
  LAUNCH1D(lrelu_mask_inplace, (size_t)B * h4 * w4 * 32, st, ts->dcat3.p, ts->dcat3.lo, ts->cat3.p, ts->cat3.Hp, ts->cat3.Wp, 1, 1, 832,
           512, B, h4, w4, 256, 0.1f);
  if (int rc = fork_side(ts, st)) return rc;
  if (int rc = bias_grad(ts, ts->dcat3, B, 512, 256, G + ts->off[P_DECONV4].b, sw)) return rc;
  if (int rc = run_wgrad(tm.wg_deconv4, tm.wg_bn_d4, s3, WG_DECONV, 1026, 256, 4, G + ts->off[P_DECONV4].w, sw)) return rc;
  if (int rc = run_generic(ctx, tm.deconv4_dgrad, tm.g_deconv4_dgrad, B, st, s3)) return rc;
  // Convolution2 (adds to dcat2), upsample_flow6to5
  if (int rc = thin_wgrad<2>(ts, ts->cat2, 1026, B, h5, w5, ts->dflow5, G + ts->off[P_CONV2D].w, G + ts->off[P_CONV2D].b, sw)) return rc;  // dflow5 was final before the last fork
  LAUNCH1D(thin_dgrad2, (size_t)B * h5 * w5 * 1088, st, ts->dflow5, ts->thin_w[1], 1026, B, h5, w5, ts->dcat2.p, ts->dcat2.lo,
           ts->dcat2.Hp, ts->dcat2.Wp, 1, 1, 1088, 1088, 1);
  if (int rc = thin_deconv_bwd(ts->flow6, B, h6, w6, M + ts->off[P_UP65].w, ts->dcat2, 1024, h5, w5, ts->dflow6, G + ts->off[P_UP65].w,
                               G + ts->off[P_UP65].b, st, sw, ts))
    return rc;
  // deconv5
  LAUNCH1D(lrelu_mask_inplace, (size_t)B * h5 * w5 * 64, st, ts->dcat2.p, ts->dcat2.lo, ts->cat2.p, ts->cat2.Hp, ts->cat2.Wp, 1, 1, 1088,
           512, B, h5, w5, 512, 0.1f);
  if (int rc = fork_side(ts, st)) return rc;
  if (int rc = bias_grad(ts, ts->dcat2, B, 512, 512, G + ts->off[P_DECONV5].b, sw)) return rc;
  if (int rc = run_wgrad(tm.wg_deconv5, tm.wg_bn_d5, s3, WG_DECONV, 1024, 512, 4, G + ts->off[P_DECONV5].w, sw)) return rc;
  // Convolution1 -> partial gradient of ReLU10, + fc6 data gradient, then deconv5's data gradient closes dZ of conv6_1
  if (int rc = thin_wgrad<2>(ts, ts->act10b, 1024, B, h6, w6, ts->dflow6, G + ts->off[P_CONV1D].w, G + ts->off[P_CONV1D].b, sw)) return rc;  // dflow6: before the last fork
  LAUNCH1D(thin_dgrad2, (size_t)B * h6 * w6 * 1024, st, ts->dflow6, ts->thin_w[0], 1024, B, h6, w6, ts->dA10p.p, ts->dA10p.lo,
           ts->dA10p.Hp, ts->dA10p.Wp, 0, 0, 1024, 1024, 0);
  (s3 ? fc6_dgrad_kernel<true> : fc6_dgrad_kernel<false>)<<<81920 / 64, 256, 0, st>>>(ts->dh6, ns->fc6_w_hi, ns->fc6_w_lo, B, ts->dA10p.p,
                                                                                       ts->dA10p.lo);
  DIM_LAUNCH_CHECK();
  if (int rc = run_generic(ctx, tm.deconv5_dgrad, tm.g_deconv5_dgrad, B, st, s3)) return rc;
  DIM_CHECK(cudaEventRecord(ts->ev_phase[5], st));
  // encoder
  if (ns->input_depth)
    LAUNCH1D((s3 ? strip_to_nhwc64_kernel<true> : strip_to_nhwc64_kernel<false>), (size_t)B * g[0].rows * 8 * g[0].cols, st, ns->act_hi[0],
             ns->act_lo[0], ts->s2d64.p, ts->s2d64.lo, (size_t)B * g[0].rows * 8 * g[0].cols, g[0].cols);
  else
    LAUNCH1D((s3 ? strip_to_nhwc32_kernel<true> : strip_to_nhwc32_kernel<false>), (size_t)B * g[0].rows * 4 * g[0].cols, st, ns->act_hi[0],
             ns->act_lo[0], ts->s2d32.p, ts->s2d32.lo, (size_t)B * g[0].rows * 4 * g[0].cols, g[0].cols);
  for (int i = 9; i >= 0; --i) {
    const LayerSpec &s = kLayers[i];
    if (int rc = fork_side(ts, st)) return rc;  // gz[i] is complete on st
    if (i == 9)  // heads, decoder (thin kernels on st, deconvolution wgrads on sw): tensors 10..23 are done
      if (int rc = record_buckets(io, 10, 1 << 30, sw)) return rc;
    if (int rc = bias_grad(ts, ts->gz[i], B, 0, s.Cout, G + ts->off[i].b, sw)) return rc;
    if (i == 0 && ns->input_depth) {
      if (int rc = run_wgrad(tm.wg[0], tm.wg_bn[0], s3, WG_CONV1_RGBD, 64, 10, 7, G + ts->off[0].w, sw)) return rc;
    } else if (i == 0) {
      if (int rc = run_wgrad_conv1(ctx, ts, tm.wg[0], G + ts->off[0].w, sw)) return rc;
    } else if (int rc = run_wgrad(tm.wg[i], tm.wg_bn[i], s3, WG_CONV, s.Cout, s.Cin, s.k, G + ts->off[i].w, sw)) return rc;
    if (int rc = record_buckets(io, i, i + 1, sw)) return rc;
    if (i >= 1)
      if (int rc = run_classes(ctx, ts, tm.dgrad[i], tm.g_dgrad[i], tm.n_dgrad[i], B, st)) return rc;
  }
  DIM_CHECK(cudaEventRecord(ts->ev_phase[6], st));
  DIM_CHECK(cudaEventRecord(ts->ev_side, sw));
  DIM_CHECK(cudaStreamWaitEvent(st, ts->ev_side, 0));
  DIM_CHECK(cudaEventRecord(ts->ev_phase[7], st));
  return 0;
}

int train_sgd_update(dim_ctx *ctx, const float *grads, float lr, float momentum, float wd, float rescale, cudaStream_t st) {
  TrainState *ts = train_of(ctx);
  DIM_REQUIRE(ts != nullptr && grads != nullptr, "dim_train_sgd_update: bad state");
  SgdSegs segs;
  for (int i = 0; i < 22; ++i) {
    segs.end[2 * i] = ts->off[i].w + ts->off[i].wn;
    segs.end[2 * i + 1] = ts->off[i].b + ts->off[i].bn;
  }
  const size_t n = ts->off[21].b + ts->off[21].bn;  // the two bilinear upsampling kernels behind it are frozen (lr_mult 0)
  if (ctx->net->repack_done) DIM_CHECK(cudaStreamWaitEvent(st, ctx->net->repack_done, 0));  // a previous refresh still reads the master
  LAUNCH1D(sgd_kernel, n, st, ts->master, ts->mom, grads, n, segs, lr, momentum, wd, rescale);
  // The bf16 operand packs are refreshed on the internal stream, so the caller's stream is free for the work that does
  // not need them (re-render + labels of the next inner iteration, the zoom front); net_forward waits for `repack_done`.
  cudaStream_t sw = ts->side[3];
  DIM_CHECK(cudaEventRecord(ts->ev_fork, st));
  DIM_CHECK(cudaStreamWaitEvent(sw, ts->ev_fork, 0));
  if (int rc = repack_all(ctx, sw, ts->s3)) return rc;  // the bf16x3 step reads the lo halves: refresh them too
  DIM_CHECK(cudaEventRecord(ts->ev_repack, sw));
  ctx->net->repack_done = ts->ev_repack;
  return 0;
}

// test / debugging hook: copy an intermediate to the host.  id: 0 flow6, 1 flow5, 2 flow4, 3 mask4, 4 dflow4, 5 dmask4,
// 6 dflow5, 7 dflow6, 8 h6 (the fc6 activation kept for the backward pass), 9 dh6 (gradient of fc6's pre-activation) (fp32);
// 10 cat2, 11 cat3, 12 dcat2, 13 dcat3, 14 dA10p, 15 act10b, 20+i gz[i] (bf16, whole bordered buffer); 100 + one of the bf16 ids:
// that buffer's lo half (exists once the step has run in bf16x3); the pose heads (fp32): 30 h7 [B][256], 31 rot_raw [B][4],
// 32 ztrans [B][3], 33 rot_n [B][4], 34 trans_est [B][3], 35 pts_est and 36 dpts [B][3][N] (N of the last step), 37 drot_n [B][4], 38 dtrans [B][3], 39 drot [B][4], 40 dh7 [B][256], 41 dfull [B][3][H][W]
int train_debug_tensor(dim_ctx *ctx, int id, void *host, size_t bytes) {
  TrainState *ts = train_of(ctx);
  DIM_REQUIRE(ts != nullptr, "no training state");
  const void *src = nullptr;
  size_t have = 0;
  const int B = ctx->max_batch;
  const LayerGeom *g = ctx->net->g;
  const bool lo = id >= 100;
  if (lo) id -= 100;
  auto fb = [&](const Buf &b) { src = lo ? b.lo : b.p; have = b.per_image() * B * 2; };
  const bool bf16_id = (id >= 10 && id < 16) || (id >= 20 && id < 30);  // only these have lo halves
  switch (lo && !bf16_id ? -1 : id) {
    case 0: src = ts->flow6; have = (size_t)B * g[9].Ho * g[9].Wo * 8; break;
    case 1: src = ts->flow5; have = (size_t)B * g[7].Ho * g[7].Wo * 8; break;
    case 2: src = ts->flow4; have = (size_t)B * g[5].Ho * g[5].Wo * 8; break;
    case 3: src = ts->mask4; have = (size_t)B * g[5].Ho * g[5].Wo * 4; break;
    case 4: src = ts->dflow4; have = (size_t)B * g[5].Ho * g[5].Wo * 8; break;
    case 5: src = ts->dmask4; have = (size_t)B * g[5].Ho * g[5].Wo * 4; break;
    case 6: src = ts->dflow5; have = (size_t)B * g[7].Ho * g[7].Wo * 8; break;
    case 7: src = ts->dflow6; have = (size_t)B * g[9].Ho * g[9].Wo * 8; break;
    case 8: src = ts->h6; have = (size_t)B * 256 * 4; break;
    case 9: src = ts->dh6; have = (size_t)B * 256 * 4; break;
    case 10: fb(ts->cat2); break;
    case 11: fb(ts->cat3); break;
    case 12: fb(ts->dcat2); break;
    case 13: fb(ts->dcat3); break;
    case 14: fb(ts->dA10p); break;
    case 15: fb(ts->act10b); break;
    case 30: src = ts->h7; have = (size_t)B * 256 * 4; break;
    case 31: src = ts->rot_raw; have = (size_t)B * 4 * 4; break;
    case 32: src = ts->ztrans; have = (size_t)B * 3 * 4; break;
    case 33: src = ts->rot_n; have = (size_t)B * 4 * 4; break;
    case 34: src = ts->trans_est; have = (size_t)B * 3 * 4; break;
    case 35: src = ts->pts_est; have = (size_t)B * 3 * ts->max_points * 4; break;
    case 36: src = ts->dpts; have = (size_t)B * 3 * ts->max_points * 4; break;
    case 37: src = ts->drot_n; have = (size_t)B * 4 * 4; break;
    case 38: src = ts->dtrans; have = (size_t)B * 3 * 4; break;
    case 39: src = ts->drot; have = (size_t)B * 4 * 4; break;
    case 40: src = ts->dh7; have = (size_t)B * 256 * 4; break;
    case 41: src = ts->dfull; have = (size_t)B * 3 * ctx->H * ctx->W * 4; break;
    default:
      if (id >= 20 && id < 30) fb(ts->gz[id - 20]);
  }
  DIM_REQUIRE(src != nullptr && bytes <= have, "bad debug tensor id or size");
  DIM_CHECK(cudaDeviceSynchronize());
  DIM_CHECK(cudaMemcpy(host, src, bytes, cudaMemcpyDeviceToHost));
  return 0;
}

// milliseconds of the phases of the last forward_backward on the caller's stream: encoder fwd, decoder fwd, losses + pose heads,
// fc / head backward, decoder backward, encoder backward (data-gradient chain), wait for the weight-gradient stream
int train_debug_phases(dim_ctx *ctx, float *ms7) {
  TrainState *ts = train_of(ctx);
  DIM_REQUIRE(ts != nullptr, "no training state");
  DIM_CHECK(cudaDeviceSynchronize());
  for (int i = 0; i < 7; ++i) DIM_CHECK(cudaEventElapsedTime(&ms7[i], ts->ev_phase[i], ts->ev_phase[i + 1]));
  return 0;
}

void train_debug_geometry(dim_ctx *ctx, int id, int *out /*Hp, Wp, py, px, C, H, W*/) {
  TrainState *ts = train_of(ctx);
  const Buf *b = nullptr;
  if (id >= 100) id -= 100;  // a lo half has its buffer's geometry
  if (id == 10) b = &ts->cat2; else if (id == 11) b = &ts->cat3; else if (id == 12) b = &ts->dcat2; else if (id == 13) b = &ts->dcat3;
  else if (id == 14) b = &ts->dA10p; else if (id == 15) b = &ts->act10b; else if (id >= 20 && id < 30) b = &ts->gz[id - 20];
  if (!b) { for (int k = 0; k < 7; ++k) out[k] = 0; return; }
  out[0] = b->Hp; out[1] = b->Wp; out[2] = b->py; out[3] = b->px; out[4] = b->C; out[5] = b->H; out[6] = b->W;
}

}  // namespace dim
