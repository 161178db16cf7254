// net.cu -- FlowNetS encoder + fc + heads on the device (deepim/symbols/deepIM_flownet.py:53-116 and
// 716-726), weight repacking, tensor-map construction and layer scheduling.
//
//   conv tower : conv1_kernel + 9 x conv_igemm_persistent_kernel (wgmma + TMA, conv_igemm.cuh)
//   fc6        : 81920 -> 256, a pure weight stream (HBM-bound): split-K mma.sync kernel (batch = M = 16),
//                deterministic two-pass reduction (partials reduced in fixed order by the head kernel)
//   head       : fc6 reduce + bias + LeakyReLU -> fc7 -> LeakyReLU -> rot(4), trans(3) ->
//                ZoomTrans^-1 (zoom_trans.py:30-31) -> se3 (B,7)
#include <cuda_fp16.h>
#include <string.h>

#include <memory>
#include <mutex>

#include "launch.cuh"
#include "net_state.cuh"

namespace dim {

// --------------------------------------------------------------------------------- geometry
static void build_geometry(NetState *ns, int H, int W) {
  int h = H, w = W;
  for (int i = 0; i < 10; ++i) {
    const LayerSpec &s = kLayers[i];
    LayerGeom &g = ns->g[i];
    g.Cin = s.Cin; g.Cout = s.Cout; g.k = s.k; g.stride = s.stride; g.pad = s.pad;
    g.Hin = h; g.Win = w;
    g.Ho = (h + 2 * s.pad - s.k) / s.stride + 1;
    g.Wo = (w + 2 * s.pad - s.k) / s.stride + 1;
    if (g.Ho < 1) g.Ho = 1;
    if (g.Wo < 1) g.Wo = 1;
    int Hp = h + 2 * s.pad, Wp = w + 2 * s.pad;
    if (s.stride == 2) { Hp += Hp & 1; Wp += Wp & 1; }
    g.py = g.px = s.pad;
    if (i == 0 && ns->input_depth) {
      // RGB-D conv1 (Cin = 10): space-to-depth with 16-channel phase chunks -> 4x4 taps over 64 channels (K = 1024)
      g.Cin = 10;
      g.rows = Hp / 2; g.cols = Wp / 2; g.Cbuf = 64;
      g.KH = g.KW = 4; g.stride_eff = 1; g.Ceff = 64; g.Hq = g.rows;
      g.BLOCK_K = 64; g.BLOCK_N = 64;
    } else if (i == 0) {
      // conv1 (Cin = 8, 7x7 s2): space-to-depth -> 4x4 stride-1 taps over 32 channels
      g.rows = Hp / 2; g.cols = Wp / 2; g.Cbuf = 32;
      g.KH = g.KW = 4; g.stride_eff = 1; g.Ceff = 32; g.Hq = g.rows;
      g.BLOCK_K = 32; g.BLOCK_N = 64;
    } else {
      g.rows = Hp; g.cols = Wp; g.Cbuf = s.Cin;
      g.KH = g.KW = s.k; g.stride_eff = s.stride; g.Ceff = s.Cin;
      g.Hq = (s.stride == 2) ? Hp / 2 : Hp;
      g.BLOCK_K = 64; g.BLOCK_N = s.Cout >= 256 ? 256 : 128;
    }
    // M tile: BW x BH rectangle of output pixels with BW | Wo and BW*BH <= 128.  Maximise the rows
    // used; keep boxes at least 8 pixels wide (>= 1 KB contiguous per TMA row) when possible.
    int best_bw = 0, best_score = -1;
    for (int pass = 0; pass < 2 && best_bw == 0; ++pass)
      for (int d = 1; d <= g.Wo && d <= 128; ++d) {
        if (g.Wo % d) continue;
        if (pass == 0 && d < 8) continue;
        const int score = d * (128 / d) * 1000 + d;
        if (score > best_score) { best_score = score; best_bw = d; }
      }
    if (best_bw == 0) best_bw = 1;  // degenerate geometry (tiny geometry-only contexts)
    g.BW = best_bw; g.BH = 128 / best_bw;
    g.n_col_tiles = g.Wo > 0 ? g.Wo / g.BW : 0;
    if (i == 0) {  // conv1 strip kernel: one output row x BW columns per tile, BW = ceil(Wo / ceil(Wo/128))
      const int nt = cdiv(g.Wo, 128);
      g.BW = cdiv(g.Wo, nt); g.BH = 1; g.n_col_tiles = nt;
    }
    g.kblocks = g.KH * g.KW * (g.Ceff / g.BLOCK_K);
    h = g.Ho; w = g.Wo;
  }
}

// --------------------------------------------------------------------------------- tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int encode_map(CUtensorMap *m, void *base, int rank, const uint64_t *dims, const uint64_t *strides_bytes,
                      const uint32_t *box, int block_k /*64: SW128, 32: SW64, 0: no swizzle*/) {
  EncodeTiledFn fn = get_encode();
  DIM_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled entry point not available (driver too old?)");
  cuuint64_t gd[5]; cuuint64_t gs[5]; cuuint32_t bx[5]; cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i < rank - 1; ++i) gs[i] = strides_bytes[i];
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, base, gd, gs, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE,
                  block_k == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                : (block_k == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE),
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu %llu %llu box %u %u %u)", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)(rank > 2 ? dims[2] : 0),
              box[0], box[1], rank > 2 ? box[2] : 0);
    return 3;
  }
  return 0;
}

static int build_maps(NetState *ns, int B, bool f16, TensorMaps &tm) {
  for (int i = 0; i < 10; ++i) {
    const LayerGeom &g = ns->g[i];
    ConvKParams &kp = tm.kp[i];
    memset(&kp, 0, sizeof(kp));
    for (int lo = 0; lo < 2; ++lo) {
      __nv_bfloat16 *base = lo ? ns->act_lo[i] : ns->act_hi[i];
      CUtensorMap *maps = lo ? kp.a_lo_map : kp.a_map;
      // conv2 ... conv6_1: one box per consumer warpgroup (BW x BH/2 pixels; conv_igemm.cuh)
      const uint32_t box[3] = {(uint32_t)g.BLOCK_K, (uint32_t)g.BW, (uint32_t)(g.BH / 2)};
      if (i == 0 && ns->input_depth) {
        // RGB-D conv1 strip layout [B*rows][8 chunks][cols][8 ch]: box = 8 ch x (BW+3) cols x 8 chunks x 1 row
        const uint64_t dims[4] = {8, (uint64_t)g.cols, 8, (uint64_t)B * g.rows};
        const uint64_t str[3] = {16, (uint64_t)g.cols * 16, (uint64_t)g.cols * 128};
        const uint32_t box4[4] = {8, (uint32_t)(g.BW + 3), 8, 1};
        if (int rc = encode_map(&maps[0], base, 4, dims, str, box4, 0)) return rc;
        maps[1] = maps[2] = maps[3] = maps[0];
      } else if (i == 0) {
        // conv1_kernel reads its strips with plain bulk copies (kp.in_hi / in_lo): no activation map
      } else if (g.stride_eff == 1) {
        const uint64_t dims[3] = {(uint64_t)g.Cbuf, (uint64_t)g.cols, (uint64_t)B * g.rows};
        const uint64_t str[2] = {(uint64_t)g.Cbuf * 2, (uint64_t)g.cols * g.Cbuf * 2};
        if (int rc = encode_map(&maps[0], base, 3, dims, str, box, g.BLOCK_K)) return rc;
        maps[1] = maps[2] = maps[3] = maps[0];
      } else {
        for (int ph = 0; ph < 2; ++ph)
          for (int pw = 0; pw < 2; ++pw) {
            const uint64_t dims[3] = {(uint64_t)g.Cbuf, (uint64_t)g.cols / 2, (uint64_t)B * g.rows / 2};
            const uint64_t str[2] = {(uint64_t)2 * g.Cbuf * 2, (uint64_t)2 * g.cols * g.Cbuf * 2};
            __nv_bfloat16 *vb = base + ((size_t)ph * g.cols + pw) * g.Cbuf;
            if (int rc = encode_map(&maps[(ph << 1) | pw], vb, 3, dims, str, box, g.BLOCK_K)) return rc;
          }
      }
    }
    {
      const uint64_t Ktot = (uint64_t)g.KH * g.KW * g.Ceff;
      const uint64_t dims[2] = {Ktot, (uint64_t)g.Cout};
      const uint64_t str[1] = {Ktot * 2};
      // RGB-D conv1 loads its resident weights in boxes of 16 output channels (bf16x3 CTAs own 16 of them)
      const uint32_t box[2] = {(uint32_t)g.BLOCK_K, (uint32_t)(i == 0 && ns->input_depth ? 16 : g.BLOCK_N)};
      __nv_bfloat16 *wop = f16 ? ns->w_f16[i] : ns->w_hi[i];
      if (int rc = encode_map(&kp.b_map, wop, 2, dims, str, box, g.BLOCK_K)) return rc;
      if (int rc = encode_map(&kp.b_lo_map, ns->w_lo[i], 2, dims, str, box, g.BLOCK_K)) return rc;
    }
    kp.KH = g.KH; kp.KW = g.KW; kp.stride = g.stride_eff; kp.cchunks = g.Ceff / g.BLOCK_K;
    kp.BW = g.BW; kp.BH = g.BH; kp.n_col_tiles = g.n_col_tiles;
    kp.Hq = g.Hq; kp.Ho = g.Ho; kp.Wo = g.Wo; kp.Bn = B;
    if (i < 9) {
      const LayerGeom &nx = ns->g[i + 1];
      kp.out_Hp = nx.rows; kp.out_Wp = nx.cols; kp.out_py = nx.py; kp.out_px = nx.px;
    } else {
      kp.out_Hp = g.Ho; kp.out_Wp = g.Wo; kp.out_py = 0; kp.out_px = 0;
    }
    kp.Cout = g.Cout;
    kp.kblocks = g.kblocks;
    kp.slope = 0.1f;
    kp.bias = ns->bias[i];
    kp.out_hi = ns->act_hi[i + 1];
    kp.out_lo = ns->act_lo[i + 1];
    if (i == 0 && !ns->input_depth) {
      // conv1_kernel: strips from the space-to-depth input
      kp.in_hi = ns->act_hi[0];
      kp.in_lo = ns->act_lo[0];
      kp.in_cols = g.cols;
    }
    if (i > 0 || !ns->input_depth) {
      // output tiles TMA-stored into the next layer's buffer through a 4-D map (Cout, Wo, Ho, B) whose origin is the
      // interior's first pixel: the zero border lies outside every box.  conv1_kernel stores hi and lo rows of kConv1StoreN
      // pixels; conv_igemm a warpgroup's BW x BH/2 pixels, which must not span more than two images
      DIM_REQUIRE(i == 0 || (g.BH % 2 == 0 && g.BH / 2 <= g.Hq && g.BW * (g.BH / 2) <= 64),
                  "conv_igemm: a consumer warpgroup's box must be whole output rows within two images");
      const uint64_t cb = (uint64_t)g.Cout * 2;
      const uint64_t dims[4] = {(uint64_t)g.Cout, (uint64_t)g.Wo, (uint64_t)g.Ho, (uint64_t)B};
      const uint64_t str[3] = {cb, (uint64_t)kp.out_Wp * cb, (uint64_t)kp.out_Hp * kp.out_Wp * cb};
      const uint32_t box[4] = {64, (uint32_t)(i == 0 ? kConv1StoreN : g.BW), (uint32_t)(i == 0 ? 1 : g.BH / 2), 1};
      const size_t interior = ((size_t)kp.out_py * kp.out_Wp + kp.out_px) * g.Cout;
      for (int lo = 0; lo < (i == 0 ? 2 : 1); ++lo)
        if (int rc = encode_map(&kp.out_map[lo], (lo ? ns->act_lo[i + 1] : ns->act_hi[i + 1]) + interior, 4, dims, str, box, 64))
          return rc;
    }
  }
  return 0;
}

// --------------------------------------------------------------------------------- fc6 + head
// fc6 split-K on the legacy tensor path: the batch (<= 16 instances) is exactly the M = 16 of
// mma.sync.m16n8k16, so each warp streams its weight rows once (16 B per lane, K-permuted so that the
// 8 consecutive bf16 a lane loads feed two MMA steps) and multiplies them against the activation
// chunk staged in shared memory.  HBM-bound by design: 42 MB of bf16 weights per call (84 MB with the
// lo halves in bf16x3 mode).  CTA s owns k in [s*KC, (s+1)*KC) for all 256 outputs; partials are
// reduced in fixed order by the head kernel (deterministic, no atomics).
template <bool F16>
__device__ __forceinline__ void mma_bf16_16816(float *c, const uint32_t *a, uint32_t b0, uint32_t b1) {
  if (F16)
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// S3: bf16 hi/lo operands (3 MMAs per step); F16: IEEE half operands (one MMA per step, like plain bf16)
template <bool S3, bool F16 = false>
__global__ void __launch_bounds__(256) fc6_mma_kernel(const __nv_bfloat16 *__restrict__ act_hi,
                                                      const __nv_bfloat16 *__restrict__ act_lo,
                                                      const __nv_bfloat16 *__restrict__ w_hi,
                                                      const __nv_bfloat16 *__restrict__ w_lo, int B, int max_batch,
                                                      float *__restrict__ partial) {
  constexpr int PITCH = FC6_KC * 2 + 64;  // bytes; +64 keeps the 16-B fragment loads conflict-free
  __shared__ __align__(16) uint8_t a_hi_s[16 * PITCH];
  __shared__ __align__(16) uint8_t a_lo_s[S3 ? 16 * PITCH : 16];
  const int s = blockIdx.x, k0 = s * FC6_KC;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  for (int b0 = 0; b0 < B; b0 += 16) {
    const int nb = min(16, B - b0);
    __syncthreads();
    for (int idx = threadIdx.x; idx < 16 * (FC6_KC / 8); idx += blockDim.x) {
      const int r = idx / (FC6_KC / 8), c8 = idx - r * (FC6_KC / 8);
      uint4 vh = make_uint4(0, 0, 0, 0), vl = make_uint4(0, 0, 0, 0);
      if (r < nb) {
        const size_t o = (size_t)(b0 + r) * FC6_K + k0 + c8 * 8;
        vh = *reinterpret_cast<const uint4 *>(act_hi + o);
        if (S3) vl = *reinterpret_cast<const uint4 *>(act_lo + o);
      }
      *reinterpret_cast<uint4 *>(a_hi_s + r * PITCH + c8 * 16) = vh;
      if (S3) *reinterpret_cast<uint4 *>(a_lo_s + r * PITCH + c8 * 16) = vl;
    }
    __syncthreads();
    float acc[4][4];
#pragma unroll
    for (int t = 0; t < 4; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[t][e] = 0.f;
#pragma unroll 2
    for (int kc = 0; kc < FC6_KC; kc += 32) {
      // activation fragments for both MMA steps of this 32-k chunk: rows g and g+8, 8 bf16 each
      const uint4 ah0 = *reinterpret_cast<const uint4 *>(a_hi_s + g * PITCH + (kc + q * 8) * 2);
      const uint4 ah1 = *reinterpret_cast<const uint4 *>(a_hi_s + (g + 8) * PITCH + (kc + q * 8) * 2);
      const uint32_t A0[4] = {ah0.x, ah1.x, ah0.y, ah1.y}, A1[4] = {ah0.z, ah1.z, ah0.w, ah1.w};
      uint32_t L0[4] = {0, 0, 0, 0}, L1[4] = {0, 0, 0, 0};
      if (S3) {
        const uint4 al0 = *reinterpret_cast<const uint4 *>(a_lo_s + g * PITCH + (kc + q * 8) * 2);
        const uint4 al1 = *reinterpret_cast<const uint4 *>(a_lo_s + (g + 8) * PITCH + (kc + q * 8) * 2);
        L0[0] = al0.x; L0[1] = al1.x; L0[2] = al0.y; L0[3] = al1.y;
        L1[0] = al0.z; L1[1] = al1.z; L1[2] = al0.w; L1[3] = al1.w;
      }
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int j = warp * 32 + t * 8 + g;  // output row whose weights this lane streams
        const size_t wo = (size_t)j * FC6_K + k0 + kc + q * 8;
        const uint4 wh = __ldg(reinterpret_cast<const uint4 *>(w_hi + wo));
        mma_bf16_16816<F16>(acc[t], A0, wh.x, wh.y);
        mma_bf16_16816<F16>(acc[t], A1, wh.z, wh.w);
        if (S3) {
          const uint4 wl = __ldg(reinterpret_cast<const uint4 *>(w_lo + wo));
          mma_bf16_16816<false>(acc[t], L0, wh.x, wh.y);
          mma_bf16_16816<false>(acc[t], L1, wh.z, wh.w);
          mma_bf16_16816<false>(acc[t], A0, wl.x, wl.y);
          mma_bf16_16816<false>(acc[t], A1, wl.z, wl.w);
        }
      }
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int j = warp * 32 + t * 8 + q * 2;
      if (g < nb)
        *reinterpret_cast<float2 *>(partial + ((size_t)s * max_batch + b0 + g) * 256 + j) = make_float2(acc[t][0], acc[t][1]);
      if (g + 8 < nb)
        *reinterpret_cast<float2 *>(partial + ((size_t)s * max_batch + b0 + g + 8) * 256 + j) = make_float2(acc[t][2], acc[t][3]);
    }
  }
}

// one CTA of 1024 threads per instance: 4 thread groups share the fc6 split reduction and the fc7
// reduction (fixed summation order -> deterministic)
__global__ void __launch_bounds__(1024) head_kernel(const float *__restrict__ partial, int max_batch,
                                                    const float *__restrict__ fc6_b, const float *__restrict__ fc7_wT,
                                                    const float *__restrict__ fc7_b, const float *__restrict__ rot_w,
                                                    const float *__restrict__ rot_b, const float *__restrict__ trans_w,
                                                    const float *__restrict__ trans_b,
                                                    const float *__restrict__ zoom_factor /*nullable*/,
                                                    float *__restrict__ rot_out, float *__restrict__ trans_out,
                                                    float *__restrict__ se3_out, float *__restrict__ h6_out,
                                                    float *__restrict__ h7_out) {
  __shared__ float red[4][256];
  __shared__ float h6[256], h7[256], outv[8];
  const int b = blockIdx.x, j = threadIdx.x & 255, grp = threadIdx.x >> 8;
  float a = 0.f;
#pragma unroll 8
  for (int s = grp; s < FC6_SPLITS; s += 4) a += partial[((size_t)s * max_batch + b) * 256 + j];
  red[grp][j] = a;
  __syncthreads();
  if (grp == 0) {
    const float v = (((red[0][j] + red[1][j]) + red[2][j]) + red[3][j]) + fc6_b[j];
    h6[j] = v > 0.f ? v : 0.1f * v;
  }
  __syncthreads();
  float c = 0.f;
#pragma unroll 8
  for (int k = grp * 64; k < grp * 64 + 64; ++k) c = fmaf(h6[k], fc7_wT[k * 256 + j], c);
  red[grp][j] = c;
  __syncthreads();
  if (grp == 0) {
    const float v = (((red[0][j] + red[1][j]) + red[2][j]) + red[3][j]) + fc7_b[j];
    h7[j] = v > 0.f ? v : 0.1f * v;
    if (h6_out) { h6_out[b * 256 + j] = h6[j]; h7_out[b * 256 + j] = h7[j]; }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < 7) {
    const float *wrow = warp < 4 ? rot_w + warp * 256 : trans_w + (warp - 4) * 256;
    float v = 0.f;
    for (int k = lane; k < 256; k += 32) v = fmaf(h7[k], wrow[k], v);
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) outv[warp] = v + (warp < 4 ? rot_b[warp] : trans_b[warp - 4]);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (rot_out)
      for (int k = 0; k < 4; ++k) rot_out[4 * b + k] = outv[k];
    if (trans_out)
      for (int k = 0; k < 3; ++k) trans_out[3 * b + k] = outv[4 + k];
    if (se3_out) {
      // invZoomTrans (zoom_trans.py:30-31, b_inv_zoom=True): wx for both axes
      const float w = zoom_factor[4 * b];
      for (int k = 0; k < 4; ++k) se3_out[7 * b + k] = outv[k];
      se3_out[7 * b + 4] = outv[4] * w;
      se3_out[7 * b + 5] = outv[5] * w;
      se3_out[7 * b + 6] = outv[6];
    }
  }
}

// --------------------------------------------------------------------------------- host API
int net_create(dim_ctx *ctx) {
  NetState *ns = new NetState();
  ctx->net = ns;
  ns->max_batch = ctx->max_batch;
  build_geometry(ns, ctx->H, ctx->W);
  if ((size_t)ns->g[9].Ho * ns->g[9].Wo * ns->g[9].Cout != (size_t)FC6_K) return 0;  // geometry-only context
  for (int i = 0; i <= 10; ++i) {
    size_t per;
    if (i < 10) per = (size_t)ns->g[i].rows * ns->g[i].cols * ns->g[i].Cbuf;
    else per = (size_t)ns->g[9].Ho * ns->g[9].Wo * ns->g[9].Cout;
    ns->act_elems_per_image[i] = per;
    // borders must be (and stay) zero: the epilogues only ever write interior pixels
    if (int rc = dev_alloc(ctx, &ns->act_hi[i], per * ctx->max_batch, true)) return rc;
    if (int rc = dev_alloc(ctx, &ns->act_lo[i], per * ctx->max_batch, true)) return rc;
  }
  ns->net_ok = ns->act_elems_per_image[10] == (size_t)FC6_K;  // fc6 is 81920 -> 256: needs 480x640
  if (int rc = dev_alloc(ctx, &ns->fc6_partial, (size_t)FC6_SPLITS * ctx->max_batch * 256, true)) return rc;
  return 0;
}

void net_destroy(dim_ctx *ctx) {
  if (ctx->net && ctx->net->layer_events) {
    for (int i = 0; i < 11; ++i) cudaEventDestroy(ctx->net->layer_events[i]);
    delete[] ctx->net->layer_events;
  }
  delete ctx->net;
  ctx->net = nullptr;
}

// ------------------------------------------------------------------------------ weight packing
// fp32 weights in the flat parameter vector's layouts -> 16-bit operand packs.  The same kernels serve dim_net_load (from a
// staging copy of the checkpoint) and the training step (from the fp32 master after every update).
//
// forward pack [Cout][kh][kw][Cin] of conv2 ... conv6_1: block = (co, 64 input channels), which reads k*k-float rows
// (contiguous) into shared memory and writes 64 consecutive 16-bit values per tap
__global__ void __launch_bounds__(256) pack_conv_fwd_kernel(const float *w, int Cout, int Cin, int k, __nv_bfloat16 *hi,
                                                            __nv_bfloat16 *lo, __nv_bfloat16 *f16) {
  __shared__ float tile[64 * 25];
  const int co = blockIdx.x, c0 = blockIdx.y * 64, kk = k * k;
  const int nc = min(64, Cin - c0);
  const float *src = w + ((size_t)co * Cin + c0) * kk;
  for (int i = threadIdx.x; i < nc * kk; i += 256) tile[i] = src[i];
  __syncthreads();
#pragma unroll 2  // the compiler's 4 with the optional fp16 store takes 40 registers (6 blocks per SM instead of 8)
  for (int i = threadIdx.x; i < nc * kk; i += 256) {
    const int tap = i / nc, cl = i - tap * nc;
    store_split(hi, lo, ((size_t)co * kk + tap) * Cin + c0 + cl, tile[cl * kk + tap], f16);
  }
}
// RGB-D conv1 space-to-depth pack [64][4][4][64]: W'[co][dh][dw][(ph*2 + pw)*16 + c] = W[co][c][2dh+ph][2dw+pw] for c < 10
// (0 beyond 7x7 and for c >= 10)
__global__ void __launch_bounds__(256) pack_conv1_rgbd_kernel(const float *w, __nv_bfloat16 *hi, __nv_bfloat16 *lo,
                                                              __nv_bfloat16 *f16) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 64 * 1024) return;
  const int co = i >> 10, tap = (i >> 6) & 15, phase = (i >> 4) & 3, c = i & 15;
  const int kh = 2 * (tap >> 2) + (phase >> 1), kw = 2 * (tap & 3) + (phase & 1);
  store_split(hi, lo, i, (c < 10 && kh < 7 && kw < 7) ? w[((co * 10 + c) * 7 + kh) * 7 + kw] : 0.f, f16);
}
// conv1 space-to-depth pack [64][4][4][32] of a (64, cin, 7, 7) weight: W'[co][dh][dw][conv1_kslot(dw,ph,pw) + c] =
// W[co][c][2dh+ph][2dw+pw] (0 beyond 7x7); cin = 8, or 6 for the image-only network, whose mask lanes 6-7 get zero columns
__global__ void __launch_bounds__(256) pack_conv1_kernel(const float *w, int cin, __nv_bfloat16 *hi, __nv_bfloat16 *lo,
                                                         __nv_bfloat16 *f16) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 64 * 512) return;
  const int c = i & 7, pw = (i >> 3) & 1, ph = (i >> 4) & 1, dw = (i >> 5) & 3, dh = (i >> 7) & 3, co = i >> 9;
  const int kh = 2 * dh + ph, kw = 2 * dw + pw;
  store_split(hi, lo, (i & ~31) + conv1_kslot(dw, ph, pw) + c,
              (c < cin && kh < 7 && kw < 7) ? w[((co * cin + c) * 7 + kh) * 7 + kw] : 0.f, f16);
}
// fc6 (out, hw, c) fp32 -> 16-bit operand (same order)
__global__ void __launch_bounds__(256) pack_fc6_kernel(const float *w, __nv_bfloat16 *hi, __nv_bfloat16 *lo, __nv_bfloat16 *f16) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)256 * FC6_K) return;
  store_split(hi, lo, i, w[i], f16);
}
// fc7 (out, in) -> fp32 [in][out] for head_kernel
__global__ void transpose256_kernel(const float *w, float *wT) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 65536) wT[(i & 255) * 256 + (i >> 8)] = w[i];
}

// first call allocates, later calls return at once: a reload overwrites in place, so the tensor maps cached in
// NetState::maps keep pointing at valid storage
int net_alloc_weights(dim_ctx *ctx) {
  NetState *ns = ctx->net;
  if (ns->trans_b) return 0;  // allocated last
  for (int i = 0; i < 10; ++i) {
    const LayerGeom &g = ns->g[i];
    const size_t n = (size_t)g.Cout * g.KH * g.KW * g.Ceff;
    if (int rc = dev_alloc(ctx, &ns->w_hi[i], n)) return rc;
    if (int rc = dev_alloc(ctx, &ns->w_lo[i], n)) return rc;
    if (int rc = dev_alloc(ctx, &ns->w_f16[i], n)) return rc;
    if (int rc = dev_alloc(ctx, &ns->bias[i], g.Cout)) return rc;
  }
  const size_t n6 = (size_t)256 * FC6_K;
  if (int rc = dev_alloc(ctx, &ns->fc6_w_hi, n6)) return rc;
  if (int rc = dev_alloc(ctx, &ns->fc6_w_lo, n6)) return rc;
  if (int rc = dev_alloc(ctx, &ns->fc6_w_f16, n6)) return rc;
  if (int rc = dev_alloc(ctx, &ns->fc6_b, 256)) return rc;
  if (int rc = dev_alloc(ctx, &ns->fc7_wT, 256 * 256)) return rc;
  if (int rc = dev_alloc(ctx, &ns->fc7_b, 256)) return rc;
  if (int rc = dev_alloc(ctx, &ns->rot_w, 4 * 256)) return rc;
  if (int rc = dev_alloc(ctx, &ns->rot_b, 4)) return rc;
  if (int rc = dev_alloc(ctx, &ns->trans_w, 3 * 256)) return rc;
  return dev_alloc(ctx, &ns->trans_b, 3);
}

// w[0..9]: conv1 ... conv6_1 (Cout, Cin, k, k), w[10]: fc6 (256, hw, c), w[11]: fc7 (out, in), device fp32.  Packs are
// written on st, each rounded once from w.  `packs` (PACK_*) names the packs to write: PACK_HI means new weights, so every
// pack left out goes stale; without it only the packs named are brought up to w (a lazy refresh from an unchanged master).
int net_pack_weights(dim_ctx *ctx, const float *const *w, cudaStream_t st, unsigned packs) {
  NetState *ns = ctx->net;
  auto H = [packs](__nv_bfloat16 *p) { return packs & PACK_HI ? p : nullptr; };
  auto L = [packs](__nv_bfloat16 *p) { return packs & PACK_LO ? p : nullptr; };
  auto F = [packs](__nv_bfloat16 *p) { return packs & PACK_F16 ? p : nullptr; };
  if (ns->input_depth)
    pack_conv1_rgbd_kernel<<<64 * 1024 / 256, 256, 0, st>>>(w[0], H(ns->w_hi[0]), L(ns->w_lo[0]), F(ns->w_f16[0]));
  else
    pack_conv1_kernel<<<64 * 512 / 256, 256, 0, st>>>(w[0], ns->input_mask ? 8 : 6, H(ns->w_hi[0]), L(ns->w_lo[0]),
                                                      F(ns->w_f16[0]));
  DIM_LAUNCH_CHECK();
  for (int i = 1; i < 10; ++i) {
    const LayerSpec &s = kLayers[i];
    pack_conv_fwd_kernel<<<dim3(s.Cout, cdiv(s.Cin, 64)), 256, 0, st>>>(w[i], s.Cout, s.Cin, s.k, H(ns->w_hi[i]),
                                                                          L(ns->w_lo[i]), F(ns->w_f16[i]));
    DIM_LAUNCH_CHECK();
  }
  pack_fc6_kernel<<<256 * FC6_K / 256, 256, 0, st>>>(w[10], H(ns->fc6_w_hi), L(ns->fc6_w_lo), F(ns->fc6_w_f16));
  DIM_LAUNCH_CHECK();
  if (packs & PACK_HI) {
    transpose256_kernel<<<256, 256, 0, st>>>(w[11], ns->fc7_wT);
    DIM_LAUNCH_CHECK();
    ns->lo_stale = ns->f16_stale = true;
  }
  if (packs & PACK_LO) ns->lo_stale = false;
  if (packs & PACK_F16) ns->f16_stale = false;
  return 0;
}

int net_load(dim_ctx *ctx, const float *const *W, const float *const *Bv) {
  NetState *ns = ctx->net;
  DIM_REQUIRE(ns != nullptr, "net not created");
  DIM_REQUIRE(ns->net_ok, "dim_net_load: FlowNetS + fc6 (81920 inputs) needs a 480x640 context");
  DIM_REQUIRE(!ns->train_aliased, "dim_net_load: this context trains; use dim_train_load_params (it owns the weights)");
  if (ns->loaded) DIM_CHECK(cudaDeviceSynchronize());  // a reload must not race kernels still reading the old weights
  if (int rc = net_alloc_weights(ctx)) return rc;
  // the packed tensors W[0..11] are staged on the device as fp32 for net_pack_weights (~180 MB, freed on return)
  size_t n[12], off[13] = {0};
  for (int i = 0; i < 10; ++i) {
    const LayerGeom &g = ns->g[i];
    const int cin = i == 0 && !ns->input_depth ? (ns->input_mask ? 8 : 6) : g.Cin;
    n[i] = (size_t)g.Cout * cin * g.k * g.k;
  }
  n[10] = (size_t)256 * FC6_K;
  n[11] = 256 * 256;
  for (int i = 0; i < 12; ++i) off[i + 1] = off[i] + n[i];
  float *stage_p = nullptr;
  DIM_CHECK(cudaMalloc(&stage_p, off[12] * sizeof(float)));
  std::unique_ptr<float, cudaError_t (*)(void *)> stage(stage_p, cudaFree);
  auto put = [](float *dst, const float *src, size_t count) {
    return cudaMemcpy(dst, src, count * sizeof(float), cudaMemcpyHostToDevice);
  };
  const float *w[12];
  for (int i = 0; i < 12; ++i) {
    w[i] = stage.get() + off[i];
    if (i != 10) DIM_CHECK(put(stage.get() + off[i], W[i], n[i]));
  }
  {  // fc6: (out, c*80 + h*10 + w) -> (out, (h*10+w)*1024 + c)   (NCHW flatten, deepIM_flownet.py:110)
    std::vector<float> p((size_t)256 * FC6_K);
    for (int o = 0; o < 256; ++o)
      for (int c = 0; c < 1024; ++c)
        for (int hw = 0; hw < 80; ++hw) p[(size_t)o * FC6_K + (size_t)hw * 1024 + c] = W[10][(size_t)o * FC6_K + (size_t)c * 80 + hw];
    DIM_CHECK(put(stage.get() + off[10], p.data(), n[10]));
  }
  for (int i = 0; i < 10; ++i) DIM_CHECK(put(ns->bias[i], Bv[i], ns->g[i].Cout));
  DIM_CHECK(put(ns->fc6_b, Bv[10], 256));
  DIM_CHECK(put(ns->fc7_b, Bv[11], 256));
  DIM_CHECK(put(ns->rot_w, W[12], 4 * 256));
  DIM_CHECK(put(ns->rot_b, Bv[12], 4));
  DIM_CHECK(put(ns->trans_w, W[13], 3 * 256));
  DIM_CHECK(put(ns->trans_b, Bv[13], 3));
  if (int rc = net_pack_weights(ctx, w, 0, PACK_HI | PACK_LO | PACK_F16)) return rc;
  DIM_CHECK(cudaStreamSynchronize(0));
  ns->loaded = true;
  return 0;
}

template <int BN, int ST, bool S3, bool F16>
static int launch_conv(const ConvKParams &kp, int total_tiles, int n_tiles, int cap, cudaStream_t st) {
  using S = ConvSmem2<BN, ST, S3, 0>;
  static bool attr_set = false;
  if (!attr_set) {
    DIM_CHECK(cudaFuncSetAttribute(conv_igemm_persistent_kernel<BN, ST, S3, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   S::TOTAL));
    attr_set = true;
  }
  const int grid = total_tiles < cap ? total_tiles : cap;
  conv_igemm_persistent_kernel<BN, ST, S3, F16><<<grid, 384, S::TOTAL, st>>>(kp, total_tiles, n_tiles);
  DIM_LAUNCH_CHECK();
  return 0;
}

template <int N, int ST, bool S3, bool F16>
static int launch_conv1(const ConvKParams &kp, int grid, int rows_total, int rpc, int chunks, cudaStream_t st) {
  using S = Conv1Smem<N, ST, S3>;
  static bool set = false;
  if (!set) {
    DIM_CHECK(cudaFuncSetAttribute(conv1_kernel<N, ST, S3, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    set = true;
  }
  conv1_kernel<N, ST, S3, F16><<<grid, 384, S::TOTAL, st>>>(kp, rows_total, rpc, chunks);
  DIM_LAUNCH_CHECK();
  return 0;
}

template <int ST, bool S3, bool F16, int NB>
static int launch_conv1_rgbd(const ConvKParams &kp, int grid, int rows_total, int rpc, int chunks, int strip_bytes,
                             cudaStream_t st) {
  const int smem_bytes = 16 * NB * 128 * (S3 ? 2 : 1) + ST * (S3 ? 2 : 1) * strip_bytes + kConv1Slack + 1024 + 256;
  DIM_REQUIRE(smem_bytes <= 227 * 1024, "conv1 (RGB-D): image too wide for the rolling-strip ring");
  static int set = 0;
  if (set < smem_bytes) {
    DIM_CHECK(cudaFuncSetAttribute(conv1_rgbd_kernel<ST, S3, F16, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   smem_bytes));
    set = smem_bytes;
  }
  conv1_rgbd_kernel<ST, S3, F16, NB><<<grid, 384, smem_bytes, st>>>(kp, rows_total, rpc, chunks, strip_bytes);
  DIM_LAUNCH_CHECK();
  return 0;
}

// switches conv1 between the 8-channel and the 10-channel (RGB-D) input; only before any weights are loaded.  The wider
// input buffer is allocated on the first switch and kept.
int net_set_input_depth(dim_ctx *ctx, bool enable) {
  NetState *ns = ctx->net;
  DIM_REQUIRE(ns != nullptr, "net not created");
  if (ns->input_depth == enable) return 0;
  DIM_REQUIRE(!ns->loaded, "dim_ctx_set_input_depth: call it before dim_net_load (this context's weights are loaded)");
  if (!ns->act0_rgb_hi) { ns->act0_rgb_hi = ns->act_hi[0]; ns->act0_rgb_lo = ns->act_lo[0]; }
  ns->input_depth = enable;
  build_geometry(ns, ctx->H, ctx->W);
  ns->maps.clear();
  const LayerGeom &g = ns->g[0];
  const size_t per = (size_t)g.rows * g.cols * g.Cbuf;
  ns->act_elems_per_image[0] = per;
  if (enable && ns->net_ok && !ns->act0_rgbd_hi) {
    if (int rc = dev_alloc(ctx, &ns->act0_rgbd_hi, per * ctx->max_batch, true)) return rc;
    if (int rc = dev_alloc(ctx, &ns->act0_rgbd_lo, per * ctx->max_batch, true)) return rc;
  }
  ns->act_hi[0] = enable ? ns->act0_rgbd_hi : ns->act0_rgb_hi;
  ns->act_lo[0] = enable ? ns->act0_rgbd_lo : ns->act0_rgb_lo;
  return 0;
}

bool net_input_depth(dim_ctx *ctx) { return ctx->net && ctx->net->input_depth; }

// switches flow_conv1 between the 8-channel and the 6-channel (image-only) weight; only before any weights are loaded.
// Nothing else changes: the input buffer, its geometry and conv1_kernel are the 8-channel ones.
int net_set_input_mask(dim_ctx *ctx, bool enable) {
  NetState *ns = ctx->net;
  DIM_REQUIRE(ns != nullptr, "net not created");
  if (ns->input_mask == enable) return 0;
  DIM_REQUIRE(!ns->loaded, "dim_ctx_set_input_mask: call it before dim_net_load (this context's weights are loaded)");
  ns->input_mask = enable;
  return 0;
}

bool net_input_mask(dim_ctx *ctx) { return !ctx->net || ctx->net->input_mask; }

// where conv1's input buffer expects pixel (i,j) of the 8-channel blob (space-to-depth, pad 3)
void net_input_geometry(dim_ctx *ctx, int *rows, int *cols, int *pad, __nv_bfloat16 **hi, __nv_bfloat16 **lo) {
  NetState *ns = ctx->net;
  *rows = ns->g[0].rows; *cols = ns->g[0].cols; *pad = ns->g[0].py;
  *hi = ns->act_hi[0]; *lo = ns->act_lo[0];
}

// runs conv tower + fc6 + head on the already-filled conv1 input buffer
int net_forward(dim_ctx *ctx, int B, int precision, const float *zoom_factor, float *rot_out, float *trans_out,
                float *se3_out, cudaStream_t st, cudaEvent_t after_conv) {
  NetState *ns = ctx->net;
  DIM_REQUIRE(ns && ns->loaded, "dim_net_load has not been called");
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch, "batch exceeds max_batch");
  DIM_REQUIRE(precision == DIM_PREC_BF16 || precision == DIM_PREC_BF16X3 || precision == DIM_PREC_FP16,
              "unknown precision (DIM_PREC_BF16 / DIM_PREC_BF16X3 / DIM_PREC_FP16)");
  const bool s3 = precision == DIM_PREC_BF16X3, f16 = precision == DIM_PREC_FP16;
  const int key = B + (f16 ? kF16MapKey : 0);
  auto it = ns->maps.find(key);
  if (it == ns->maps.end()) {
    TensorMaps tm;
    if (int rc = build_maps(ns, B, f16, tm)) return rc;
    it = ns->maps.emplace(key, tm).first;
  }
  const TensorMaps &tm = it->second;
  if (ns->repack_done) DIM_CHECK(cudaStreamWaitEvent(st, ns->repack_done, 0));
  if (s3 && ns->lo_stale)
    if (int rc = train_refresh_lo(ctx, st)) return rc;
  if (f16 && ns->f16_stale)
    if (int rc = train_refresh_f16(ctx, st)) return rc;
  if (ns->layer_events) DIM_CHECK(cudaEventRecord(ns->layer_events[0], st));
  for (int i = 0; i < 10; ++i) {
    const LayerGeom &g = ns->g[i];
    const ConvKParams &kp = tm.kp[i];
    const int n_tiles = g.Cout / g.BLOCK_N;
    const int total_tiles = cdiv(B * g.Hq, g.BH) * g.n_col_tiles * n_tiles;
    const int sms = ctx->num_sms;
    int rc;
    if (i == 0 && ns->input_depth) {
      // RGB-D conv1: the same rolling strips, 8 chunk planes per strip; bf16x3 splits the output channels four ways
      const int nsplit = s3 ? 4 : 1;
      const int rows_total = B * g.Hq;
      int chunks = sms / (g.n_col_tiles * nsplit);
      if (chunks > cdiv(rows_total, 16)) chunks = cdiv(rows_total, 16);
      if (chunks < 1) chunks = 1;
      const int rpc = cdiv(rows_total, chunks);
      chunks = cdiv(rows_total, rpc);
      const int strip_bytes = cdiv((g.BW + 3) * 128, 128) * 128;
      const int grid = g.n_col_tiles * chunks * nsplit;
      rc = s3 ? launch_conv1_rgbd<5, true, false, 16>(kp, grid, rows_total, rpc, chunks, strip_bytes, st)
              : (f16 ? launch_conv1_rgbd<6, false, true, 64>(kp, grid, rows_total, rpc, chunks, strip_bytes, st)
                     : launch_conv1_rgbd<6, false, false, 64>(kp, grid, rows_total, rpc, chunks, strip_bytes, st));
    } else if (i == 0) {
      // conv1: a CTA walks down a run of output rows of one column tile (N = 160 pixels, bf16x3: 80), one new input strip
      // per row.  Built for the network's 480 x 640 input: Wo = 320 is a whole number of column tiles.
      // The kernel skips the strips past the input's last row (row B * Hq): they must feed only virtual rows.
      DIM_REQUIRE(g.Wo == 320 && g.cols >= g.Wo + 3 && g.Hq == g.rows && g.Hq == g.Ho + 3,
                  "conv1_kernel is built for a 480x640 input (320 output columns)");
      const int n_col = g.Wo / (s3 ? 80 : 160);
      const int rows_total = B * g.Hq;
      int chunks = sms / n_col;
      if (chunks > cdiv(rows_total, 16)) chunks = cdiv(rows_total, 16);  // keep the 3-row halo below ~20 %
      if (chunks < 1) chunks = 1;
      const int rpc = cdiv(rows_total, chunks);
      chunks = cdiv(rows_total, rpc);
      const int grid = n_col * chunks;
      rc = s3 ? launch_conv1<80, 5, true, false>(kp, grid, rows_total, rpc, chunks, st)
              : (f16 ? launch_conv1<160, 8, false, true>(kp, grid, rows_total, rpc, chunks, st)
                     : launch_conv1<160, 8, false, false>(kp, grid, rows_total, rpc, chunks, st));
    } else if (g.BLOCK_N == 128) {
      rc = s3 ? launch_conv<128, 3, true, false>(kp, total_tiles, n_tiles, sms, st)
              : (f16 ? launch_conv<128, 6, false, true>(kp, total_tiles, n_tiles, sms, st)
                     : launch_conv<128, 6, false, false>(kp, total_tiles, n_tiles, sms, st));
    } else {
      rc = s3 ? launch_conv<256, 2, true, false>(kp, total_tiles, n_tiles, sms, st)
              : (f16 ? launch_conv<256, 4, false, true>(kp, total_tiles, n_tiles, sms, st)
                     : launch_conv<256, 4, false, false>(kp, total_tiles, n_tiles, sms, st));
    }
    if (rc) return rc;
    if (ns->layer_events && i < 9) DIM_CHECK(cudaEventRecord(ns->layer_events[i + 1], st));
  }
  if (ns->layer_events) DIM_CHECK(cudaEventRecord(ns->layer_events[10], st));
  if (after_conv) DIM_CHECK(cudaEventRecord(after_conv, st));
  if (s3)
    fc6_mma_kernel<true><<<FC6_SPLITS, 256, 0, st>>>(ns->act_hi[10], ns->act_lo[10], ns->fc6_w_hi, ns->fc6_w_lo, B,
                                                     ctx->max_batch, ns->fc6_partial);
  else if (f16)
    fc6_mma_kernel<false, true><<<FC6_SPLITS, 256, 0, st>>>(ns->act_hi[10], nullptr, ns->fc6_w_f16, nullptr, B,
                                                            ctx->max_batch, ns->fc6_partial);
  else
    fc6_mma_kernel<false><<<FC6_SPLITS, 256, 0, st>>>(ns->act_hi[10], nullptr, ns->fc6_w_hi, nullptr, B,
                                                      ctx->max_batch, ns->fc6_partial);
  DIM_LAUNCH_CHECK();
  head_kernel<<<B, 1024, 0, st>>>(ns->fc6_partial, ctx->max_batch, ns->fc6_b, ns->fc7_wT, ns->fc7_b, ns->rot_w,
                                 ns->rot_b, ns->trans_w, ns->trans_b, zoom_factor, rot_out, trans_out, se3_out, ns->save_h6,
                                 ns->save_h7);
  DIM_LAUNCH_CHECK();
  return 0;
}

// the refinement chain may be captured into a CUDA graph only when nothing host-dependent hangs on the forward pass
bool net_graph_safe(dim_ctx *ctx) {
  NetState *ns = ctx->net;
  return ns && ns->loaded && !ns->layer_events && !ns->train_aliased;
}

// tuning hook: per-layer device times of the LAST net_forward (11 events: before conv1, after each of the 10 layers)
int net_layer_profile(dim_ctx *ctx, int enable, float *ms10) {
  NetState *ns = ctx->net;
  DIM_REQUIRE(ns != nullptr, "net not created");
  if (enable && !ns->layer_events) {
    ns->layer_events = new cudaEvent_t[11];
    for (int i = 0; i < 11; ++i) DIM_CHECK(cudaEventCreate(&ns->layer_events[i]));
  }
  if (ms10 && ns->layer_events) {
    DIM_CHECK(cudaDeviceSynchronize());
    for (int i = 0; i < 10; ++i) DIM_CHECK(cudaEventElapsedTime(&ms10[i], ns->layer_events[i], ns->layer_events[i + 1]));
  }
  if (!enable && ns->layer_events) {
    for (int i = 0; i < 11; ++i) cudaEventDestroy(ns->layer_events[i]);
    delete[] ns->layer_events;
    ns->layer_events = nullptr;
  }
  return 0;
}

// debugging / test hook: copy the bf16 activation buffer (input of layer `idx`, 10 = fc6 input) to host
int net_debug_activation(dim_ctx *ctx, int idx, int lo, void *host_dst, size_t bytes) {
  NetState *ns = ctx->net;
  DIM_REQUIRE(ns && idx >= 0 && idx <= 10, "bad activation index");
  const size_t have = ns->act_elems_per_image[idx] * ctx->max_batch * 2;
  DIM_REQUIRE(bytes <= have, "activation copy larger than buffer");
  DIM_CHECK(cudaMemcpy(host_dst, lo ? ns->act_lo[idx] : ns->act_hi[idx], bytes, cudaMemcpyDeviceToHost));
  return 0;
}

void net_layer_geometry(dim_ctx *ctx, int idx, int *out /*rows, cols, Cbuf, py, px, Ho, Wo, Cout*/) {
  NetState *ns = ctx->net;
  if (idx < 10) {
    const LayerGeom &g = ns->g[idx];
    out[0] = g.rows; out[1] = g.cols; out[2] = g.Cbuf; out[3] = g.py; out[4] = g.px; out[5] = g.Ho; out[6] = g.Wo;
    out[7] = g.Cout;
  } else {
    const LayerGeom &g = ns->g[9];
    out[0] = g.Ho; out[1] = g.Wo; out[2] = g.Cout; out[3] = 0; out[4] = 0; out[5] = 0; out[6] = 0; out[7] = 256;
  }
}

}  // namespace dim
