// conv_igemm.cuh -- implicit-GEMM convolution on Hopper tensor cores (wgmma.mma_async, fp32 accumulators in
// registers) fed by TMA (cp.async.bulk.tensor) through an mbarrier ring.  sm_90a.
//
// Replaces the cuDNN Convolution + LeakyReLU(0.1) pairs of the FlowNetS tower
// (deepim/symbols/deepIM_flownet.py:63-107).
//
// Data layout (DESIGN.md "HBM layout"): activations are NHWC bf16 in buffers that carry the
// convolution's zero border physically ([B, Hp, Wp, C], interior at (py,px)) and images are stacked
// along the row axis, so one 3-D tensor map (C, cols, B*rows) addresses every tap with in-bounds
// coordinates.  For a stride-2 layer the buffer is read through four parity views (row parity,
// col parity): tap (kh,kw) = (2dh+ph, 2dw+pw) of output pixel (g,ow) is element (g+dh, ow+dw) of view
// (ph,pw).  An M tile is a BW x BH rectangle of output pixels (BW*BH <= 128), i.e. exactly one TMA
// box per tap, landing in shared memory as the K-major 128B-swizzled operand tile wgmma expects.
// Weights are [Cout][kh][kw][Cin] bf16 (K-major), one 2-D tensor map.
//
// Warp roles (384 threads = 3 warpgroups): warp 0 = TMA producer (elected lane), warpgroups 1 and 2 = consumers.  Each
// consumer issues the wgmmas of 64 of the tile's 128 rows (M = 64 per instruction) into its own register accumulator and
// runs the epilogue for them (bias + LeakyReLU -> bf16 NHWC stores into the next layer's bordered buffer).  The producer
// keeps loading the next tile while the consumers drain the current one.
//
// SPLIT3 = bf16x3 precision mode: operands are hi/lo bf16 pairs (x = hi + lo); each K step issues
// hi*hi + lo*hi + hi*lo into the same fp32 accumulator (error ~2^-16 relative, near-fp32).
// F16 = fp16 precision mode (DIM_PREC_FP16): the same one-pass kernels with IEEE half operands (11 significant bits
// instead of bf16's 8) and epilogues that store saturating fp16; the 16-bit activation / weight buffers are shared with
// the bf16 modes (typed __nv_bfloat16* in the signatures, the bits are whatever the mode stores).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include "common.cuh"
#include "wgmma.cuh"

namespace dim {

struct ConvKParams {
  CUtensorMap a_map[4];     // activation views (hi); [0] only for stride 1
  CUtensorMap a_lo_map[4];  // activation views (lo), SPLIT3 only
  CUtensorMap b_map;        // weights hi (fp16 pack in F16 mode)
  CUtensorMap b_lo_map;     // weights lo
  int KH, KW, stride, cchunks;  // taps and channel chunks (Cin_eff / BLOCK_K)
  int BW, BH, n_col_tiles;
  int Hq, Ho, Wo, Bn;           // virtual rows per image, valid output extent, batch
  int out_Hp, out_Wp, out_py, out_px, Cout;
  int kblocks;
  float slope;
  const float *bias;
  __nv_bfloat16 *out_hi, *out_lo;
  // ---- generic epilogue (EPI = 1: decoder deconvolutions as parity sub-convolutions, data gradients)
  //   TMA coordinates get (in_off_c, in_off_r) added; virtual output pixel (oh, ow) of image n lands at
  //   interior pixel (oh*out_sy + out_oy, ow*out_sx + out_ox) of the output buffer when that is inside
  //   [0,out_H) x [0,out_W);  value = (acc + bias + addend) then LeakyReLU (mask.p == nullptr, slope 1 = none)
  //   or * (mask > 0 ? 1 : slope) for channels < mask_climit (LeakyReLU backward through the stored
  //   activation).  All side buffers are bf16 NHWC with their own border / channel stride.
  int in_off_r, in_off_c;
  int out_sy, out_sx, out_oy, out_ox, out_H, out_W, out_cs, out_coff;
  struct PixBuf { const __nv_bfloat16 *p; int Hp, Wp, py, px, cs, coff; } addend, mask;
  int mask_climit;
};

namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// One lane of a CONVERGED warp.  The TMA producer runs its loop with all 32 lanes (warp-uniform control flow and
// operands) and only the instruction that must be issued once sits under elect.sync: descriptors, coordinates and barrier
// addresses then live in uniform registers instead of being re-broadcast around every issue from `if (lane == 0)`.
// Every function below that says "elected lane" must be called by all 32 lanes of the warp.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\telect.sync _|p, 0xFFFFFFFF;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx_raw(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d_raw(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d_raw(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::
          "r"(smem_u32(dst)),
      "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// elected lane
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  if (elect_one())
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap *m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)m) : "memory");
}
// elected lane
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1) {
  if (elect_one())
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// elected lane
__device__ __forceinline__ void tma_load_3d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, int c2) {
  if (elect_one())
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::
            "r"(smem_u32(dst)),
        "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// elected lane
__device__ __forceinline__ void tma_load_4d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, int c2, int c3) {
  if (elect_one())
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::
            "r"(smem_u32(dst)),
        "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// wgmma shared-memory operand descriptor (PTX ISA "matrix descriptor"): start >> 4 in [0,14), leading byte offset >> 4 in
// [16,30), stride byte offset >> 4 in [32,46), layout in [62,64) (0 = no swizzle, 1 = 128B, 2 = 64B swizzle).
//   K-major, swizzled : SBO = 8 rows * row bytes, LBO unused (1)
//   K-major, none     : core matrices of 8 rows x 16 B; LBO = bytes between K-adjacent core matrices, SBO = between 8-row groups
//   MN-major, swizzled: LBO = bytes between 64- (128B) / 32-element (64B) groups along M/N, SBO = between groups of 8 K rows
// A descriptor advanced by `bytes` is desc + (bytes >> 4): the 14-bit start field cannot carry below 256 KB.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)layout << 62;
  return d;
}
constexpr uint32_t kSW128 = 1u, kSW64 = 2u, kNoSwizzle = 0u;

// register split between the producer warpgroup and the two consumer warpgroups (128 * 40 + 256 * 232 <= 64 K)
__device__ __forceinline__ void regs_producer() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void regs_consumer() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }

}  // namespace ptx

// two fp32 -> packed 16-bit pair (element 0 in the low half).  fp16 saturates to +-65504 instead of
// overflowing to inf (the reference computes in fp32: a finite value must stay finite).
__device__ __forceinline__ uint32_t pack2_f16(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
__device__ __forceinline__ uint32_t pack2_bf16(float a, float b) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}

// conv1: MMA rows >= BW of the last ring slot read up to (128 - BW) * 16 bytes past it
constexpr int kConv1Slack = 2048;


// Rows of the m64nN accumulator fragment owned by thread `t` of a warpgroup: row0 and row0 + 8; columns 8j + 2(t & 3) (+1).
__device__ __forceinline__ int frag_row(int t) { return ((t >> 5) << 4) + ((t & 31) >> 2); }

// One fragment row pair (j-th 8-column group) of the forward epilogue: + bias, LeakyReLU, 16-bit store (hi[, lo]).
template <bool SPLIT3, bool F16>
__device__ __forceinline__ void store_pair(float v0, float v1, float2 b, float slope, __nv_bfloat16 *out_hi, __nv_bfloat16 *out_lo,
                                           long long off) {
  v0 += b.x;
  v1 += b.y;
  v0 = v0 > 0.f ? v0 : v0 * slope;
  v1 = v1 > 0.f ? v1 : v1 * slope;
  if (F16) {
    *reinterpret_cast<uint32_t *>(out_hi + off) = pack2_f16(v0, v1);
  } else {
    const uint32_t h = pack2_bf16(v0, v1);
    *reinterpret_cast<uint32_t *>(out_hi + off) = h;
    if (SPLIT3)
      *reinterpret_cast<uint32_t *>(out_lo + off) = pack2_bf16(v0 - __uint_as_float(h << 16), v1 - __uint_as_float(h & 0xFFFF0000u));
  }
}

// generic epilogue of the training-step kernels (see ConvKParams): two channels n, n + 1 of one output pixel
__device__ __forceinline__ void store_pair_generic(float v0, float v1, const ConvKParams &p, int n, bool valid, long long off,
                                                   long long add_off, long long mask_off) {
  if (!valid || n >= p.Cout) return;
  if (p.bias) {
    v0 += __ldg(p.bias + n);
    v1 += __ldg(p.bias + n + 1);
  }
  if (p.addend.p) {
    const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162 *>(p.addend.p + add_off);
    v0 += __low2float(a);
    v1 += __high2float(a);
  }
  if (p.mask.p) {
    if (n < p.mask_climit) {
      const __nv_bfloat162 m = *reinterpret_cast<const __nv_bfloat162 *>(p.mask.p + mask_off);
      if (!(__low2float(m) > 0.f)) v0 *= p.slope;
      if (!(__high2float(m) > 0.f)) v1 *= p.slope;
    }
  } else {
    v0 = v0 > 0.f ? v0 : v0 * p.slope;
    v1 = v1 > 0.f ? v1 : v1 * p.slope;
  }
  *reinterpret_cast<__nv_bfloat162 *>(p.out_hi + off) = __floats2bfloat162_rn(v0, v1);
}

// ---------------------------------------------------------------------------------------------
// Persistent, warp-specialised implicit GEMM.  grid = min(#tiles, SMs); CTA c walks tiles c, c+G, c+2G ... (tile id =
// m*Nn + n, n fastest so CTAs that share an activation tile run side by side and hit it in L2 together).  The smem ring
// runs across tile boundaries: the producer is already loading tile t+1 while the consumers store tile t.  A consumer
// keeps one K block of wgmmas in flight (wait_group 1) and hands the stage of the previous block back to the producer.
template <int BLOCK_N, int STAGES, bool SPLIT3>
struct ConvSmem2 {
  static constexpr int A_BYTES = 128 * 64 * 2;
  static constexpr int B_BYTES = BLOCK_N * 64 * 2;
  static constexpr int NPREC = SPLIT3 ? 2 : 1;
  static constexpr int STAGE_BYTES = (A_BYTES + B_BYTES) * NPREC;
  static constexpr int TOTAL = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

template <int BLOCK_N, int STAGES, bool SPLIT3, bool F16, int EPI = 0>
__global__ void __launch_bounds__(384, 1) conv_igemm_persistent_kernel(const __grid_constant__ ConvKParams p,
                                                                       const int total_tiles, const int n_tiles) {
  using S = ConvSmem2<BLOCK_N, STAGES, SPLIT3>;
  constexpr uint32_t SBO = 1024u;

  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + STAGES * S::STAGE_BYTES);
  uint64_t *empty_bar = full_bar + STAGES;

  const int wgi = threadIdx.x >> 7, warp = threadIdx.x >> 5;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);  // one arrive per consumer warpgroup
    }
    ptx::fence_barrier_init();
    ptx::prefetch_tmap(&p.b_map);
    ptx::prefetch_tmap(&p.a_map[0]);
  }
  __syncthreads();

  if (wgi == 0) {
    ptx::regs_producer();
    if (warp == 0) {
      // ------------------------------------------------------------------ TMA producer (whole warp, elected lane issues)
      const uint32_t tx = (uint32_t)(p.BW * p.BH * 64 * 2 + BLOCK_N * 64 * 2) * S::NPREC;
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nt = tile % n_tiles, mt = tile / n_tiles;
        const int col_tile = mt % p.n_col_tiles, row_tile = mt / p.n_col_tiles;
        const int g0 = row_tile * p.BH, ow0 = col_tile * p.BW, n0 = nt * BLOCK_N;
        for (int kb = 0; kb < p.kblocks; ++kb) {
          ptx::mbar_wait(&empty_bar[s], ph ^ 1u);
          const int tap = kb / p.cchunks, cc = kb - tap * p.cchunks;
          const int kh = tap / p.KW, kw = tap - kh * p.KW;
          int view = 0, dr = kh, dc = kw;
          if (p.stride == 2) {
            view = ((kh & 1) << 1) | (kw & 1);
            dr = kh >> 1;
            dc = kw >> 1;
          }
          uint8_t *st = smem + s * S::STAGE_BYTES;
          if (EPI) { dr += p.in_off_r; dc += p.in_off_c; }
          if (ptx::elect_one()) {
            ptx::mbar_expect_tx_raw(&full_bar[s], tx);
            ptx::tma_load_3d_raw(st, &p.a_map[view], &full_bar[s], cc * 64, ow0 + dc, g0 + dr);
            ptx::tma_load_2d_raw(st + S::A_BYTES, &p.b_map, &full_bar[s], kb * 64, n0);
            if (SPLIT3) {
              ptx::tma_load_3d_raw(st + S::A_BYTES + S::B_BYTES, &p.a_lo_map[view], &full_bar[s], cc * 64, ow0 + dc, g0 + dr);
              ptx::tma_load_2d_raw(st + 2 * S::A_BYTES + S::B_BYTES, &p.b_lo_map, &full_bar[s], kb * 64, n0);
            }
          }
          __syncwarp();
          if (++s == STAGES) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else {
    ptx::regs_consumer();
    // ------------------------------------------------------------------ consumers: rows 64*(wgi-1) .. +63 of the M tile
    const int t = threadIdx.x & 127;
    const int half = wgi - 1;
    const int r0 = half * 64 + frag_row(t), q2 = (t & 3) * 2;
    const bool arriver = t == 0;
    const uint32_t base = ptx::smem_u32(smem);
    float acc[BLOCK_N / 2];
    int s = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int prev = -1;
      for (int kb = 0; kb < p.kblocks; ++kb) {
        ptx::mbar_wait(&full_bar[s], ph);
        const uint32_t a_hi = base + s * S::STAGE_BYTES + half * 8192;
        const uint32_t b_hi = base + s * S::STAGE_BYTES + S::A_BYTES;
        const uint64_t da0 = ptx::gmma_desc(a_hi, 16, SBO, ptx::kSW128), db0 = ptx::gmma_desc(b_hi, 16, SBO, ptx::kSW128);
        const uint64_t dal0 = da0 + ((S::A_BYTES + S::B_BYTES) >> 4), dbl0 = db0 + ((S::A_BYTES + S::B_BYTES) >> 4);
        wg::fence_acc(acc);
        wg::fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t da = da0 + (uint64_t)(2 * k), db = db0 + (uint64_t)(2 * k);  // + k * 32 bytes
          wg::mma<BLOCK_N, F16, 0, 0>(acc, da, db, (kb > 0 || k > 0) ? 1u : 0u);
          if (SPLIT3) {
            wg::mma<BLOCK_N, false, 0, 0>(acc, dal0 + (uint64_t)(2 * k), db, 1u);
            wg::mma<BLOCK_N, false, 0, 0>(acc, da, dbl0 + (uint64_t)(2 * k), 1u);
          }
        }
        wg::commit();
        wg::wait<1>();
        wg::fence_acc(acc);
        if (prev >= 0 && arriver) ptx::mbar_arrive(&empty_bar[prev]);
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1u; }
      }
      wg::wait<0>();
      wg::fence_acc(acc);
      if (prev >= 0 && arriver) ptx::mbar_arrive(&empty_bar[prev]);

      const int nt = tile % n_tiles, mt = tile / n_tiles;
      const int col_tile = mt % p.n_col_tiles, row_tile = mt / p.n_col_tiles;
      const int n0 = nt * BLOCK_N;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int m = r0 + rr * 8;
        const int bh = m / p.BW, bw = m - bh * p.BW;
        const int g = row_tile * p.BH + bh, ow = col_tile * p.BW + bw;
        const int n_img = g / p.Hq, oh = g - n_img * p.Hq;
        if (EPI == 1) {
          const int y = oh * p.out_sy + p.out_oy, x = ow * p.out_sx + p.out_ox;
          const bool valid = (m < p.BW * p.BH) && (n_img < p.Bn) && (oh < p.Ho) && (ow < p.Wo) && y >= 0 && y < p.out_H &&
                             x >= 0 && x < p.out_W;
          const long long off =
              (((long long)n_img * p.out_Hp + y + p.out_py) * p.out_Wp + x + p.out_px) * p.out_cs + p.out_coff + n0 + q2;
          const long long add_off =
              (((long long)n_img * p.addend.Hp + y + p.addend.py) * p.addend.Wp + x + p.addend.px) * p.addend.cs + p.addend.coff +
              n0 + q2;
          const long long mask_off =
              (((long long)n_img * p.mask.Hp + y + p.mask.py) * p.mask.Wp + x + p.mask.px) * p.mask.cs + p.mask.coff + n0 + q2;
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j)
            store_pair_generic(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1], p, n0 + 8 * j + q2, valid, off + 8 * j,
                               add_off + 8 * j, mask_off + 8 * j);
        } else {
          const bool valid = (m < p.BW * p.BH) && (n_img < p.Bn) && (oh < p.Ho) && (ow < p.Wo);
          if (valid) {
            const long long off = (((long long)n_img * p.out_Hp + oh + p.out_py) * p.out_Wp + ow + p.out_px) * p.Cout + n0 + q2;
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j)
              store_pair<SPLIT3, F16>(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1],
                                      make_float2(__ldg(p.bias + n0 + 8 * j + q2), __ldg(p.bias + n0 + 8 * j + q2 + 1)), p.slope, p.out_hi,
                                      p.out_lo, off + 8 * j);
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// conv1 (flow_conv1: 8 -> 64, 7x7 s2, i.e. 16 taps x 32 space-to-depth channels).  The generic path
// fetches every tap's operand tile from L2 separately (16x re-read of the input).  Here one TMA box per filter row dh
// brings the (BW+3)-pixel input strip into shared memory ONCE, in the un-swizzled K-major layout
//     addr(pixel r, channel-chunk c) = base + c*LBO + 16*r          (8-channel chunks of 16 B)
// in which the row index is linear in memory, so the four horizontal taps dw = 0..3 are the same
// strip read through descriptors whose start address is shifted by dw*16 bytes.
// Input buffer layout (written by the zoom kernel): [B*Hs rows][4 chunks][Ws cols][8 ch] bf16.
// Tile = one output row x BW output columns (BW <= 128; MMA rows >= BW are don't-care and read past the strip into the
// slack behind the ring).  Weights: the whole 64 x 512 matrix stays resident in shared memory (64B-swizzled, 16 tap tiles).
//
// Rolling strips: a CTA owns one column tile and a CONTIGUOUS run of output rows [g_lo, g_hi) and walks down it: output
// row t uses the input strips t .. t+3 (one per filter row dh), so moving to the next row needs ONE new strip; every strip
// travels L2 -> shared memory once (plus a 3-row halo per chunk).  The two consumer warpgroups take alternate rows (each
// the full M = 128 as two m64 halves) so that one runs its epilogue while the other's wgmmas run.  Strip s is used by rows
// s-3 .. s; the warpgroup of parity p is done with strips <= t+1 after its row t (its next row t+2 starts at strip t+2),
// so after row t it releases strips t and t+1: every strip gets one arrival from each warpgroup (the parity-1 warpgroup
// never uses strip 0 and releases it up front).
// Structurally-zero K steps are not issued: filter row 7 (dh = 3, odd input row) and filter column 7 (dw = 3, odd input
// column) lie outside the 7 x 7 filter, so dh = 3 has no second K step and dw = 3 has ONE step over the input chunks
// (0, 2) (weights packed in that order: conv1_kslot).
template <int STAGES, bool SPLIT3, bool F16>
__global__ void __launch_bounds__(384, 1) conv1_kernel(const __grid_constant__ ConvKParams p, const int rows_total,
                                                       const int rows_per_chunk, const int chunks_per_col,
                                                       const int strip_bytes /*per precision, multiple of 128*/) {
  constexpr int NPREC = SPLIT3 ? 2 : 1;
  constexpr int B_BYTES = 64 * 32 * 2, RES_BYTES = 16 * B_BYTES * NPREC;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t *res = smem;
  uint8_t *ring = smem + RES_BYTES;
  const int stage_bytes = strip_bytes * NPREC;
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(ring + STAGES * stage_bytes + kConv1Slack);
  uint64_t *empty_bar = full_bar + STAGES;
  uint64_t *res_bar = empty_bar + STAGES;

  const int wgi = threadIdx.x >> 7, warp = threadIdx.x >> 5;
  const int R = p.BW + 3;
  const uint32_t LBO = (uint32_t)R * 16u;
  const int ct = blockIdx.x / chunks_per_col, ck = blockIdx.x - ct * chunks_per_col;
  const int g_lo = ck * rows_per_chunk;
  const int g_hi = min(rows_total, g_lo + rows_per_chunk);
  const int n_rows = max(0, g_hi - g_lo);          // output rows (tiles) of this CTA
  const int n_strips = n_rows > 0 ? n_rows + 3 : 0;
  const int ow0 = ct * p.BW;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);
    }
    ptx::mbar_init(res_bar, 1);
    ptx::fence_barrier_init();
    ptx::prefetch_tmap(&p.b_map);
    ptx::prefetch_tmap(&p.a_map[0]);
  }
  __syncthreads();

  if (wgi == 0) {
    ptx::regs_producer();
    if (warp == 0 && n_rows > 0) {
      if (ptx::elect_one()) {
        ptx::mbar_expect_tx_raw(res_bar, (uint32_t)RES_BYTES);
        for (int kb = 0; kb < 16; ++kb) {
          ptx::tma_load_2d_raw(res + kb * B_BYTES, &p.b_map, res_bar, kb * 32, 0);
          if (SPLIT3) ptx::tma_load_2d_raw(res + (16 + kb) * B_BYTES, &p.b_lo_map, res_bar, kb * 32, 0);
        }
      }
      __syncwarp();
      const uint32_t tx = (uint32_t)(R * 64) * NPREC;
      for (int s = 0; s < n_strips; ++s) {
        const int slot = s % STAGES;
        ptx::mbar_wait(&empty_bar[slot], (((uint32_t)(s / STAGES)) & 1u) ^ 1u);
        uint8_t *st = ring + slot * stage_bytes;
        ptx::mbar_expect_tx(&full_bar[slot], tx);
        ptx::tma_load_4d(st, &p.a_map[0], &full_bar[slot], 0, ow0, 0, g_lo + s);
        if (SPLIT3) ptx::tma_load_4d(st + strip_bytes, &p.a_lo_map[0], &full_bar[slot], 0, ow0, 0, g_lo + s);
      }
    }
  } else if (n_rows > 0) {
    ptx::regs_consumer();
    const int set = wgi - 1, t = threadIdx.x & 127;
    const bool arriver = t == 0;
    const int r0 = frag_row(t), q2 = (t & 3) * 2;
    float2 bias[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) bias[j] = make_float2(__ldg(p.bias + 8 * j + q2), __ldg(p.bias + 8 * j + q2 + 1));
    const uint32_t ring_a = ptx::smem_u32(ring);
    // everything that does not depend on the row is formed once: ring-slot descriptor = dring + slot * slot_step
    const uint64_t dring = ptx::gmma_desc(ring_a, LBO, 128, ptx::kNoSwizzle);
    const uint64_t dring3 = ptx::gmma_desc(ring_a, 2u * LBO, 128, ptx::kNoSwizzle) + 3u;  // dw = 3: chunks 0 and 2, 3 pixels in
    const uint64_t lo_step = (uint64_t)((uint32_t)strip_bytes >> 4);
    const uint64_t slot_step = (uint64_t)((uint32_t)stage_bytes >> 4);
    const uint64_t kstep = (uint64_t)(2u * LBO >> 4);
    const uint64_t dres = ptx::gmma_desc(ptx::smem_u32(res), 16, 512, ptx::kSW64);
    const uint64_t dres_lo = dres + (uint64_t)((16 * B_BYTES) >> 4);
    const int n_cols_valid = min(p.BW, p.Wo - ow0);
    ptx::mbar_wait(res_bar, 0);
    if (set == 1 && arriver) ptx::mbar_arrive(&empty_bar[0]);
    for (int row = set; row < n_rows; row += 2) {
      float acc[2][32];
#pragma unroll
      for (int dh = 0; dh < 4; ++dh) {
        const int s = row + dh;
        ptx::mbar_wait(&full_bar[s % STAGES], ((uint32_t)(s / STAGES)) & 1u);
      }
      wg::fence_acc(acc[0]);
      wg::fence_acc(acc[1]);
      wg::fence();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int dh = 0; dh < 4; ++dh) {
          const uint64_t so = (uint64_t)((row + dh) % STAGES) * slot_step + (uint64_t)(h * 64);  // + 64 pixels of 16 B
#pragma unroll
          for (int k = 0; k < 2; ++k) {
#pragma unroll
            for (int dw = 0; dw < 4; ++dw) {
              if ((dh == 3 || dw == 3) && k == 1) continue;  // kh = 7 / kw = 7: outside the 7x7 filter, all-zero weights
              const uint64_t da = (dw == 3 ? dring3 : dring + (uint64_t)dw + (uint64_t)k * kstep) + so;
              const uint64_t wo = (uint64_t)((dh * 4 + dw) * (B_BYTES >> 4) + 2 * k);
              wg::mma<64, F16, 0, 0>(acc[h], da, dres + wo, (dh | dw | k) ? 1u : 0u);
              if (SPLIT3) {
                wg::mma<64, false, 0, 0>(acc[h], da + lo_step, dres + wo, 1u);
                wg::mma<64, false, 0, 0>(acc[h], da, dres_lo + wo, 1u);
              }
            }
          }
        }
      }
      wg::commit();
      wg::wait<0>();
      wg::fence_acc(acc[0]);
      wg::fence_acc(acc[1]);
      if (arriver) {
        ptx::mbar_arrive(&empty_bar[row % STAGES]);
        ptx::mbar_arrive(&empty_bar[(row + 1) % STAGES]);
      }
      const int g = g_lo + row;
      const int n_img = g / p.Hq, oh = g - n_img * p.Hq;
      if (n_img < p.Bn && oh < p.Ho) {
        const long long row_off = (((long long)n_img * p.out_Hp + oh + p.out_py) * p.out_Wp + ow0 + p.out_px) * 64 + q2;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int m = h * 64 + r0 + rr * 8;
            if (m < n_cols_valid) {
#pragma unroll
              for (int j = 0; j < 8; ++j)
                store_pair<SPLIT3, F16>(acc[h][4 * j + 2 * rr], acc[h][4 * j + 2 * rr + 1], bias[j], p.slope, p.out_hi, p.out_lo,
                                        row_off + (long long)m * 64 + 8 * j);
            }
          }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// conv1 of the RGB-D network (flow_conv1: 10 -> 64, 7x7 s2; deepIM_flownet.py:33-51 with INPUT_DEPTH).  Same rolling-strip
// schedule as conv1_kernel; the space-to-depth input has 16-channel chunks: each of the four 2x2 phases (ph, pw) is a pair
// of 8-channel chunk planes, channels 0-7 then 8-9 (+ 6 zero channels), so a strip is 8 chunk planes
//     addr(pixel r, plane c) = base + c*LBO + 16*r,  plane c = (ph*2 + pw)*2 + half
// and K step k (16 channels) of tap (dh, dw) is exactly phase k = ph*2 + pw: planes 2k, 2k + 1.  Phases with kh = 7
// (dh = 3, ph = 1) or kw = 7 (dw = 3, pw = 1) lie outside the 7 x 7 filter and are not issued (49 of the 64 K steps run).
// Input buffer: [B*Hs rows][8 planes][Ws cols][8 ch] bf16 / fp16.  Weights: [64][16 taps][4 phases][16 ch] = K 1024,
// resident in shared memory as 16 SW128 tap tiles of NB x 64, loaded in boxes of 16 output channels.
// NB = output channels per CTA.  The 64 x 1024 16-bit weight matrix (128 KB) fits beside a 6-deep strip ring; bf16x3's hi +
// lo pair (256 KB) does not, so that mode runs NB = 16 (64 KB of weights) with four CTAs per (column tile, row run), each
// re-reading the strips from L2: the parity mode is correct rather than fast.
template <int STAGES, bool SPLIT3, bool F16, int NB>
__global__ void __launch_bounds__(384, 1) conv1_rgbd_kernel(const __grid_constant__ ConvKParams p, const int rows_total,
                                                            const int rows_per_chunk, const int chunks_per_col,
                                                            const int strip_bytes /*per precision, multiple of 128*/) {
  constexpr int NPREC = SPLIT3 ? 2 : 1;
  constexpr int TAP_BYTES = NB * 128, RES_BYTES = 16 * TAP_BYTES * NPREC;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t *res = smem;
  uint8_t *ring = smem + RES_BYTES;
  const int stage_bytes = strip_bytes * NPREC;
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(ring + STAGES * stage_bytes + kConv1Slack);
  uint64_t *empty_bar = full_bar + STAGES;
  uint64_t *res_bar = empty_bar + STAGES;

  const int wgi = threadIdx.x >> 7, warp = threadIdx.x >> 5;
  const int R = p.BW + 3;
  const uint32_t LBO = (uint32_t)R * 16u;
  const int per_split = p.n_col_tiles * chunks_per_col;
  const int nsplit = blockIdx.x / per_split, cidx = blockIdx.x - nsplit * per_split;
  const int ct = cidx / chunks_per_col, ck = cidx - ct * chunks_per_col;
  const int n0 = nsplit * NB;
  const int g_lo = ck * rows_per_chunk;
  const int g_hi = min(rows_total, g_lo + rows_per_chunk);
  const int n_rows = max(0, g_hi - g_lo);
  const int n_strips = n_rows > 0 ? n_rows + 3 : 0;
  const int ow0 = ct * p.BW;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);
    }
    ptx::mbar_init(res_bar, 1);
    ptx::fence_barrier_init();
    ptx::prefetch_tmap(&p.b_map);
    ptx::prefetch_tmap(&p.a_map[0]);
  }
  __syncthreads();

  if (wgi == 0) {
    ptx::regs_producer();
    if (warp == 0 && n_rows > 0) {
      if (ptx::elect_one()) {
        ptx::mbar_expect_tx_raw(res_bar, (uint32_t)RES_BYTES);
        for (int kb = 0; kb < 16; ++kb)
          for (int r = 0; r < NB / 16; ++r) {
            ptx::tma_load_2d_raw(res + kb * TAP_BYTES + r * 2048, &p.b_map, res_bar, kb * 64, n0 + r * 16);
            if (SPLIT3) ptx::tma_load_2d_raw(res + (16 + kb) * TAP_BYTES + r * 2048, &p.b_lo_map, res_bar, kb * 64, n0 + r * 16);
          }
      }
      __syncwarp();
      const uint32_t tx = (uint32_t)(R * 128) * NPREC;
      for (int s = 0; s < n_strips; ++s) {
        const int slot = s % STAGES;
        ptx::mbar_wait(&empty_bar[slot], (((uint32_t)(s / STAGES)) & 1u) ^ 1u);
        uint8_t *st = ring + slot * stage_bytes;
        ptx::mbar_expect_tx(&full_bar[slot], tx);
        ptx::tma_load_4d(st, &p.a_map[0], &full_bar[slot], 0, ow0, 0, g_lo + s);
        if (SPLIT3) ptx::tma_load_4d(st + strip_bytes, &p.a_lo_map[0], &full_bar[slot], 0, ow0, 0, g_lo + s);
      }
    }
  } else if (n_rows > 0) {
    ptx::regs_consumer();
    const int set = wgi - 1, t = threadIdx.x & 127;
    const bool arriver = t == 0;
    const int r0 = frag_row(t), q2 = (t & 3) * 2;
    float2 bias[NB / 8];
#pragma unroll
    for (int j = 0; j < NB / 8; ++j)
      bias[j] = make_float2(__ldg(p.bias + n0 + 8 * j + q2), __ldg(p.bias + n0 + 8 * j + q2 + 1));
    const uint32_t ring_a = ptx::smem_u32(ring);
    const uint64_t dring = ptx::gmma_desc(ring_a, LBO, 128, ptx::kNoSwizzle);
    const uint64_t lo_step = (uint64_t)((uint32_t)strip_bytes >> 4);
    const uint64_t slot_step = (uint64_t)((uint32_t)stage_bytes >> 4);
    const uint64_t phase_step = (uint64_t)(2u * LBO >> 4);  // two chunk planes
    const uint64_t dres = ptx::gmma_desc(ptx::smem_u32(res), 16, 1024, ptx::kSW128);
    const uint64_t dres_lo = dres + (uint64_t)((16 * TAP_BYTES) >> 4);
    const int n_cols_valid = min(p.BW, p.Wo - ow0);
    ptx::mbar_wait(res_bar, 0);
    if (set == 1 && arriver) ptx::mbar_arrive(&empty_bar[0]);
    for (int row = set; row < n_rows; row += 2) {
      float acc[2][NB / 2];
#pragma unroll
      for (int dh = 0; dh < 4; ++dh) {
        const int s = row + dh;
        ptx::mbar_wait(&full_bar[s % STAGES], ((uint32_t)(s / STAGES)) & 1u);
      }
      wg::fence_acc(acc[0]);
      wg::fence_acc(acc[1]);
      wg::fence();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int dh = 0; dh < 4; ++dh) {
          const uint64_t so = (uint64_t)((row + dh) % STAGES) * slot_step + (uint64_t)(h * 64);  // + 64 pixels of 16 B
#pragma unroll
          for (int k = 0; k < 4; ++k) {
#pragma unroll
            for (int dw = 0; dw < 4; ++dw) {
              if ((dh == 3 && (k >> 1)) || (dw == 3 && (k & 1))) continue;  // kh = 7 / kw = 7: outside the 7x7 filter
              const uint64_t da = dring + (uint64_t)k * phase_step + (uint64_t)dw + so;
              const uint64_t wo = (uint64_t)((dh * 4 + dw) * (TAP_BYTES >> 4) + 2 * k);
              wg::mma<NB, F16, 0, 0>(acc[h], da, dres + wo, (dh | dw | k) ? 1u : 0u);
              if (SPLIT3) {
                wg::mma<NB, false, 0, 0>(acc[h], da + lo_step, dres + wo, 1u);
                wg::mma<NB, false, 0, 0>(acc[h], da, dres_lo + wo, 1u);
              }
            }
          }
        }
      }
      wg::commit();
      wg::wait<0>();
      wg::fence_acc(acc[0]);
      wg::fence_acc(acc[1]);
      if (arriver) {
        ptx::mbar_arrive(&empty_bar[row % STAGES]);
        ptx::mbar_arrive(&empty_bar[(row + 1) % STAGES]);
      }
      const int g = g_lo + row;
      const int n_img = g / p.Hq, oh = g - n_img * p.Hq;
      if (n_img < p.Bn && oh < p.Ho) {
        const long long row_off = (((long long)n_img * p.out_Hp + oh + p.out_py) * p.out_Wp + ow0 + p.out_px) * 64 + n0 + q2;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int m = h * 64 + r0 + rr * 8;
            if (m < n_cols_valid) {
#pragma unroll
              for (int j = 0; j < NB / 8; ++j)
                store_pair<SPLIT3, F16>(acc[h][4 * j + 2 * rr], acc[h][4 * j + 2 * rr + 1], bias[j], p.slope, p.out_hi, p.out_lo,
                                        row_off + (long long)m * 64 + 8 * j);
            }
          }
      }
    }
  }
}

}  // namespace dim
