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
// runs the epilogue for them (bias + LeakyReLU -> 16-bit NHWC into the next layer's bordered buffer).  The producer
// keeps loading the next tile while the consumers drain the current one.
//
// Forward layers (EPI = 0) load each stage's activation tile as two boxes of BW x BH/2 pixels, one per consumer
// (shared-memory rows 0 and 64), so a consumer's rows are whole output rows even when BW does not divide 64 (BW = 20,
// 10: rows 60-63 of each half are never stored).  In fp16 / bf16 a consumer writes its packed results with stmatrix into a
// 128B-swizzled [64 px][64 ch] staging block per 64-channel group and one thread TMA-stores each block as one box through
// out_map, whose extent keeps the zero border, the virtual rows and images >= B from being written; the few boxes that run
// into the next image store those rows from the fragments.  The TMA stores drain while the next tile's wgmmas run.
// bf16x3 stores from the fragments: its hi + lo ring leaves no room for a staging tile.
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
  // output store maps (Cout, Wo, Ho, B) over the INTERIOR of the next layer's bordered buffer, box = 64 ch x a pixel
  // rectangle, SW128: conv1_kernel (hi, lo; kConv1StoreN x 1 px) and the fp16 / bf16 EPI = 0 conv_igemm kernels ([0];
  // BW x BH/2 px).  conv1_kernel also reads the space-to-depth input with plain bulk copies ([rows][4 chunks][in_cols][8 ch])
  CUtensorMap out_map[2];
  const __nv_bfloat16 *in_hi, *in_lo;
  int in_cols;
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
  //   activation).  All side buffers are bf16 NHWC with their own border / channel stride.  SPLIT3: the addend is
  //   read as hi + lo (lo at the same offset of addend.lo) and the result is stored as a hi / lo pair (out_hi, out_lo).
  int in_off_r, in_off_c;
  int out_sy, out_sx, out_oy, out_ox, out_H, out_W, out_cs, out_coff;
  struct PixBuf { const __nv_bfloat16 *p; int Hp, Wp, py, px, cs, coff; const __nv_bfloat16 *lo; } addend, mask;
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

// contiguous global -> shared copy (bytes and both addresses multiples of 16), completing on `bar`
__device__ __forceinline__ void bulk_load_raw(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// shared -> global tensor store (bulk-group completion: commit, then wait on the issuing thread)
__device__ __forceinline__ void tma_store_4d(const CUtensorMap *map, const void *src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"((uint64_t)map),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the committed stores have finished reading their shared-memory source
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... and their global writes are done
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// four 8x8 16-bit matrices, each stored transposed: fragment column c becomes the 16-byte row at lane (8 * matrix + c)'s address
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]),
               "r"(r[2]), "r"(r[3])
               : "memory");
}
// ... stored as they are: fragment row r becomes the 16-byte row at lane (8 * matrix + r)'s address
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]),
               "r"(r[3])
               : "memory");
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

// conv1_rgbd_kernel: MMA rows >= BW of the last ring slot read up to (128 - BW) * 16 bytes past it
constexpr int kConv1Slack = 2048;


// Rows of the m64nN accumulator fragment owned by thread `t` of a warpgroup: row0 and row0 + 8; columns 8j + 2(t & 3) (+1).
__device__ __forceinline__ int frag_row(int t) { return ((t >> 5) << 4) + ((t & 31) >> 2); }

// the bf16 residuals (v - hi) of a packed bf16 pair hi = pack2_bf16(v0, v1): hi + lo carries ~16 significant bits
__device__ __forceinline__ uint32_t pack2_bf16_lo(float v0, float v1, uint32_t hi) {
  return pack2_bf16(v0 - __uint_as_float(hi << 16), v1 - __uint_as_float(hi & 0xFFFF0000u));
}

// The forward epilogue of two accumulator values: + bias, LeakyReLU, packed 16-bit pair (hi[, lo]; element 0 low).
template <bool SPLIT3, bool F16>
__device__ __forceinline__ void epi_pack(float v0, float v1, float b0, float b1, float slope, uint32_t &hi, uint32_t &lo) {
  v0 += b0;
  v1 += b1;
  v0 = v0 > 0.f ? v0 : v0 * slope;
  v1 = v1 > 0.f ? v1 : v1 * slope;
  if (F16) {
    hi = pack2_f16(v0, v1);
  } else {
    hi = pack2_bf16(v0, v1);
    if (SPLIT3) lo = pack2_bf16_lo(v0, v1, hi);
  }
}

// One fragment row pair (j-th 8-column group) of the forward epilogue: + bias, LeakyReLU, 16-bit store (hi[, lo]).
template <bool SPLIT3, bool F16>
__device__ __forceinline__ void store_pair(float v0, float v1, float2 b, float slope, __nv_bfloat16 *out_hi, __nv_bfloat16 *out_lo,
                                           long long off) {
  uint32_t h, l = 0;
  epi_pack<SPLIT3, F16>(v0, v1, b.x, b.y, slope, h, l);
  *reinterpret_cast<uint32_t *>(out_hi + off) = h;
  if (SPLIT3) *reinterpret_cast<uint32_t *>(out_lo + off) = l;
}

// generic epilogue of the training-step kernels (see ConvKParams): two channels n, n + 1 of one output pixel.
// SPLIT3: the addend is hi + lo (exact in fp32) and the result is stored as a hi / lo pair split like epi_pack.  The mask
// reads the hi half only: its sign is the sign of hi + lo, because |lo| <= ulp(hi) / 2 and hi = 0 implies lo = 0.
template <bool SPLIT3>
__device__ __forceinline__ void store_pair_generic(float v0, float v1, const ConvKParams &p, int n, bool valid, long long off,
                                                   long long add_off, long long mask_off) {
  if (!valid || n >= p.Cout) return;
  if (p.bias) {
    v0 += __ldg(p.bias + n);
    v1 += __ldg(p.bias + n + 1);
  }
  if (p.addend.p) {
    const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162 *>(p.addend.p + add_off);
    if (SPLIT3) {
      const __nv_bfloat162 al = *reinterpret_cast<const __nv_bfloat162 *>(p.addend.lo + add_off);
      v0 += __low2float(a) + __low2float(al);
      v1 += __high2float(a) + __high2float(al);
    } else {
      v0 += __low2float(a);
      v1 += __high2float(a);
    }
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
  if (SPLIT3) {
    const uint32_t h = pack2_bf16(v0, v1);
    *reinterpret_cast<uint32_t *>(p.out_hi + off) = h;
    *reinterpret_cast<uint32_t *>(p.out_lo + off) = pack2_bf16_lo(v0, v1, h);
  } else {
    *reinterpret_cast<__nv_bfloat162 *>(p.out_hi + off) = __floats2bfloat162_rn(v0, v1);
  }
}

// ---------------------------------------------------------------------------------------------
// Persistent, warp-specialised implicit GEMM.  grid = min(#tiles, SMs); CTA c walks tiles c, c+G, c+2G ... (tile id =
// m*Nn + n, n fastest so CTAs that share an activation tile run side by side and hit it in L2 together).  The smem ring
// runs across tile boundaries: the producer is already loading tile t+1 while the consumers store tile t.  A consumer
// keeps one K block of wgmmas in flight (wait_group 1) and hands the stage of the previous block back to the producer.
// Layout: the ring, then (TMA_EPI) the two consumers' staging tiles, then the barriers.  A staging tile holds STG_GROUPS
// [64 px][64 ch] blocks of 8 KB: all of BLOCK_N when that fits beside the ring, else half of it, and the tile is stored in
// two rounds.
template <int BLOCK_N, int STAGES, bool SPLIT3, int EPI>
struct ConvSmem2 {
  static constexpr int A_BYTES = 128 * 64 * 2;
  static constexpr int B_BYTES = BLOCK_N * 64 * 2;
  static constexpr int NPREC = SPLIT3 ? 2 : 1;
  static constexpr int STAGE_BYTES = (A_BYTES + B_BYTES) * NPREC;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int LIMIT = 227 * 1024, FIXED = 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr bool TMA_EPI = EPI == 0 && !SPLIT3;
  static constexpr int STG_GROUPS =
      !TMA_EPI ? 0 : (RING_BYTES + 2 * BLOCK_N * 128 + FIXED <= LIMIT ? BLOCK_N / 64 : BLOCK_N / 128);
  static constexpr int STG_ROUNDS = TMA_EPI ? BLOCK_N / 64 / STG_GROUPS : 0;
  static constexpr int STG_BYTES = STG_GROUPS * 8192;  // per consumer warpgroup
  static constexpr int TOTAL = RING_BYTES + 2 * STG_BYTES + FIXED;
  static_assert(TOTAL <= LIMIT, "conv_igemm shared memory");
};

template <int BLOCK_N, int STAGES, bool SPLIT3, bool F16, int EPI = 0>
__global__ void __launch_bounds__(384, 1) conv_igemm_persistent_kernel(const __grid_constant__ ConvKParams p,
                                                                       const int total_tiles, const int n_tiles) {
  using S = ConvSmem2<BLOCK_N, STAGES, SPLIT3, EPI>;
  constexpr uint32_t SBO = 1024u;

  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t *stg = smem + S::RING_BYTES;
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(stg + 2 * S::STG_BYTES);
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
    if (S::TMA_EPI) ptx::prefetch_tmap(&p.out_map[0]);
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
            for (int pr = 0; pr < S::NPREC; ++pr) {
              uint8_t *sa = st + pr * (S::A_BYTES + S::B_BYTES);
              const CUtensorMap *am = pr ? &p.a_lo_map[view] : &p.a_map[view];
              ptx::tma_load_3d_raw(sa, am, &full_bar[s], cc * 64, ow0 + dc, g0 + dr);
              if (EPI == 0) ptx::tma_load_3d_raw(sa + S::A_BYTES / 2, am, &full_bar[s], cc * 64, ow0 + dc, g0 + dr + (p.BH >> 1));
              ptx::tma_load_2d_raw(sa + S::A_BYTES, pr ? &p.b_lo_map : &p.b_map, &full_bar[s], kb * 64, n0);
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
    const int q2 = (t & 3) * 2;
    const bool arriver = t == 0;
    const uint32_t base = ptx::smem_u32(smem);
    // TMA_EPI staging: stmatrix x4 of 8-channel groups (j, j + 1): matrix mi = lane / 8 is (pixels 16 * warp + 8 * (mi & 1)
    // .. +7, group j + mi / 2); lane addresses pixel 16 * warp + 8 * (mi & 1) + lane % 8, whose 16-byte chunk c of a 128-byte
    // row sits at c ^ (pixel % 8) (SW128, blocks 1024-byte aligned)
    uint8_t *my_stg = stg + half * S::STG_BYTES;
    const int lane = t & 31;
    const uint32_t st_addr = ptx::smem_u32(my_stg) + (uint32_t)((16 * (t >> 5) + 8 * ((lane >> 3) & 1) + (lane & 7)) * 128);
    const uint32_t st_sw = (uint32_t)(((lane >> 4) & 1) ^ (lane & 7));
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
      if constexpr (S::TMA_EPI) {
        // this warpgroup's box: output rows gs .. gs + BH/2 - 1 (virtual rows over the batch, BH/2 <= Hq: at most two
        // images), columns ow0 .. ow0 + BW - 1
        const int gs = row_tile * p.BH + half * (p.BH >> 1), ow0 = col_tile * p.BW;
        const int n_img = gs / p.Hq, oh = gs - n_img * p.Hq;
        const bool store0 = n_img < p.Bn && oh < p.Ho, store1 = n_img + 1 < p.Bn && oh + (p.BH >> 1) > p.Hq;
#pragma unroll
        for (int rd = 0; rd < S::STG_ROUNDS; ++rd) {
          if (arriver) ptx::bulk_wait_read0();  // the previous stores have left the staging tile
          ptx::named_bar_sync(1 + half, 128);
#pragma unroll
          for (int i = 0; i < S::STG_GROUPS * 4; ++i) {  // 8-channel groups j, j + 1 = chunks 2 (i & 3) (+1) of block i / 4
            const int j = rd * S::STG_GROUPS * 8 + 2 * i;
            const float *bj = p.bias + n0 + 8 * j + q2;
            const float b0 = __ldg(bj), b1 = __ldg(bj + 1), b2 = __ldg(bj + 8), b3 = __ldg(bj + 9);
            uint32_t h[4], unused;
            epi_pack<false, F16>(acc[4 * j + 0], acc[4 * j + 1], b0, b1, p.slope, h[0], unused);
            epi_pack<false, F16>(acc[4 * j + 2], acc[4 * j + 3], b0, b1, p.slope, h[1], unused);
            epi_pack<false, F16>(acc[4 * j + 4], acc[4 * j + 5], b2, b3, p.slope, h[2], unused);
            epi_pack<false, F16>(acc[4 * j + 6], acc[4 * j + 7], b2, b3, p.slope, h[3], unused);
            ptx::stmatrix_x4(st_addr + (uint32_t)((i >> 2) * 8192) + (((uint32_t)(2 * (i & 3)) ^ st_sw) << 4), h);
          }
          ptx::fence_proxy_async();  // the generic-proxy staging writes become visible to the TMA store
          ptx::named_bar_sync(1 + half, 128);
          if (arriver && store0) {
            for (int q = 0; q < S::STG_GROUPS; ++q)
              ptx::tma_store_4d(&p.out_map[0], my_stg + q * 8192, n0 + (rd * S::STG_GROUPS + q) * 64, ow0, oh, n_img);
            ptx::bulk_commit();
          }
        }
        if (store1) {
          // the box's rows past image n_img's virtual rows are rows of image n_img + 1; a box there would start at a negative
          // row, so they are stored from the fragments
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int lr = frag_row(t) + rr * 8, bh = lr / p.BW;
            const int oh1 = oh + bh - p.Hq, ow = ow0 + lr - bh * p.BW;
            if (lr < p.BW * (p.BH >> 1) && oh1 >= 0 && oh1 < p.Ho) {
              const long long off =
                  (((long long)(n_img + 1) * p.out_Hp + oh1 + p.out_py) * p.out_Wp + ow + p.out_px) * p.Cout + n0 + q2;
#pragma unroll
              for (int j = 0; j < BLOCK_N / 8; ++j)
                store_pair<false, F16>(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1],
                                       make_float2(__ldg(p.bias + n0 + 8 * j + q2), __ldg(p.bias + n0 + 8 * j + q2 + 1)), p.slope,
                                       p.out_hi, p.out_lo, off + 8 * j);
            }
          }
        }
      } else {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          // EPI = 0: row lr of this warpgroup's BW x BH/2 box; EPI = 1: row m of the BW x BH tile
          const int lr = frag_row(t) + rr * 8, m = EPI ? half * 64 + lr : lr;
          const bool in_tile = EPI ? m < p.BW * p.BH : lr < p.BW * (p.BH >> 1);
          const int bh = m / p.BW, bw = m - bh * p.BW;
          const int g = row_tile * p.BH + (EPI ? 0 : half * (p.BH >> 1)) + bh, ow = col_tile * p.BW + bw;
          const int n_img = g / p.Hq, oh = g - n_img * p.Hq;
          if (EPI == 1) {
            const int y = oh * p.out_sy + p.out_oy, x = ow * p.out_sx + p.out_ox;
            const bool valid = in_tile && (n_img < p.Bn) && (oh < p.Ho) && (ow < p.Wo) && y >= 0 && y < p.out_H &&
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
              store_pair_generic<SPLIT3>(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1], p, n0 + 8 * j + q2, valid, off + 8 * j,
                                 add_off + 8 * j, mask_off + 8 * j);
          } else {
            const bool valid = in_tile && (n_img < p.Bn) && (oh < p.Ho) && (ow < p.Wo);
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
    if (S::TMA_EPI && arriver) ptx::bulk_wait0();
  }
}

// ---------------------------------------------------------------------------------------------
// conv1 (flow_conv1: 8 -> 64, 7x7 s2, i.e. 16 taps x 32 space-to-depth channels), computed transposed:
//     D^T [64 Cout x N px] = W [64 x K] . X [K x N px]
// so the output pixels run along the wgmma N axis (N = 160 divides Wo = 320: no MMA column is wasted) and one m64nNk16 per K
// step covers a whole column tile.
//   A = the whole 64 x 512 weight matrix, resident in shared memory (64B-swizzled K-major, 16 tap tiles; conv1_kslot order).
//   B = the (N+3)-pixel input strip of one input row, in the un-swizzled K-major layout
//         addr(pixel r, channel-chunk c) = base + c*LBO + 16*r          (8-channel chunks of 16 B, LBO = (N+3)*16)
//       in which the pixel index is linear in memory, so the four horizontal taps dw = 0..3 are the same strip read through
//       descriptors whose start address is shifted by dw*16 bytes.  Input buffer layout (written by the zoom kernel):
//       [B*Hs rows][4 chunks][Ws cols][8 ch], so a strip is four contiguous runs of (N+3)*16 bytes, one bulk copy each.
//
// Rolling strips: a CTA owns one column tile and a CONTIGUOUS run of output rows [g_lo, g_hi) and walks down it: output
// row t uses the input strips t .. t+3 (one per filter row dh), so moving to the next row needs ONE new strip; every strip
// travels L2 -> shared memory once (plus a 3-row halo per run).  The two consumer warpgroups take alternate rows so that
// one runs its epilogue while the other's wgmmas run.  Strip s is used by rows s-3 .. s; the warpgroup of parity p is done
// with strips <= t+1 after its row t (its next row t+2 starts at strip t+2), so after row t it releases strips t and t+1:
// every strip gets one arrival from each warpgroup (the parity-1 warpgroup never uses strip 0 and releases it up front).
// Structurally-zero K steps are not issued: filter row 7 (dh = 3, odd input row) and filter column 7 (dw = 3, odd input
// column) lie outside the 7 x 7 filter, so dh = 3 has no second K step and dw = 3 has ONE step over the input chunks
// (0, 2) (weights packed in that order: conv1_kslot).  25 K steps per row, in the same order for every output element.
//
// Epilogue: bias + LeakyReLU + 16-bit pack in registers (epi_pack, the arithmetic of every forward epilogue), transposed
// into a per-warpgroup [N px][64 ch] staging tile with stmatrix .trans (128B-swizzled: conflict-free), then TMA-stored in
// boxes of kConv1StoreN pixels through a map that covers only the interior of the next layer's buffer, so the zero border
// cannot be written.  Virtual rows (oh >= Ho) are not stored.
//
// N = 160 for fp16 / bf16 (2 column tiles at Wo = 320); bf16x3's hi + lo weights take 128 KB, which leaves room for N = 80
// (4 column tiles) with a 5-deep hi + lo ring: a 6th stage would need 236 KB with the two warpgroups' hi + lo staging
// tiles, over the 227 KB a CTA may use.
//
// The bulk copies are not bounds-checked by the hardware (a tensor map would clip them), so strips past the input's last
// row are never loaded: the runs end 3 strips past their last output row, and at the end of the batch those 3 strips lie
// past the buffer; they feed only the last image's virtual rows.
constexpr int kConv1StoreN = 80;

template <int N, int STAGES, bool SPLIT3>
struct Conv1Smem {
  static constexpr int NPREC = SPLIT3 ? 2 : 1;
  static constexpr int TAP_BYTES = 64 * 32 * 2;                            // one 64 x 32 tap tile of the weights
  static constexpr int RES_BYTES = 16 * TAP_BYTES * NPREC;
  static constexpr int STG_BYTES = N * 128;                                // [N px][64 ch] 16-bit, per precision
  static constexpr int PLANE_BYTES = (N + 3) * 16;                         // one chunk plane of a strip (= LBO)
  static constexpr int STRIP_BYTES = (4 * PLANE_BYTES + 127) / 128 * 128;  // per precision
  static constexpr int STAGE_BYTES = STRIP_BYTES * NPREC;
  static constexpr int TOTAL = RES_BYTES + 2 * STG_BYTES * NPREC + STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(N % kConv1StoreN == 0 && N % 16 == 0 && STG_BYTES % 1024 == 0, "conv1 tile width");
  static_assert(TOTAL <= 227 * 1024, "conv1 shared memory");
};

template <int N, int STAGES, bool SPLIT3, bool F16>
__global__ void __launch_bounds__(384, 1) conv1_kernel(const __grid_constant__ ConvKParams p, const int rows_total,
                                                       const int rows_per_chunk, const int chunks_per_col) {
  using S = Conv1Smem<N, STAGES, SPLIT3>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t *res = smem;
  uint8_t *stg = res + S::RES_BYTES;  // consumer warpgroup w: hi tile at stg + w * NPREC * STG_BYTES, lo tile behind it
  uint8_t *ring = stg + 2 * S::NPREC * S::STG_BYTES;
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(ring + STAGES * S::STAGE_BYTES);
  uint64_t *empty_bar = full_bar + STAGES;
  uint64_t *res_bar = empty_bar + STAGES;

  const int wgi = threadIdx.x >> 7, warp = threadIdx.x >> 5;
  const int ct = blockIdx.x / chunks_per_col, ck = blockIdx.x - ct * chunks_per_col;
  const int g_lo = ck * rows_per_chunk;
  const int g_hi = min(rows_total, g_lo + rows_per_chunk);
  const int n_rows = max(0, g_hi - g_lo);          // output rows of this CTA
  const int n_strips = n_rows > 0 ? n_rows + 3 : 0;
  const int ow0 = ct * N;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);
    }
    ptx::mbar_init(res_bar, 1);
    ptx::fence_barrier_init();
    ptx::prefetch_tmap(&p.b_map);
    ptx::prefetch_tmap(&p.out_map[0]);
  }
  __syncthreads();

  if (wgi == 0) {
    ptx::regs_producer();
    if (warp == 0 && n_rows > 0) {
      if (ptx::elect_one()) {
        ptx::mbar_expect_tx_raw(res_bar, (uint32_t)S::RES_BYTES);
        for (int kb = 0; kb < 16; ++kb) {
          ptx::tma_load_2d_raw(res + kb * S::TAP_BYTES, &p.b_map, res_bar, kb * 32, 0);
          if (SPLIT3) ptx::tma_load_2d_raw(res + (16 + kb) * S::TAP_BYTES, &p.b_lo_map, res_bar, kb * 32, 0);
        }
      }
      __syncwarp();
      const size_t plane = (size_t)p.in_cols * 16;  // bytes between the chunk planes of one input row
      const uint8_t *src_hi = reinterpret_cast<const uint8_t *>(p.in_hi) + (size_t)ow0 * 16;
      const uint8_t *src_lo = reinterpret_cast<const uint8_t *>(p.in_lo) + (size_t)ow0 * 16;
      for (int s = 0; s < n_strips; ++s) {
        const int slot = s % STAGES;
        ptx::mbar_wait(&empty_bar[slot], (((uint32_t)(s / STAGES)) & 1u) ^ 1u);
        uint8_t *st = ring + slot * S::STAGE_BYTES;
        if (g_lo + s >= rows_total) {
          // past the input's last row (the input has Hq = rows_total / B rows per image): the last run's final three
          // strips feed only the last image's virtual rows, which are never stored, so nothing is read
          if (ptx::elect_one()) ptx::mbar_arrive(&full_bar[slot]);
        } else if (ptx::elect_one()) {
          ptx::mbar_expect_tx_raw(&full_bar[slot], (uint32_t)(4 * S::PLANE_BYTES * S::NPREC));
          const size_t row = (size_t)(g_lo + s) * 4 * plane;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            ptx::bulk_load_raw(st + c * S::PLANE_BYTES, src_hi + row + c * plane, S::PLANE_BYTES, &full_bar[slot]);
            if (SPLIT3)
              ptx::bulk_load_raw(st + S::STRIP_BYTES + c * S::PLANE_BYTES, src_lo + row + c * plane, S::PLANE_BYTES, &full_bar[slot]);
          }
        }
        __syncwarp();
      }
    }
  } else if (n_rows > 0) {
    ptx::regs_consumer();
    const int set = wgi - 1, t = threadIdx.x & 127, lane = t & 31;
    const bool leader = t == 0;
    // this thread's accumulator rows are output channels co and co + 8
    const int co = frag_row(t);
    const float b0 = __ldg(p.bias + co), b1 = __ldg(p.bias + co + 8);
    const uint32_t ring_a = ptx::smem_u32(ring);
    // everything that does not depend on the row is formed once: ring-slot descriptor = dring + slot * slot_step
    const uint64_t dring = ptx::gmma_desc(ring_a, S::PLANE_BYTES, 128, ptx::kNoSwizzle);
    const uint64_t dring3 = ptx::gmma_desc(ring_a, 2u * S::PLANE_BYTES, 128, ptx::kNoSwizzle) + 3u;  // dw = 3: chunks 0, 2
    const uint64_t lo_step = (uint64_t)(S::STRIP_BYTES >> 4);
    const uint64_t slot_step = (uint64_t)(S::STAGE_BYTES >> 4);
    const uint64_t kstep = (uint64_t)(2 * S::PLANE_BYTES >> 4);
    const uint64_t dres = ptx::gmma_desc(ptx::smem_u32(res), 16, 512, ptx::kSW64);
    const uint64_t dres_lo = dres + (uint64_t)((16 * S::TAP_BYTES) >> 4);
    // stmatrix x4 of column groups (2i, 2i + 1): matrix m = lane / 8 is (column group 2i + m / 2, channels 16 * warp + 8 * (m & 1)
    // .. +7); lane addresses row lane % 8 of it = pixel 16i + 8 * (m / 2) + lane % 8, 16-byte chunk 2 * warp + (m & 1), stored
    // at chunk ^ (pixel % 8) of the pixel's 128-byte row (SW128, tiles 1024-byte aligned)
    uint8_t *my_stg = stg + set * S::NPREC * S::STG_BYTES;
    const int st_px = ((lane >> 4) << 3) + (lane & 7), st_chunk = 2 * (t >> 5) + ((lane >> 3) & 1);
    const uint32_t st_addr = ptx::smem_u32(my_stg) + (uint32_t)(st_px * 128 + ((st_chunk ^ (lane & 7)) << 4));
    ptx::mbar_wait(res_bar, 0);
    if (set == 1 && leader) ptx::mbar_arrive(&empty_bar[0]);
    for (int row = set; row < n_rows; row += 2) {
      float acc[N / 2];
#pragma unroll
      for (int dh = 0; dh < 4; ++dh) {
        const int s = row + dh;
        ptx::mbar_wait(&full_bar[s % STAGES], ((uint32_t)(s / STAGES)) & 1u);
      }
      wg::fence_acc(acc);
      wg::fence();
#pragma unroll
      for (int dh = 0; dh < 4; ++dh) {
        const uint64_t so = (uint64_t)((row + dh) % STAGES) * slot_step;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
#pragma unroll
          for (int dw = 0; dw < 4; ++dw) {
            if ((dh == 3 || dw == 3) && k == 1) continue;  // kh = 7 / kw = 7: outside the 7x7 filter, all-zero weights
            const uint64_t db = (dw == 3 ? dring3 : dring + (uint64_t)dw + (uint64_t)k * kstep) + so;
            const uint64_t wo = (uint64_t)((dh * 4 + dw) * (S::TAP_BYTES >> 4) + 2 * k);
            wg::mma<N, F16, 0, 0>(acc, dres + wo, db, (dh | dw | k) ? 1u : 0u);
            if (SPLIT3) {
              wg::mma<N, false, 0, 0>(acc, dres + wo, db + lo_step, 1u);
              wg::mma<N, false, 0, 0>(acc, dres_lo + wo, db, 1u);
            }
          }
        }
      }
      wg::commit();
      wg::wait<0>();
      wg::fence_acc(acc);
      if (leader) {
        ptx::mbar_arrive(&empty_bar[row % STAGES]);
        ptx::mbar_arrive(&empty_bar[(row + 1) % STAGES]);
      }
      const int g = g_lo + row;
      const int n_img = g / p.Hq, oh = g - n_img * p.Hq;
      if (n_img < p.Bn && oh < p.Ho) {
        if (leader) ptx::bulk_wait_read0();  // this warpgroup's previous row has left the staging tile
        ptx::named_bar_sync(1 + set, 128);
#pragma unroll
        for (int i = 0; i < N / 16; ++i) {
          uint32_t h[4], l[4] = {0, 0, 0, 0};
          epi_pack<SPLIT3, F16>(acc[8 * i + 0], acc[8 * i + 1], b0, b0, p.slope, h[0], l[0]);
          epi_pack<SPLIT3, F16>(acc[8 * i + 2], acc[8 * i + 3], b1, b1, p.slope, h[1], l[1]);
          epi_pack<SPLIT3, F16>(acc[8 * i + 4], acc[8 * i + 5], b0, b0, p.slope, h[2], l[2]);
          epi_pack<SPLIT3, F16>(acc[8 * i + 6], acc[8 * i + 7], b1, b1, p.slope, h[3], l[3]);
          ptx::stmatrix_x4_trans(st_addr + (uint32_t)(i * 16 * 128), h);
          if (SPLIT3) ptx::stmatrix_x4_trans(st_addr + (uint32_t)(S::STG_BYTES + i * 16 * 128), l);
        }
        ptx::fence_proxy_async();  // the generic-proxy staging writes become visible to the TMA store
        ptx::named_bar_sync(1 + set, 128);
        if (leader) {
#pragma unroll
          for (int q = 0; q < N / kConv1StoreN; ++q) {
            ptx::tma_store_4d(&p.out_map[0], my_stg + q * kConv1StoreN * 128, 0, ow0 + q * kConv1StoreN, oh, n_img);
            if (SPLIT3)
              ptx::tma_store_4d(&p.out_map[1], my_stg + S::STG_BYTES + q * kConv1StoreN * 128, 0, ow0 + q * kConv1StoreN, oh, n_img);
          }
          ptx::bulk_commit();
        }
      }
    }
    if (leader) ptx::bulk_wait0();
  }
}

// ---------------------------------------------------------------------------------------------
// conv1 of the RGB-D network (flow_conv1: 10 -> 64, 7x7 s2; deepIM_flownet.py:33-51 with INPUT_DEPTH).  Same rolling-strip
// schedule as conv1_kernel, but with the pixels on the MMA M axis: a tile is one output row x BW <= 128 columns (MMA rows
// >= BW are don't-care and read past the strip into the slack behind the ring), each warpgroup issuing it as two m64 halves,
// with the strips loaded as 4-D TMA boxes and the output stored straight from the fragments.  The space-to-depth input has
// 16-channel chunks: each of the four 2x2 phases (ph, pw) is a pair of 8-channel chunk planes, channels 0-7 then 8-9 (+ 6 zero channels), so a strip is 8 chunk planes
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
