// conv_wgrad.cuh -- weight gradients of the convolutions / deconvolutions on wgmma (training step,
// SURVEY 8 row a10; replaces cuDNN's backward-filter behind mx.symbol.Convolution/Deconvolution).
//
//   dW[m][tap][n] = sum over pixels (b, y, x) of  Z[b, y, x, m] * A[b, y*s + kh, x*s + kw, n]
//
// i.e. per filter tap one GEMM with M = channels of Z (the output gradient dZ for a convolution, the input
// activation for a deconvolution), N = channels of A and the pixel index as the contraction dimension.
// Both operands are NHWC, so the contraction index is the STRIDED one: the tiles are MN-major (transposed)
// wgmma operands, which is exactly what a TMA box {64 channels, BW, BH} with the 128-byte swizzle produces
// (row = pixel, 128 B = 64 channels): LBO = bytes between 64-channel groups (one TMA box = 8 KB), SBO = 1024
// (8 pixel rows of 128 B).
// A K block is a BW x BH = 64 pixel rectangle of ONE image (4-D tensor maps carry the batch index, so a
// block never straddles images); rows/cols beyond the buffer are zero-filled by TMA, the zero border of the
// Z buffer makes overhanging pixels contribute nothing.
// Work item = (K slice, tap, M tile, N tile); fp32 partial tiles are reduced (fixed order -> deterministic)
// and re-laid out to the MXNet parameter layout by wgrad_reduce_kernel.
// Warp roles as in conv_igemm.cuh: warp 0 loads, warpgroups 1 and 2 each own 64 of the 128 M rows.
// SPLIT3 (bf16x3 training step): both operands are hi / lo pairs, a stage holds the hi set and the lo set behind it, and each
// K step issues hi*hi + lo*hi + hi*lo into the same fp32 accumulator; the ring is shallower so that a stage of two operand
// sets still fits (WgradSmem / Conv1WgradSmem assert the totals).
#pragma once
#include "conv_igemm.cuh"

namespace dim {

struct WgradParams {
  CUtensorMap z_map;     // (C, cols, rows, B), box {64, BW, BH, 1}, SWIZZLE_128B
  CUtensorMap a_map[4];  // (C, cols, rows, B) views ((row parity, col parity) for stride 2), box {min(BN,64), BW, BH, 1}
  CUtensorMap z_lo_map, a_lo_map[4];  // the same views of the lo halves (SPLIT3 only)
  int KH, KW, stride;
  int BW, BH, rects_x, rects_y, Bn;
  int z_off_r, z_off_c, a_off_r, a_off_c;
  int m_tiles, n_tiles, kslices, kb_per_slice, kb_total;
  float *partial;  // [kslices][taps][m_tiles*128][n_tiles*BN]
};

// consumer side shared by both wgrad kernels: K blocks [kb0, kb1) of the ring, then the fp32 tile rows of this warpgroup
// (M rows 64*half .. +63) to dst (row stride ld floats).  a_off: byte offset of this warpgroup's M half in a stage.
// SPLIT3: the lo operands sit LO_BYTES behind the hi ones in every stage.
template <int BN, int STAGES, int STAGE_BYTES, int A_BYTES, bool SPLIT3 = false, int LO_BYTES = 0>
__device__ __forceinline__ void wgrad_consume(uint8_t *smem, uint64_t *full_bar, uint64_t *empty_bar, int kb0, int kb1, int half,
                                              uint64_t da_proto, uint32_t a_kstep, uint64_t db_proto, uint32_t b_kstep,
                                              float *dst, size_t ld) {
  const int t = threadIdx.x & 127;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  const uint32_t base = ptx::smem_u32(smem);
  int s = 0, prev = -1;
  uint32_t ph = 0;
  for (int kb = kb0; kb < kb1; ++kb) {
    ptx::mbar_wait(&full_bar[s], ph);
    const uint32_t st = base + s * STAGE_BYTES;
    const uint64_t da0 = da_proto + (uint64_t)(st >> 4), db0 = db_proto + (uint64_t)((st + A_BYTES) >> 4);
    wg::fence_acc(acc);
    wg::fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {  // 64 pixels = 4 x K 16
      const uint64_t da = da0 + (uint64_t)(k * a_kstep), db = db0 + (uint64_t)(k * b_kstep);
      wg::mma<BN, false, 1, 1>(acc, da, db, 1u);
      if (SPLIT3) {
        wg::mma<BN, false, 1, 1>(acc, da + (uint64_t)(LO_BYTES >> 4), db, 1u);
        wg::mma<BN, false, 1, 1>(acc, da, db + (uint64_t)(LO_BYTES >> 4), 1u);
      }
    }
    wg::commit();
    wg::wait<1>();
    wg::fence_acc(acc);
    if (prev >= 0 && t == 0) ptx::mbar_arrive(&empty_bar[prev]);
    prev = s;
    if (++s == STAGES) { s = 0; ph ^= 1u; }
  }
  wg::wait<0>();
  wg::fence_acc(acc);
  if (prev >= 0 && t == 0) ptx::mbar_arrive(&empty_bar[prev]);
  const int r = half * 64 + frag_row(t), q2 = (t & 3) * 2;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    *reinterpret_cast<float2 *>(dst + (size_t)r * ld + 8 * j + q2) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2 *>(dst + (size_t)(r + 8) * ld + 8 * j + q2) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
}

template <int BN, int STAGES, bool SPLIT3 = false>
struct WgradSmem {
  static constexpr int A_BYTES = 2 * 8192;                     // 128 channels x 64 pixels
  static constexpr int B_BYTES = BN >= 64 ? (BN / 64) * 8192 : 4096;
  static constexpr int SET_BYTES = A_BYTES + B_BYTES;          // one operand set (hi, or lo at + SET_BYTES)
  static constexpr int STAGE_BYTES = SET_BYTES * (SPLIT3 ? 2 : 1);
  static constexpr int TOTAL = STAGES * STAGE_BYTES + 1024 + 256;
  static_assert(TOTAL <= 227 * 1024, "conv_wgrad shared memory");
};

template <int BN, int STAGES, bool SPLIT3 = false>
__global__ void __launch_bounds__(384, 1) conv_wgrad_kernel(const __grid_constant__ WgradParams p) {
  using S = WgradSmem<BN, STAGES, SPLIT3>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + STAGES * S::STAGE_BYTES);
  uint64_t *empty_bar = full_bar + STAGES;

  const int wgi = threadIdx.x >> 7, warp = threadIdx.x >> 5;
  const int taps = p.KH * p.KW;
  int w = blockIdx.x;
  const int nt = w % p.n_tiles; w /= p.n_tiles;
  const int mt = w % p.m_tiles; w /= p.m_tiles;
  const int tap = w % taps;
  const int slice = w / taps;
  const int kb0 = slice * p.kb_per_slice;
  const int kb1 = min(p.kb_total, kb0 + p.kb_per_slice);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);
    }
    ptx::fence_barrier_init();
    ptx::prefetch_tmap(&p.z_map);
    ptx::prefetch_tmap(&p.a_map[0]);
  }
  __syncthreads();

  if (wgi == 0) {
    ptx::regs_producer();
    if (warp == 0) {  // whole warp; the elected lane issues (conv_igemm.cuh ptx::elect_one)
      const int kh = tap / p.KW, kw = tap - kh * p.KW;
      int view = 0, dr = kh, dc = kw;
      if (p.stride == 2) {
        view = ((kh & 1) << 1) | (kw & 1);
        dr = kh >> 1;
        dc = kw >> 1;
      }
      int s = 0;
      uint32_t ph = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        ptx::mbar_wait(&empty_bar[s], ph ^ 1u);
        const int rx = kb % p.rects_x;
        const int t = kb / p.rects_x;
        const int ry = t % p.rects_y, b = t / p.rects_y;
        const int oy0 = ry * p.BH, ox0 = rx * p.BW;
        uint8_t *st = smem + s * S::STAGE_BYTES;
        ptx::mbar_expect_tx(&full_bar[s], (uint32_t)S::STAGE_BYTES);
        ptx::tma_load_4d(st, &p.z_map, &full_bar[s], mt * 128, ox0 + p.z_off_c, oy0 + p.z_off_r, b);
        ptx::tma_load_4d(st + 8192, &p.z_map, &full_bar[s], mt * 128 + 64, ox0 + p.z_off_c, oy0 + p.z_off_r, b);
        uint8_t *bs = st + S::A_BYTES;
        if (BN >= 64) {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j)
            ptx::tma_load_4d(bs + j * 8192, &p.a_map[view], &full_bar[s], nt * BN + j * 64, ox0 + dc + p.a_off_c,
                             oy0 + dr + p.a_off_r, b);
        } else {
          ptx::tma_load_4d(bs, &p.a_map[view], &full_bar[s], nt * BN, ox0 + dc + p.a_off_c, oy0 + dr + p.a_off_r, b);
        }
        if (SPLIT3) {
          uint8_t *sl = st + S::SET_BYTES;
          ptx::tma_load_4d(sl, &p.z_lo_map, &full_bar[s], mt * 128, ox0 + p.z_off_c, oy0 + p.z_off_r, b);
          ptx::tma_load_4d(sl + 8192, &p.z_lo_map, &full_bar[s], mt * 128 + 64, ox0 + p.z_off_c, oy0 + p.z_off_r, b);
          if (BN >= 64) {
#pragma unroll
            for (int j = 0; j < BN / 64; ++j)
              ptx::tma_load_4d(sl + S::A_BYTES + j * 8192, &p.a_lo_map[view], &full_bar[s], nt * BN + j * 64, ox0 + dc + p.a_off_c,
                               oy0 + dr + p.a_off_r, b);
          } else {
            ptx::tma_load_4d(sl + S::A_BYTES, &p.a_lo_map[view], &full_bar[s], nt * BN, ox0 + dc + p.a_off_c, oy0 + dr + p.a_off_r, b);
          }
        }
        if (++s == STAGES) { s = 0; ph ^= 1u; }
      }
    }
  } else {
    ptx::regs_consumer();
    const int half = wgi - 1;
    const size_t Mp = (size_t)p.m_tiles * 128, Np = (size_t)p.n_tiles * BN;
    float *dst = p.partial + (((size_t)slice * taps + tap) * Mp + (size_t)mt * 128) * Np + (size_t)nt * BN;
    // A: this warpgroup's 64 channels are one 8 KB box; per K step of 16 pixels both operands advance 16 rows
    const uint64_t da = ptx::gmma_desc(half * 8192, 8192, 1024, ptx::kSW128);
    const uint64_t db = BN >= 64 ? ptx::gmma_desc(0, 8192, 1024, ptx::kSW128) : ptx::gmma_desc(0, 4096, 512, ptx::kSW64);
    wgrad_consume<BN, STAGES, S::STAGE_BYTES, S::A_BYTES, SPLIT3, S::SET_BYTES>(smem, full_bar, empty_bar, kb0, kb1, half, da, 128,
                                                                                db, BN >= 64 ? 128 : 64, dst, Np);
  }
}

// kinds of parameter tensors the reduction writes (MXNet layouts, SURVEY App. B-22)
enum { WG_CONV = 0, WG_CONV1_S2D = 1, WG_DECONV = 2, WG_CONV1_ROW = 3, WG_CONV1_RGBD = 4 };

// grad[dst] = sum_slices partial[slice][tap][m][n]; one thread per SOURCE element (tap, m, n) with n fastest, so the
// partial tiles are read coalesced; the (Cout,Cin,kh,kw) destination is written with a k*k-element stride.
//   WG_CONV      : m = co, n = ci            -> (Cout, Cin, k, k)
//   WG_CONV1_S2D : m = co, n = ph*16+pw*8+c  -> (64, 8, 7, 7), kh = 2dh+ph, kw = 2dw+pw      (taps = 16)
//   WG_CONV1_ROW : m = dw*32+ph*16+pw*8+c, n = co, tap = dh -> (64, D1, 7, 7)                 (conv1_wgrad_kernel, taps = 4;
//                  D1 = 8, or 6 for the image-only network: its zero mask lanes c >= 6 are dropped)
//   WG_DECONV    : m = ci, n = co            -> (Cin, Cout, k, k)
//   WG_CONV1_RGBD: m = co, n = ph*32+pw*16+c -> (64, 10, 7, 7), kh = 2dh+ph, kw = 2dw+pw  (RGB-D conv1, taps = 16; c >= 10 and
//                  taps outside the 7 x 7 filter are the layout's zero padding and are dropped)
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float *__restrict__ partial, int kslices, int taps,
                                                           int Mp, int Np, int kind, int D0, int D1, int k,
                                                           float *__restrict__ grad) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)taps * Mp * Np) return;
  const int n = (int)(idx % Np), m = (int)((idx / Np) % Mp), tap = (int)(idx / ((size_t)Np * Mp));
  int d0, d1, kh, kw;
  if (kind == WG_CONV1_S2D) {
    d0 = m; d1 = n & 7;
    kh = 2 * (tap >> 2) + ((n >> 4) & 1); kw = 2 * (tap & 3) + ((n >> 3) & 1);
    if (n >= 32) return;
  } else if (kind == WG_CONV1_RGBD) {
    d0 = m; d1 = n & 15;
    kh = 2 * (tap >> 2) + (n >> 5); kw = 2 * (tap & 3) + ((n >> 4) & 1);
  } else if (kind == WG_CONV1_ROW) {
    d0 = n; d1 = m & 7;
    kh = 2 * tap + ((m >> 4) & 1); kw = 2 * (m >> 5) + ((m >> 3) & 1);
  } else {
    d0 = m; d1 = n; kh = tap / k; kw = tap - kh * k;
  }
  if (d0 >= D0 || d1 >= D1 || kh >= k || kw >= k) return;
  float acc = 0.f;
  for (int s = 0; s < kslices; ++s) acc += partial[(size_t)s * taps * Mp * Np + idx];
  grad[(((size_t)d0 * D1 + d1) * k + kh) * k + kw] = acc;
}

// ---------------------------------------------------------------------------------------------
// conv1 weight gradient (64 x 8 x 7 x 7 from 240 x 320 output pixels): the generic kernel would run 16 taps of
// 128(64 used) x 32 tiles and fetch dZ 16 times.  Here one GEMM per filter ROW dh: M = (dw, 32 space-to-depth channels) =
// 128 rows assembled from FOUR column-shifted TMA boxes of the NHWC-32 input copy (64-byte rows, SWIZZLE_64B, MN-major
// groups LBO = 4 KB apart), N = 64 output channels of dZ (one SWIZZLE_128B box), K = 64 pixels: dZ is fetched 4x instead of
// 16x and no MMA row is padding.
template <int STAGES, bool SPLIT3 = false>
struct Conv1WgradSmem {
  static constexpr int A_BYTES = 4 * 4096, B_BYTES = 8192, SET_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGE_BYTES = SET_BYTES * (SPLIT3 ? 2 : 1);
  static constexpr int TOTAL = STAGES * STAGE_BYTES + 1024 + 256;
  static_assert(TOTAL <= 227 * 1024, "conv1_wgrad shared memory");
};

template <int STAGES, bool SPLIT3 = false>
__global__ void __launch_bounds__(384, 1) conv1_wgrad_kernel(const __grid_constant__ WgradParams p) {
  using S = Conv1WgradSmem<STAGES, SPLIT3>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + STAGES * S::STAGE_BYTES);
  uint64_t *empty_bar = full_bar + STAGES;
  const int wgi = threadIdx.x >> 7, warp = threadIdx.x >> 5;
  const int dh = blockIdx.x % 4, slice = blockIdx.x / 4;
  const int kb0 = slice * p.kb_per_slice;
  const int kb1 = min(p.kb_total, kb0 + p.kb_per_slice);
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 2);
    }
    ptx::fence_barrier_init();
    ptx::prefetch_tmap(&p.z_map);
    ptx::prefetch_tmap(&p.a_map[0]);
  }
  __syncthreads();
  if (wgi == 0) {
    ptx::regs_producer();
    if (warp == 0) {  // whole warp; the elected lane issues (conv_igemm.cuh ptx::elect_one)
      int s = 0;
      uint32_t ph = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        ptx::mbar_wait(&empty_bar[s], ph ^ 1u);
        const int rx = kb % p.rects_x;
        const int t = kb / p.rects_x;
        const int ry = t % p.rects_y, b = t / p.rects_y;
        const int oy0 = ry * p.BH, ox0 = rx * p.BW;
        uint8_t *st = smem + s * S::STAGE_BYTES;
        ptx::mbar_expect_tx(&full_bar[s], (uint32_t)S::STAGE_BYTES);
#pragma unroll
        for (int dw = 0; dw < 4; ++dw) ptx::tma_load_4d(st + dw * 4096, &p.a_map[0], &full_bar[s], 0, ox0 + dw, oy0 + dh, b);
        ptx::tma_load_4d(st + S::A_BYTES, &p.z_map, &full_bar[s], 0, ox0 + p.z_off_c, oy0 + p.z_off_r, b);
        if (SPLIT3) {
#pragma unroll
          for (int dw = 0; dw < 4; ++dw)
            ptx::tma_load_4d(st + S::SET_BYTES + dw * 4096, &p.a_lo_map[0], &full_bar[s], 0, ox0 + dw, oy0 + dh, b);
          ptx::tma_load_4d(st + S::SET_BYTES + S::A_BYTES, &p.z_lo_map, &full_bar[s], 0, ox0 + p.z_off_c, oy0 + p.z_off_r, b);
        }
        if (++s == STAGES) { s = 0; ph ^= 1u; }
      }
    }
  } else {
    ptx::regs_consumer();
    const int half = wgi - 1;
    float *dst = p.partial + ((size_t)slice * 4 + dh) * 128 * 64;
    // A: this warpgroup's 64 rows are two 32-channel boxes (dw = 2 half, 2 half + 1), 4 KB apart
    const uint64_t da = ptx::gmma_desc(half * 8192, 4096, 512, ptx::kSW64);
    const uint64_t db = ptx::gmma_desc(0, 8192, 1024, ptx::kSW128);
    wgrad_consume<64, STAGES, S::STAGE_BYTES, S::A_BYTES, SPLIT3, S::SET_BYTES>(smem, full_bar, empty_bar, kb0, kb1, half, da, 64, db,
                                                                                128, dst, 64);
  }
}

}  // namespace dim
