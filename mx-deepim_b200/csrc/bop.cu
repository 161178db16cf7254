// bop.cu -- the BOP 2019 symmetry-aware pose errors MSSD and MSPD (dim_pose_error_sym), compiled with -fmad=false.
//
// oracle/bop.py states the contract in float64 numpy; this file restates it operation by operation.  Per instance m and
// symmetry s the GT-symmetric pose is R_gs = R_gt R_s, t_gs = R_gt t_s + t_gt; model points are transformed as
// pose_error_kernel (ADD) does and projected as pose_error2d_kernel (Proj. 2D) does, and
//   MSSD = min_s max_p |T_est p - T_gs p|,   MSPD = min_s max_p |proj(K_m, T_est p) - proj(K_m, T_gs p)|
// with MSPD(s) = +inf when a point has Z <= 0 under either pose.  Every value formed is the oracle's, and max / min / sqrt
// are exact in any order, so the results equal the oracle's bit for bit for any batch, chunking or launch shape.
//
//   sym_pass_kernel   : grid (symmetry tiles of SYM_TILE, point chunks, M), SYM_THREADS threads.  The CTA stages a tile of
//                       SYM_THREADS points -- the model point, its estimate transform and the estimate's projection, formed
//                       once and reused by all SYM_TILE symmetries -- in shared memory.  Lane l of every warp owns symmetry
//                       tile * SYM_TILE + l; warp w takes the tile's points w, w + 8, ...  Each thread keeps the running
//                       maxima of the squared 3-D and 2-D distances; the warps' maxima meet in shared memory and go to the
//                       context's scratch slot [m][s][chunk].
//   sym_finish_kernel : one CTA per instance: the max over chunks per symmetry, then the min over symmetries (lowest index
//                       on ties) and the square roots.
#include <math_constants.h>

#include <algorithm>

#include "launch.cuh"

namespace dim {

constexpr int SYM_THREADS = 256, SYM_TILE = 32, SYM_WARPS = SYM_THREADS / 32;

struct SymParams {
  const double *pose_est, *pose_gt;  // [M,12]
  const double *pts;                 // [N,3]
  const double *syms;                // [S,12]
  const double *K;                   // [M,9]
  double *partial;                   // [M][S][chunks][2] squared maxima (3-D, 2-D)
  double *err2;                      // [M,2]
  int32_t *sym_idx2;                 // [M,2], nullable
  int N, S, chunks, chunk_len;
};

__global__ void __launch_bounds__(SYM_THREADS) sym_pass_kernel(SymParams p) {
  const int m = blockIdx.z, ch = blockIdx.y, s0 = blockIdx.x * SYM_TILE;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __shared__ double Pe[12], Kk[9];
  __shared__ double pt[SYM_THREADS][8];  // x, y, z, est x, y, z, est u, est v
  __shared__ double red[SYM_WARPS][SYM_TILE][2];
  if (threadIdx.x < 12) Pe[threadIdx.x] = p.pose_est[12 * m + threadIdx.x];
  if (threadIdx.x < 9) Kk[threadIdx.x] = p.K[9 * m + threadIdx.x];
  // this lane's GT-symmetric pose: R_gs = R_gt R_s, t_gs = R_gt t_s + t_gt, elementwise in the oracle's order
  const int s = s0 + lane;
  double G[12];
  {
    const double *g = p.pose_gt + 12 * m, *q = p.syms + 12 * (s < p.S ? s : 0);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
      for (int j = 0; j < 3; ++j) G[4 * i + j] = (g[4 * i] * q[j] + g[4 * i + 1] * q[4 + j]) + g[4 * i + 2] * q[8 + j];
      G[4 * i + 3] = ((g[4 * i] * q[3] + g[4 * i + 1] * q[7]) + g[4 * i + 2] * q[11]) + g[4 * i + 3];
    }
  }
  __syncthreads();
  double d2max = 0.0, p2max = 0.0;
  const int n0 = ch * p.chunk_len, n1 = min(p.N, n0 + p.chunk_len);
  for (int t0 = n0; t0 < n1; t0 += SYM_THREADS) {
    const int cnt = min(SYM_THREADS, n1 - t0);
    if ((int)threadIdx.x < cnt) {
      const int n = t0 + threadIdx.x;
      const double x = p.pts[3 * n], y = p.pts[3 * n + 1], z = p.pts[3 * n + 2];
      double e[3], c[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) e[r] = ((Pe[4 * r] * x + Pe[4 * r + 1] * y) + Pe[4 * r + 2] * z) + Pe[4 * r + 3];
#pragma unroll
      for (int r = 0; r < 3; ++r) c[r] = (Kk[3 * r] * e[0] + Kk[3 * r + 1] * e[1]) + Kk[3 * r + 2] * e[2];
      double *o = pt[threadIdx.x];
      o[0] = x; o[1] = y; o[2] = z; o[3] = e[0]; o[4] = e[1]; o[5] = e[2];
      o[6] = c[0] / c[2]; o[7] = c[1] / c[2];
    }
    __syncthreads();
    for (int k = warp; k < cnt; k += SYM_WARPS) {
      const double *o = pt[k];
      const double x = o[0], y = o[1], z = o[2];
      double g[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) g[r] = ((G[4 * r] * x + G[4 * r + 1] * y) + G[4 * r + 2] * z) + G[4 * r + 3];
      const double dx = o[3] - g[0], dy = o[4] - g[1], dz = o[5] - g[2];
      const double d2 = (dx * dx + dy * dy) + dz * dz;
      d2max = d2 > d2max ? d2 : d2max;
      if (o[5] <= 0.0 || g[2] <= 0.0) {
        p2max = CUDART_INF;
      } else {
        double c[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) c[r] = (Kk[3 * r] * g[0] + Kk[3 * r + 1] * g[1]) + Kk[3 * r + 2] * g[2];
        const double du = o[6] - c[0] / c[2], dv = o[7] - c[1] / c[2];
        const double p2 = du * du + dv * dv;
        p2max = p2 > p2max ? p2 : p2max;
      }
    }
    __syncthreads();
  }
  red[warp][lane][0] = d2max;
  red[warp][lane][1] = p2max;
  __syncthreads();
  if (threadIdx.x < 2 * SYM_TILE) {
    const int l = threadIdx.x >> 1, k = threadIdx.x & 1;
    double v = red[0][l][k];
#pragma unroll
    for (int w = 1; w < SYM_WARPS; ++w) v = red[w][l][k] > v ? red[w][l][k] : v;
    if (s0 + l < p.S) p.partial[(((size_t)m * p.S + s0 + l) * p.chunks + ch) * 2 + k] = v;
  }
}

__global__ void __launch_bounds__(SYM_THREADS) sym_finish_kernel(SymParams p) {
  const int m = blockIdx.x;
  __shared__ double bv[2][SYM_THREADS];
  __shared__ int bi[2][SYM_THREADS];
  double best[2] = {CUDART_INF, CUDART_INF};
  int idx[2] = {0x7fffffff, 0x7fffffff};
  for (int s = threadIdx.x; s < p.S; s += SYM_THREADS) {
    const double *q = p.partial + ((size_t)m * p.S + s) * p.chunks * 2;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      double v = q[k];
      for (int c = 1; c < p.chunks; ++c) v = q[2 * c + k] > v ? q[2 * c + k] : v;
      if (v < best[k] || idx[k] == 0x7fffffff) { best[k] = v; idx[k] = s; }  // s ascends: the first minimum is kept
    }
  }
#pragma unroll
  for (int k = 0; k < 2; ++k) { bv[k][threadIdx.x] = best[k]; bi[k][threadIdx.x] = idx[k]; }
  __syncthreads();
  for (int h = SYM_THREADS / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h)
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const double v = bv[k][threadIdx.x + h];
        const int i = bi[k][threadIdx.x + h];
        if (v < bv[k][threadIdx.x] || (v == bv[k][threadIdx.x] && i < bi[k][threadIdx.x])) {
          bv[k][threadIdx.x] = v;
          bi[k][threadIdx.x] = i;
        }
      }
    __syncthreads();
  }
  if (threadIdx.x < 2) {
    p.err2[2 * m + threadIdx.x] = sqrt(bv[threadIdx.x][0]);
    if (p.sym_idx2) p.sym_idx2[2 * m + threadIdx.x] = bi[threadIdx.x][0];
  }
}

int sym_launch(dim_ctx *ctx, const SymCall &c, cudaStream_t st) {
  SymParams p;
  p.pose_est = c.pose_est; p.pose_gt = c.pose_gt; p.pts = c.pts; p.syms = c.syms; p.K = c.K;
  p.partial = ctx->sym_partial; p.err2 = c.err2; p.sym_idx2 = c.sym_idx2;
  p.N = c.N; p.S = c.S;
  // enough CTAs for SYM_WAVES waves of the schedule's SMs, within the scratch's SYM_SLOTS slots per instance and with at
  // least one point tile per chunk
  const int tiles = cdiv(c.S, SYM_TILE);
  const int want = cdiv(SYM_WAVES * ctx->num_sms, c.M * tiles);
  p.chunks = std::max(1, std::min({want, SYM_SLOTS / c.S, cdiv(c.N, SYM_THREADS)}));
  p.chunk_len = cdiv(cdiv(c.N, p.chunks), SYM_THREADS) * SYM_THREADS;
  p.chunks = cdiv(c.N, p.chunk_len);
  DimNvtxRange r("dim_pose_error_sym");
  sym_pass_kernel<<<dim3(tiles, p.chunks, c.M), SYM_THREADS, 0, st>>>(p);
  DIM_LAUNCH_CHECK();
  sym_finish_kernel<<<c.M, SYM_THREADS, 0, st>>>(p);
  DIM_LAUNCH_CHECK();
  return 0;
}

}  // namespace dim
