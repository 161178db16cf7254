// icp.cu -- projective point-to-plane ICP against the observed depth (dim_icp), compiled with -fmad=false.
//
// The reference has no ICP; oracle/icp.py defines it and this file restates it operation by operation in float64, so that
// an oracle association fed the device's pose reproduces the device's inlier count exactly.
//
// Per call: one box-only depth render at float32(P0) into ren4.w (the RGB-D loop's raster_resolve_kernel<false, true>),
// then per iteration
//   icp_assoc_kernel : grid (row chunks of ICP_ROWS rows, B).  A CTA whose rows miss the interior of the instance's vertex
//                      box exits at once; its threads walk the box columns of its rows, build the model point and normal
//                      from the rendered depth, associate it projectively with the observed depth, and accumulate the
//                      inlier's normal equations in registers.  The CTA reduces its ICP_SLOT doubles in a fixed shuffle /
//                      shared-memory order into its own slot [B][chunks][ICP_SLOT]: no atomics, so every run gives the
//                      same bits.
//   icp_solve_kernel : one thread per instance: sums the slots of the box's chunks in index order, 6x6 Cholesky, the
//                      Rodrigues update, and writes the iteration's pose, inlier count, rms and status.
#include "launch.cuh"

namespace dim {

// slot layout: the 21 upper entries of A (row-major), g[6], inlier count, sum r^2, model pixel count
constexpr int ICP_A = 0, ICP_G = 21, ICP_C = 27, ICP_E = 28, ICP_M = 29;
constexpr int ICP_THREADS = 256;

struct IcpParams {
  const float4 *ren4;         // [B,H,W], .w = rendered depth; valid only inside vbox
  const int *vbox;            // [B,4] x0, x1, y0, y1 (conservative box of the projected vertices)
  const int *cls_flag;        // [B] 2 = bad class
  const float *depth;         // [F,H,W] observed, metres
  const int32_t *frame_idx;   // nullable: frame b
  const float *K_frames;      // nullable: K9 for every instance
  const double *pose0;        // [B,3,4] the call's input pose
  double *partial;            // [B][chunks][ICP_SLOT]
  double *poses;              // [n_iter,B,3,4]
  int32_t *inliers, *status;  // [n_iter,B]
  float *rms;                 // [n_iter,B]
  float fx, fy, cx, cy, max_dist;
  int B, H, W, n_frames, chunks, min_points;
};

// the model pixels an instance may have: the interior of its vertex box within the frame's interior.  Pixels outside the
// box render empty by construction (and ren4 is stale there), so a pixel on the box's edge never has four covered
// neighbours; skipping it changes nothing and keeps every read inside the box.
struct Range { int i0, i1, j0, j1; };
__device__ __forceinline__ Range model_range(const int *vbox, int b, int H, int W) {
  const int x0 = vbox[4 * b], x1 = vbox[4 * b + 1], y0 = vbox[4 * b + 2], y1 = vbox[4 * b + 3];
  Range r{1, 0, 1, 0};
  if (x1 < x0 || y1 < y0) return r;
  r.i0 = max(y0 + 1, 1); r.i1 = min(y1 - 1, H - 2);
  r.j0 = max(x0 + 1, 1); r.j1 = min(x1 - 1, W - 2);
  return r;
}

__device__ __forceinline__ void intrinsics(const IcpParams &p, int b, double &fx, double &fy, double &cx, double &cy) {
  if (p.K_frames) {
    const float *k = p.K_frames + 9 * frame_of(p.frame_idx, p.n_frames, b);
    fx = (double)k[0]; cx = (double)k[2]; fy = (double)k[4]; cy = (double)k[5];
  } else {
    fx = (double)p.fx; fy = (double)p.fy; cx = (double)p.cx; cy = (double)p.cy;
  }
}

__global__ void __launch_bounds__(ICP_THREADS) icp_assoc_kernel(IcpParams p, const double *pose_k) {
  const int b = blockIdx.y, ch = blockIdx.x;
  const Range rg = model_range(p.vbox, b, p.H, p.W);
  const int r0 = max(ch * ICP_ROWS, rg.i0), r1 = min(ch * ICP_ROWS + ICP_ROWS - 1, rg.i1);
  if (r1 < r0 || rg.j1 < rg.j0) return;  // the solve reads only the slots of chunks that meet the range
  __shared__ double sRt[12];
  __shared__ double red[ICP_THREADS / 32][ICP_SLOT];
  if (threadIdx.x == 0) {  // R_D = R_k R0^T, t_D = t_k - R_D t0 (the oracle's increment, same order)
    const double *P0 = p.pose0 + 12 * b, *Pk = pose_k + 12 * b;
    for (int a = 0; a < 3; ++a)
      for (int c = 0; c < 3; ++c) sRt[4 * a + c] = (Pk[4 * a] * P0[4 * c] + Pk[4 * a + 1] * P0[4 * c + 1]) + Pk[4 * a + 2] * P0[4 * c + 2];
    for (int a = 0; a < 3; ++a)
      sRt[4 * a + 3] = Pk[4 * a + 3] - ((sRt[4 * a] * P0[3] + sRt[4 * a + 1] * P0[7]) + sRt[4 * a + 2] * P0[11]);
  }
  __syncthreads();
  double R[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) R[k] = sRt[k];
  double fx, fy, cx, cy;
  intrinsics(p, b, fx, fy, cx, cy);
  const double md = (double)p.max_dist;
  const size_t P = (size_t)p.H * p.W;
  const float4 *ren = p.ren4 + (size_t)b * P;
  const float *obs = p.depth + (size_t)frame_of(p.frame_idx, p.n_frames, b) * P;

  double acc[ICP_SLOT];
#pragma unroll
  for (int k = 0; k < ICP_SLOT; ++k) acc[k] = 0.0;
  const int bw = rg.j1 - rg.j0 + 1, n = bw * (r1 - r0 + 1);
  for (int q = threadIdx.x; q < n; q += ICP_THREADS) {
    const int i = r0 + q / bw, j = rg.j0 + q % bw;
    const size_t o = (size_t)i * p.W + j;
    const double d = (double)ren[o].w;
    if (!(d > 0.0)) continue;
    const double dr = (double)ren[o + 1].w, dl = (double)ren[o - 1].w, dd = (double)ren[o + p.W].w,
                 du = (double)ren[o - p.W].w;
    if (!(dr > 0.0 && dl > 0.0 && dd > 0.0 && du > 0.0)) continue;
    if (fabs(dr - d) > md || fabs(dl - d) > md || fabs(dd - d) > md || fabs(du - d) > md) continue;
    const double di = (double)i, dj = (double)j;
    const double X0 = ((dj - cx) * d) / fx, X1 = ((di - cy) * d) / fy, X2 = d;
    const double a0 = ((dj + 1.0 - cx) * dr) / fx - ((dj - 1.0 - cx) * dl) / fx;
    const double a1 = ((di - cy) * dr) / fy - ((di - cy) * dl) / fy;
    const double a2 = dr - dl;
    const double b0 = ((dj - cx) * dd) / fx - ((dj - cx) * du) / fx;
    const double b1 = ((di + 1.0 - cy) * dd) / fy - ((di - 1.0 - cy) * du) / fy;
    const double b2 = dd - du;
    const double c0 = a1 * b2 - a2 * b1, c1 = a2 * b0 - a0 * b2, c2 = a0 * b1 - a1 * b0;
    const double ln = sqrt((c0 * c0 + c1 * c1) + c2 * c2);
    if (ln == 0.0) continue;
    double n0 = c0 / ln, n1 = c1 / ln, n2 = c2 / ln;
    if (((n0 * X0 + n1 * X1) + n2 * X2) > 0.0) { n0 = -n0; n1 = -n1; n2 = -n2; }
    acc[ICP_M] += 1.0;
    const double Y0 = ((R[0] * X0 + R[1] * X1) + R[2] * X2) + R[3];
    const double Y1 = ((R[4] * X0 + R[5] * X1) + R[6] * X2) + R[7];
    const double Y2 = ((R[8] * X0 + R[9] * X1) + R[10] * X2) + R[11];
    const double m0 = (R[0] * n0 + R[1] * n1) + R[2] * n2;
    const double m1 = (R[4] * n0 + R[5] * n1) + R[6] * n2;
    const double m2 = (R[8] * n0 + R[9] * n1) + R[10] * n2;
    if (!(Y2 > 0.0)) continue;
    const double qj = rint((fx * Y0) / Y2 + cx), qi = rint((fy * Y1) / Y2 + cy);
    if (!(qj >= 0.0 && qj <= (double)(p.W - 1) && qi >= 0.0 && qi <= (double)(p.H - 1))) continue;
    const float dof = obs[(size_t)qi * p.W + (size_t)qj];
    if (!(isfinite(dof) && dof > 0.f)) continue;
    const double d_o = (double)dof;
    if (!(fabs(Y2 - d_o) < md)) continue;
    const double Z0 = ((qj - cx) * d_o) / fx, Z1 = ((qi - cy) * d_o) / fy;
    const double r = (m0 * (Y0 - Z0) + m1 * (Y1 - Z1)) + m2 * (Y2 - d_o);
    const double J[6] = {Y1 * m2 - Y2 * m1, Y2 * m0 - Y0 * m2, Y0 * m1 - Y1 * m0, m0, m1, m2};
    int k = ICP_A;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
      for (int c = a; c < 6; ++c) acc[k++] += J[a] * J[c];
#pragma unroll
    for (int a = 0; a < 6; ++a) acc[ICP_G + a] += J[a] * r;
    acc[ICP_C] += 1.0;
    acc[ICP_E] += r * r;
  }
  // fixed-order reduction: butterfly within the warp, then the warps in index order
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < ICP_SLOT; ++k) {
    double v = acc[k];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (lane == 0) red[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < ICP_SLOT) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < ICP_THREADS / 32; ++w) s += red[w][threadIdx.x];
    p.partial[((size_t)b * p.chunks + ch) * ICP_SLOT + threadIdx.x] = s;
  }
}

// exp([w]x); I + [w]x below |w| = 1e-12 (oracle/icp.py rodrigues)
__device__ void rodrigues(const double w[3], double dR[9]) {
  const double th = sqrt((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]);
  if (th < 1e-12) {
    dR[0] = 1.0; dR[1] = -w[2]; dR[2] = w[1];
    dR[3] = w[2]; dR[4] = 1.0; dR[5] = -w[0];
    dR[6] = -w[1]; dR[7] = w[0]; dR[8] = 1.0;
    return;
  }
  const double k0 = w[0] / th, k1 = w[1] / th, k2 = w[2] / th;
  const double s = sin(th), c = cos(th), C = 1.0 - c;
  dR[0] = c + C * k0 * k0; dR[1] = C * k0 * k1 - s * k2; dR[2] = C * k0 * k2 + s * k1;
  dR[3] = C * k1 * k0 + s * k2; dR[4] = c + C * k1 * k1; dR[5] = C * k1 * k2 - s * k0;
  dR[6] = C * k2 * k0 - s * k1; dR[7] = C * k2 * k1 + s * k0; dR[8] = c + C * k2 * k2;
}

// Cholesky of the 6x6 normal equations and x = -A^-1 g; false when a pivot is <= 1e-12 max(diag A)
__device__ bool solve6(const double *S, double x[6]) {
  double A[6][6], L[6][6];
  int k = ICP_A;
  for (int a = 0; a < 6; ++a)
    for (int c = a; c < 6; ++c) A[a][c] = S[k++];
  double mx = A[0][0];
  for (int a = 1; a < 6; ++a) mx = fmax(mx, A[a][a]);
  const double tol = 1e-12 * mx;
  for (int j = 0; j < 6; ++j) {
    double s = A[j][j];
    for (int q = 0; q < j; ++q) s -= L[j][q] * L[j][q];
    if (s <= tol) return false;
    L[j][j] = sqrt(s);
    for (int i = j + 1; i < 6; ++i) {
      double t = A[j][i];
      for (int q = 0; q < j; ++q) t -= L[i][q] * L[j][q];
      L[i][j] = t / L[j][j];
    }
  }
  double y[6];
  for (int i = 0; i < 6; ++i) {
    double s = -S[ICP_G + i];
    for (int q = 0; q < i; ++q) s -= L[i][q] * y[q];
    y[i] = s / L[i][i];
  }
  for (int i = 5; i >= 0; --i) {
    double s = y[i];
    for (int q = i + 1; q < 6; ++q) s -= L[q][i] * x[q];
    x[i] = s / L[i][i];
  }
  return true;
}

__global__ void icp_solve_kernel(IcpParams p, const double *pose_k, int it) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= p.B) return;
  const Range rg = model_range(p.vbox, b, p.H, p.W);
  double S[ICP_SLOT];
  for (int k = 0; k < ICP_SLOT; ++k) S[k] = 0.0;
  if (rg.i1 >= rg.i0 && rg.j1 >= rg.j0)
    for (int ch = rg.i0 / ICP_ROWS; ch <= rg.i1 / ICP_ROWS; ++ch) {
      const double *slot = p.partial + ((size_t)b * p.chunks + ch) * ICP_SLOT;
      for (int k = 0; k < ICP_SLOT; ++k) S[k] += slot[k];
    }
  int st = (p.cls_flag[b] ? 2 : 0) | (frame_bad(p.frame_idx, p.n_frames, b) ? 8 : 0);
  const double *Pk = pose_k + 12 * b;
  double *out = p.poses + ((size_t)it * p.B + b) * 12;
  double x[6];
  bool upd = false;
  if (S[ICP_M] == 0.0) st |= 1;
  else if (S[ICP_C] < (double)p.min_points || !solve6(S, x)) st |= 16;
  else upd = true;
  if (upd) {
    double dR[9];
    rodrigues(x, dR);
    for (int a = 0; a < 3; ++a) {
      for (int c = 0; c < 3; ++c) out[4 * a + c] = (dR[3 * a] * Pk[c] + dR[3 * a + 1] * Pk[4 + c]) + dR[3 * a + 2] * Pk[8 + c];
      out[4 * a + 3] = ((dR[3 * a] * Pk[3] + dR[3 * a + 1] * Pk[7]) + dR[3 * a + 2] * Pk[11]) + x[3 + a];
    }
  } else {
    for (int k = 0; k < 12; ++k) out[k] = Pk[k];
  }
  const size_t o = (size_t)it * p.B + b;
  p.inliers[o] = (int32_t)S[ICP_C];
  p.rms[o] = S[ICP_C] > 0.0 ? (float)sqrt(S[ICP_E] / S[ICP_C]) : 0.f;
  p.status[o] = st;
}

// u16 depth file values -> metres, float32(u16) / float32(depth_factor) (lib/utils/image.py:203,218)
__global__ void depth_u16_kernel(const uint16_t *in, size_t n, float factor, float *out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (float)in[i] / factor;
}

int depth_u16_launch(const uint16_t *in, size_t n, float factor, float *out, cudaStream_t st) {
  depth_u16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, n, factor, out);
  DIM_LAUNCH_CHECK();
  return 0;
}

int icp_launch(dim_ctx *ctx, const IcpCall &c, cudaStream_t st) {
  static const float K_zero[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  const float *K9 = c.K9 ? c.K9 : K_zero;
  // stage profiling (dim_profile_enable): one record of 5 events per call, stage 0 = render, stage 1 = association + solve
  cudaEvent_t *ev = nullptr;
  if (ctx->prof) {
    while (ctx->prof_events.size() < ctx->prof_used + 5) {
      cudaEvent_t e;
      DIM_CHECK(cudaEventCreate(&e));
      ctx->prof_events.push_back(e);
    }
    ev = &ctx->prof_events[ctx->prof_used];
    ctx->prof_used += 5;
    DIM_CHECK(cudaEventRecord(ev[0], st));
  }
  if (int rc = f64_to_f32_launch(c.pose_in, ctx->pose_cur_f32, c.B * 12, st)) return rc;
  {
    DimNvtxRange r("dim_icp render");
    if (int rc = render_launch(ctx, c.cls_idx, ctx->pose_cur_f32, c.B, K9, c.zn, c.zf, nullptr, 1, nullptr, nullptr, nullptr,
                               nullptr, nullptr, ctx->ren4, st, nullptr, true, false, c.K_frames, c.frame_idx, c.F))
      return rc;
  }
  if (ev) DIM_CHECK(cudaEventRecord(ev[1], st));
  IcpParams p;
  p.ren4 = ctx->ren4; p.vbox = ctx->vbox; p.cls_flag = ctx->cls_flag; p.depth = c.depth;
  p.frame_idx = c.frame_idx; p.K_frames = c.K_frames; p.pose0 = c.pose_in; p.partial = ctx->icp_partial;
  p.poses = c.poses_out; p.inliers = c.inliers; p.status = c.status; p.rms = c.rms;
  p.fx = K9[0]; p.fy = K9[4]; p.cx = K9[2]; p.cy = K9[5]; p.max_dist = c.max_dist;
  p.B = c.B; p.H = ctx->H; p.W = ctx->W; p.n_frames = c.F; p.chunks = cdiv(ctx->H, ICP_ROWS); p.min_points = c.min_points;
  DimNvtxRange r("dim_icp iterations");
  for (int it = 0; it < c.n_iter; ++it) {
    const double *pk = it == 0 ? c.pose_in : c.poses_out + (size_t)(it - 1) * c.B * 12;
    icp_assoc_kernel<<<dim3(p.chunks, c.B), ICP_THREADS, 0, st>>>(p, pk);
    DIM_LAUNCH_CHECK();
    icp_solve_kernel<<<cdiv(c.B, 64), 64, 0, st>>>(p, pk, it);
    DIM_LAUNCH_CHECK();
  }
  if (ev)
    for (int k = 2; k < 5; ++k) DIM_CHECK(cudaEventRecord(ev[k], st));
  return 0;
}

}  // namespace dim
