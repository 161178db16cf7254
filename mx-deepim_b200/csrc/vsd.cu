// vsd.cu -- the Visible Surface Discrepancy of Hodan et al. (dim_pose_error_vsd), compiled with -fmad=false.
//
// oracle/vsd.py states the contract in float64 numpy (the reference's depth_im_to_dist_im and visibility.py, pinned by
// tests/golden/ref_vsd.npz, and the paper's step cost); this file restates it operation by operation, so every count, and
// with it every error, equals the oracle's fed the same renders.
//
// Per call: the depth render at float32(P_gt), written full-frame into mask_rendered through the render's out_depth (its
// vertex box saved in vsd_box), then the box-only depth render at float32(P_est) into ren4.w (valid only inside vbox), then
//   vsd_pass_kernel   : grid (row chunks of VSD_ROWS rows, B).  A CTA whose rows miss the union of the two vertex boxes
//                       exits at once: outside both renders no pixel can be visible, so the restriction is exact.  Its
//                       threads walk the box columns of its rows, form the three distance images and the two visibility
//                       masks per pixel, and count |union|, |inter| and c_tau in registers.  The CTA sums them into its
//                       own slot [B][chunks][VSD_SLOT].
//   vsd_finish_kernel : one thread per instance: sums the slots of the box's chunks, forms e_tau and the status.
// Every sum is an integer count: the results do not depend on the order, the batch or the launch shape.
#include "launch.cuh"

namespace dim {

constexpr int VSD_THREADS = 256;

struct VsdParams {
  const float4 *ren4;        // [B,H,W], .w = estimate's depth; valid only inside vbox_est
  const float *depth_gt;     // [B,H,W] ground-truth depth render, full frame
  const int *vbox_est, *vbox_gt;  // [B,4] x0, x1, y0, y1
  const int *cls_flag;       // [B] 2 = bad class
  const float *depth;        // [F,H,W] observed, metres
  const int32_t *frame_idx;  // nullable: frame b
  const float *K_frames;     // nullable: K9 for every instance
  int32_t *partial;          // [B][chunks][VSD_SLOT]
  double *err;               // [B,n_tau]
  int32_t *status;           // [B], nullable
  double taus[VSD_MAX_TAU];
  float fx, fy, cx, cy, delta;
  int B, H, W, n_frames, chunks, n_tau;
};

struct Box { int i0, i1, j0, j1; };  // inclusive; empty when i1 < i0 or j1 < j0

__device__ __forceinline__ Box clipped_box(const int *v, int b, int H, int W) {
  Box r{max(v[4 * b + 2], 0), min(v[4 * b + 3], H - 1), max(v[4 * b], 0), min(v[4 * b + 1], W - 1)};
  if (r.i1 < r.i0 || r.j1 < r.j0) r = Box{1, 0, 1, 0};
  return r;
}

// the pixels the pass visits: the bounding box of the two clipped vertex boxes
__device__ __forceinline__ Box pass_range(const VsdParams &p, int b) {
  const Box e = clipped_box(p.vbox_est, b, p.H, p.W), g = clipped_box(p.vbox_gt, b, p.H, p.W);
  if (e.i1 < e.i0) return g;
  if (g.i1 < g.i0) return e;
  return Box{min(e.i0, g.i0), max(e.i1, g.i1), min(e.j0, g.j0), max(e.j1, g.j1)};
}

// depth_im_to_dist_im with a float32 K under numpy 2 (oracle/vsd.py dist_image): the reciprocals are float32 divisions
__device__ __forceinline__ double dist_of(float d, double di, double dj, double cx, double cy, double rfx, double rfy) {
  const double z = (double)d;
  const double X = ((dj - cx) * z) * rfx, Y = ((di - cy) * z) * rfy;
  return sqrt((X * X + Y * Y) + z * z);
}

__device__ __forceinline__ bool visible(double dist_test, double dist_model, float delta) {
  return dist_test > 0.0 && dist_model > 0.0 && (float)dist_model - (float)dist_test <= delta;
}

__global__ void __launch_bounds__(VSD_THREADS) vsd_pass_kernel(VsdParams p) {
  const int b = blockIdx.y, ch = blockIdx.x;
  const Box rg = pass_range(p, b);
  const int r0 = max(ch * VSD_ROWS, rg.i0), r1 = min(ch * VSD_ROWS + VSD_ROWS - 1, rg.i1);
  if (r1 < r0 || rg.j1 < rg.j0) return;  // the finish reads only the slots of chunks that meet the range
  __shared__ int red[VSD_THREADS / 32][VSD_SLOT];
  const int f = frame_of(p.frame_idx, p.n_frames, b);
  float fx = p.fx, fy = p.fy, cxf = p.cx, cyf = p.cy;
  if (p.K_frames) {
    const float *k = p.K_frames + 9 * f;
    fx = k[0]; cxf = k[2]; fy = k[4]; cyf = k[5];
  }
  const double rfx = (double)(1.0f / fx), rfy = (double)(1.0f / fy), cx = (double)cxf, cy = (double)cyf;
  const int ex0 = p.vbox_est[4 * b], ex1 = p.vbox_est[4 * b + 1], ey0 = p.vbox_est[4 * b + 2], ey1 = p.vbox_est[4 * b + 3];
  const size_t P = (size_t)p.H * p.W;
  const float4 *ren = p.ren4 + (size_t)b * P;
  const float *dgt = p.depth_gt + (size_t)b * P;
  const float *obs = p.depth + (size_t)f * P;

  int cnt[VSD_SLOT];
#pragma unroll
  for (int k = 0; k < VSD_SLOT; ++k) cnt[k] = 0;
  const int bw = rg.j1 - rg.j0 + 1, n = bw * (r1 - r0 + 1);
  for (int q = threadIdx.x; q < n; q += VSD_THREADS) {
    const int i = r0 + q / bw, j = rg.j0 + q % bw;
    const size_t o = (size_t)i * p.W + j;
    const float de = (i >= ey0 && i <= ey1 && j >= ex0 && j <= ex1) ? ren[o].w : 0.f;  // ren4 is stale outside the box
    const double di = (double)i, dj = (double)j;
    const double t = dist_of(obs[o], di, dj, cx, cy, rfx, rfy);
    const double g = dist_of(dgt[o], di, dj, cx, cy, rfx, rfy);
    const double e = dist_of(de, di, dj, cx, cy, rfx, rfy);
    const bool v_gt = visible(t, g, p.delta);
    const bool v_est = visible(t, e, p.delta) || (v_gt && e > 0.0);
    cnt[0] += (v_gt || v_est) ? 1 : 0;
    if (v_gt && v_est) {
      cnt[1] += 1;
      const double a = fabs(g - e);
#pragma unroll
      for (int k = 0; k < VSD_MAX_TAU; ++k)
        if (k < p.n_tau && a >= p.taus[k]) cnt[2 + k] += 1;
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < VSD_SLOT; ++k) {
    const int v = __reduce_add_sync(0xffffffffu, cnt[k]);
    if (lane == 0) red[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < VSD_SLOT) {
    int s = 0;
#pragma unroll
    for (int w = 0; w < VSD_THREADS / 32; ++w) s += red[w][threadIdx.x];
    p.partial[((size_t)b * p.chunks + ch) * VSD_SLOT + threadIdx.x] = s;
  }
}

__global__ void vsd_finish_kernel(VsdParams p) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= p.B) return;
  const Box rg = pass_range(p, b);
  int S[VSD_SLOT];
  for (int k = 0; k < VSD_SLOT; ++k) S[k] = 0;
  if (rg.i1 >= rg.i0 && rg.j1 >= rg.j0)
    for (int ch = rg.i0 / VSD_ROWS; ch <= rg.i1 / VSD_ROWS; ++ch) {
      const int32_t *slot = p.partial + ((size_t)b * p.chunks + ch) * VSD_SLOT;
      for (int k = 0; k < VSD_SLOT; ++k) S[k] += slot[k];
    }
  double *e = p.err + (size_t)b * p.n_tau;
  for (int k = 0; k < p.n_tau; ++k) e[k] = S[0] ? ((double)S[2 + k] + (double)(S[0] - S[1])) / (double)S[0] : 1.0;
  if (p.status)
    p.status[b] = (S[0] ? 0 : 1) | (p.cls_flag[b] ? 2 : 0) | (frame_bad(p.frame_idx, p.n_frames, b) ? 8 : 0);
}

int vsd_launch(dim_ctx *ctx, const VsdCall &c, cudaStream_t st) {
  static const float K_zero[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  const float *K9 = c.K9 ? c.K9 : K_zero;
  // stage profiling (dim_profile_enable): one record of 5 events per call, stage 0 = the two renders, stage 1 = VSD pass
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
  {
    DimNvtxRange r("dim_pose_error_vsd render");
    if (int rc = f64_to_f32_launch(c.pose_gt, ctx->pose_cur_f32, c.B * 12, st)) return rc;
    if (int rc = render_launch(ctx, c.cls_idx, ctx->pose_cur_f32, c.B, K9, c.zn, c.zf, nullptr, 1, nullptr, ctx->mask_rendered,
                               nullptr, nullptr, nullptr, nullptr, st, nullptr, true, false, c.K_frames, c.frame_idx, c.F))
      return rc;
    DIM_CHECK(cudaMemcpyAsync(ctx->vsd_box, ctx->vbox, sizeof(int) * 4 * c.B, cudaMemcpyDeviceToDevice, st));
    if (int rc = f64_to_f32_launch(c.pose_est, ctx->pose_cur_f32, c.B * 12, st)) return rc;
    if (int rc = render_launch(ctx, c.cls_idx, ctx->pose_cur_f32, c.B, K9, c.zn, c.zf, nullptr, 1, nullptr, nullptr, nullptr,
                               nullptr, nullptr, ctx->ren4, st, nullptr, true, false, c.K_frames, c.frame_idx, c.F))
      return rc;
  }
  if (ev) DIM_CHECK(cudaEventRecord(ev[1], st));
  VsdParams p;
  p.ren4 = ctx->ren4; p.depth_gt = ctx->mask_rendered; p.vbox_est = ctx->vbox; p.vbox_gt = ctx->vsd_box;
  p.cls_flag = ctx->cls_flag; p.depth = c.depth; p.frame_idx = c.frame_idx; p.K_frames = c.K_frames;
  p.partial = ctx->vsd_partial; p.err = c.err; p.status = c.status;
  for (int k = 0; k < VSD_MAX_TAU; ++k) p.taus[k] = k < c.n_tau ? c.taus[k] : 0.0;
  p.fx = K9[0]; p.fy = K9[4]; p.cx = K9[2]; p.cy = K9[5]; p.delta = c.delta;
  p.B = c.B; p.H = ctx->H; p.W = ctx->W; p.n_frames = c.F; p.chunks = cdiv(ctx->H, VSD_ROWS); p.n_tau = c.n_tau;
  {
    DimNvtxRange r("dim_pose_error_vsd pass");
    vsd_pass_kernel<<<dim3(p.chunks, c.B), VSD_THREADS, 0, st>>>(p);
    DIM_LAUNCH_CHECK();
    vsd_finish_kernel<<<cdiv(c.B, 64), 64, 0, st>>>(p);
    DIM_LAUNCH_CHECK();
  }
  if (ev)
    for (int k = 2; k < 5; ++k) DIM_CHECK(cudaEventRecord(ev[k], st));
  return 0;
}

}  // namespace dim
