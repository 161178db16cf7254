// vsd.cu -- the Visible Surface Discrepancy of Hodan et al. (dim_pose_error_vsd, dim_pose_error_vsd_ex), compiled with
// -fmad=false.
//
// oracle/vsd.py states the contract in float64 numpy (the reference's depth_im_to_dist_im and visibility.py, pinned by
// tests/golden/ref_vsd.npz, and the paper's step cost); this file restates it operation by operation, so every count, and
// with it every error, equals the oracle's fed the same renders.  The BOP 2019 variant (oracle/bop.py's vsd()) changes only
// the visibility rule (sensor holes are visible) and, with diameters, divides the distance difference by the instance's
// diameter before the tau test; both are template parameters of the pass, so the SIXD 2017 instantiation is the original
// kernel.
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
  FrameCams cams;
  int32_t *partial;          // [B][chunks][VSD_SLOT]
  double *err;               // [B,n_tau]
  int32_t *status;           // [B], nullable
  double taus[VSD_MAX_TAU];
  float delta;
  int B, H, W, chunks, n_tau;
  const double *diam;        // [B] with relative taus (vsd_pass_kernel<VIS, true>)
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

// VIS = 0: the SIXD 2017 rule (visibility.py); VIS = 1: BOP 2019's, where a sensor hole (dist_test == 0) counts as visible
template <int VIS>
__device__ __forceinline__ bool visible(double dist_test, double dist_model, float delta) {
  if (VIS == 0) return dist_test > 0.0 && dist_model > 0.0 && (float)dist_model - (float)dist_test <= delta;
  return dist_model > 0.0 && ((float)dist_model - (float)dist_test <= delta || dist_test == 0.0);
}

// DIAM: the taus are fractions of the instance's diameter p.diam[b] (BOP 2019), else metres
template <int VIS, bool DIAM>
__global__ void __launch_bounds__(VSD_THREADS) vsd_pass_kernel(VsdParams p) {
  const int b = blockIdx.y, ch = blockIdx.x;
  const Box rg = pass_range(p, b);
  const int r0 = max(ch * VSD_ROWS, rg.i0), r1 = min(ch * VSD_ROWS + VSD_ROWS - 1, rg.i1);
  if (r1 < r0 || rg.j1 < rg.j0) return;  // the finish reads only the slots of chunks that meet the range
  __shared__ int red[VSD_THREADS / 32][VSD_SLOT];
  const size_t P = (size_t)p.H * p.W;
  const float *obs = p.depth + (size_t)p.cams.frame(b) * P;
  const float4 k = p.cams.pinhole(b);
  const double rfx = (double)(1.0f / k.x), rfy = (double)(1.0f / k.y), cx = (double)k.z, cy = (double)k.w;
  const int ex0 = p.vbox_est[4 * b], ex1 = p.vbox_est[4 * b + 1], ey0 = p.vbox_est[4 * b + 2], ey1 = p.vbox_est[4 * b + 3];
  const float4 *ren = p.ren4 + (size_t)b * P;
  const float *dgt = p.depth_gt + (size_t)b * P;
  const double diam = DIAM ? p.diam[b] : 0.0;

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
    const bool v_gt = visible<VIS>(t, g, p.delta);
    const bool v_est = visible<VIS>(t, e, p.delta) || (v_gt && e > 0.0);
    cnt[0] += (v_gt || v_est) ? 1 : 0;
    if (v_gt && v_est) {
      cnt[1] += 1;
      const double a = DIAM ? fabs(g - e) / diam : fabs(g - e);
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
    p.status[b] = (S[0] ? 0 : 1) | (p.cls_flag[b] ? 2 : 0) | (p.cams.bad(b) ? 8 : 0);
}

int vsd_launch(dim_ctx *ctx, const VsdCall &c, cudaStream_t st) {
  // stage profiling: one record per call, stage 0 = the two renders, stage 1 = VSD pass
  cudaEvent_t *ev;
  if (int rc = prof_begin(ctx, st, &ev)) return rc;
  {
    DimNvtxRange r("dim_pose_error_vsd render");
    if (int rc = f64_to_f32_launch(c.pose_gt, ctx->pose_cur_f32, c.B * 12, st)) return rc;
    if (int rc = render_launch(ctx, c.cls_idx, ctx->pose_cur_f32, c.B, c.zn, c.zf, nullptr,
                               {.cams = c.cams, .out_depth = ctx->mask_rendered, .trunc_u8 = 1, .ren4_depth = true}, st))
      return rc;
    DIM_CHECK(cudaMemcpyAsync(ctx->vsd_box, ctx->vbox, sizeof(int) * 4 * c.B, cudaMemcpyDeviceToDevice, st));
    if (int rc = f64_to_f32_launch(c.pose_est, ctx->pose_cur_f32, c.B * 12, st)) return rc;
    if (int rc = render_launch(ctx, c.cls_idx, ctx->pose_cur_f32, c.B, c.zn, c.zf, nullptr,
                               {.cams = c.cams, .out_ren4 = ctx->ren4, .trunc_u8 = 1, .ren4_depth = true}, st))
      return rc;
  }
  if (ev) DIM_CHECK(cudaEventRecord(ev[1], st));
  VsdParams p;
  p.ren4 = ctx->ren4; p.depth_gt = ctx->mask_rendered; p.vbox_est = ctx->vbox; p.vbox_gt = ctx->vsd_box;
  p.cls_flag = ctx->cls_flag; p.depth = c.depth; p.cams = c.cams;
  p.partial = ctx->vsd_partial; p.err = c.err; p.status = c.status; p.diam = c.diam;
  for (int k = 0; k < VSD_MAX_TAU; ++k) p.taus[k] = k < c.n_tau ? c.taus[k] : 0.0;
  p.delta = c.delta;
  p.B = c.B; p.H = ctx->H; p.W = ctx->W; p.chunks = cdiv(ctx->H, VSD_ROWS); p.n_tau = c.n_tau;
  {
    DimNvtxRange r("dim_pose_error_vsd pass");
    auto pass = c.visib_mode ? (c.diam ? vsd_pass_kernel<1, true> : vsd_pass_kernel<1, false>)
                             : (c.diam ? vsd_pass_kernel<0, true> : vsd_pass_kernel<0, false>);
    pass<<<dim3(p.chunks, c.B), VSD_THREADS, 0, st>>>(p);
    DIM_LAUNCH_CHECK();
    vsd_finish_kernel<<<cdiv(c.B, 64), 64, 0, st>>>(p);
    DIM_LAUNCH_CHECK();
  }
  if (ev)
    for (int k = 2; k < 5; ++k) DIM_CHECK(cudaEventRecord(ev[k], st));
  return 0;
}

}  // namespace dim
