// launch.cuh -- every host function one translation unit defines and another calls, and the structs they exchange; the
// defining .cu includes it too, so both sides compile against one declaration, default arguments and struct layout.
#pragma once
#include "common.cuh"

namespace dim {

struct LitParams { const float *light_pos, *light_int; float a0, a1; };  // device [B,3] each; a0 = 1 - ratio, a1 = ratio

struct TrainIO {
  const float *zio, *zir, *zmo, *zmr, *zoom_factor, *zflow, *zfw, *zmask_gt, *src_pose, *pc_model, *pc_weights, *pc_observed;
  int B, N;
  float *rot_est_norm, *trans_est, *flow_est, *mask_prob, *losses, *grads;
  float *rot_raw;  // nullable: the un-normalised quaternion of the test graph (se3 = [rot_raw, trans_est], symbol:716-725)
  // gradient-bucket readiness (overlap of the NCCL all-reduce with the rest of the backward pass): event k is recorded as
  // soon as every gradient of the tensors with table index >= bucket_first_tensor[k] has been produced
  void *const *bucket_events;
  const int *bucket_first_tensor;
  int n_buckets;
  const float *zdo, *zdr;  // RGB-D network: zoomed depth_observed / depth_rendered f32 [B,1,H,W]; nullptr otherwise
};

// raster.cu
// K_frames / frame_idx / n_frames (fused loop, RefineArgs): instance b projects with row frame_of(b) of the per-frame
// intrinsics [n_frames,9]; K_frames nullptr = K9 for every instance
int render_launch(dim_ctx *ctx, const int *cls, const float *pose, int B, const float *K9, float zn, float zf,
                  const double *means, int trunc_u8, float *out_image, float *out_depth, float *out_mask, float *out_bgr,
                  int *out_bbox, float4 *out_ren4, cudaStream_t st, const LitParams *lit = nullptr, bool ren4_depth = false,
                  bool colour_box = false, const float *K_frames = nullptr, const int32_t *frame_idx = nullptr,
                  int n_frames = 0);
// the data-preparation render (dim_render_dataset): file-ready outputs of one visibility pass, each nullable; ratio and the
// light arrays of LitParams are per instance and used only for lit_bgr
struct DatasetOut {
  uint8_t *lit_bgr, *bgr;  // [B,H,W,3] BGR
  uint16_t *depth;         // [B,H,W] (uint16)(depth * depth_factor)
  uint8_t *label;          // [B,H,W] depth != 0
  const float *ratio;      // device [B] brightness ratio
  float depth_factor;
};
int render_dataset_launch(dim_ctx *ctx, const int *cls, const float *pose, int B, const float *K9, float zn, float zf,
                          const float *light_pos, const float *light_int, const DatasetOut &o, cudaStream_t st);

// zoom.cu
int zoom_gather_launch(dim_ctx *ctx, int mode, const float *src, float *dst, const float *zoom_factor, int B, int C,
                       int inv, const float *param, cudaStream_t st);
int zoom_factor_launch(dim_ctx *ctx, const float *mask_real, const float *mask_ren, int C, const float *src_pose, int B,
                       const float *K9, float *zoom_factor, int *bbox_out, int *status, cudaStream_t st,
                       const float *img_means = nullptr);
// frame_idx / n_frames: the fused loop's map from instance to observed frame (RefineArgs); nullptr = frame b
// K_frames: the fused loop's per-frame intrinsics [n_frames,9] (RefineArgs); nullptr = K9 for every instance
int zoom_factor_from_ren_launch(dim_ctx *ctx, const int *bbox_ren, const float *src_pose, int B, const float *K9,
                                float *zoom_factor, int *bbox_out, int *status, cudaStream_t st,
                                const int32_t *frame_idx = nullptr, int n_frames = 0, const float *K_frames = nullptr);
int obs_colour_box_launch(dim_ctx *ctx, const float4 *obs4, int F, int *bbox_obs, cudaStream_t st);
int zoom_factor_from_boxes_launch(dim_ctx *ctx, const int *bbox_obs, const int *bbox_ren, const float *src_pose, int B,
                                  const float *K9, float *zoom_factor, int *bbox_out, int *status, cudaStream_t st,
                                  const int32_t *frame_idx = nullptr, int n_frames = 0, const float *K_frames = nullptr);
int box_mask_launch(dim_ctx *ctx, const int *bbox, int B, float *mask, cudaStream_t st);
int zoom_fused_launch(dim_ctx *ctx, const float4 *obs4, const float4 *ren4, const float *zoom_factor,
                      const float *means_rgb, int B, int Hs, int Ws, int pad, __nv_bfloat16 *hi, __nv_bfloat16 *lo,
                      cudaStream_t st, int f16, const double *means_d, bool depth = false, bool mask = true,
                      const int32_t *frame_idx = nullptr, int n_frames = 0);
int obs4_depth_launch(dim_ctx *ctx, float4 *obs4, int B, const float *depth, const uint16_t *depth_u16, float factor,
                      cudaStream_t st);
int pack_nhwc10_launch(dim_ctx *ctx, const float *io, const float *ir, const float *dobs, const float *dren, const float *mo,
                       const float *mr, int B, int Hs, int Ws, int pad, __nv_bfloat16 *hi, __nv_bfloat16 *lo, cudaStream_t st,
                       int f16);
int pack_obs4_launch(dim_ctx *ctx, const float *img, int B, float4 *out, const double *means, cudaStream_t st);
int pack_nhwc8_launch(dim_ctx *ctx, const float *io, const float *ir, const float *mo, const float *mr, int B, int Hs,
                      int Ws, int pad, __nv_bfloat16 *hi, __nv_bfloat16 *lo, cudaStream_t st, int f16);
int group_pick_launch(const float *in, const float *group_idx, int B, int Ctot, int groups, size_t n, float *out,
                      int backward, cudaStream_t st);

// geom.cu
int flow_launch(dim_ctx *ctx, const float *depth_src, const float *depth_tgt, const float *KT, const float *Kinv, int B,
                float *flow, float *valid, float *valid2, cudaStream_t st);
int se3_compose_launch(const double *pose_src, const float *se3, int B, const double *Tm, const double *Ts, int rot_coord,
                       double *pose_out, float *pose_out_f32, cudaStream_t st);
int train_pose_launch(const float *src_pose, const float *rot_est, const float *trans_est, const float *tgt_pose, int B,
                      const double *Tm, const double *Ts, int rot_coord, const double *K9, float *pose_new_f32,
                      float *rot_label, float *trans_label, float *KT, cudaStream_t st, float *light_pos = nullptr,
                      const double *light_offset = nullptr);
int f64_to_f32_launch(const double *a, float *b, int n, cudaStream_t st);
int pose_light_launch(const double *pose, float *pose_f32, float *light_pos, int B, const double *offset, cudaStream_t st);
int zoom_trans_launch(const float *zoom_factor, const float *in, int B, int mul, int scale_xy, float *out, cudaStream_t st);
int transform3d_fwd_launch(const float *pc, const float *rot, const float *tr, const float *ps, int B, int N,
                           const float *Tm, const float *Ts, int rot_coord, float *out, cudaStream_t st);
int transform3d_bwd_launch(const float *og, const float *pc, const float *rot, const float *tr, const float *ps, int B,
                           int N, const float *Tm, const float *Ts, int rot_coord, float *rot_grad, float *trans_grad,
                           cudaStream_t st);
int transform_u8_launch(dim_ctx *ctx, const uint8_t *bgr, int B, const double *means, float *out, cudaStream_t st);
int transform_u8_obs4_launch(dim_ctx *ctx, const uint8_t *bgr, int B, const double *means, float4 *out, cudaStream_t st);
int epe_launch(const float *pred, const float *gt, const float *visible, const float *bg, int B, int P, double *out,
               cudaStream_t st);
int pose_error2d_launch(const double *pose_est, const double *pose_gt, int M, const double *pts, int N, const double *K9,
                        double *out3, cudaStream_t st);
int pose_error_launch(const double *pose_est, const double *pose_gt, int M, const double *pts, int N, int symmetric,
                      double *out, cudaStream_t st);

// augment.cu
struct BgGeom { int crop_h, crop_w, dst_h, dst_w; double scale; };  // scale = cv2.resize's fx = fy
struct BgInst {  // one instance of dim_replace_background; data == nullptr keeps the observed image
  const uint8_t *data;  // the bank photo, BGR u8 [h, stride, 3]; the crop is its top-left crop_h x crop_w
  double inv_scale;     // 1 / scale
  int stride, crop_h, crop_w, dst_h, dst_w, pad;
};
constexpr int BG_LAUNCH_MAX = 32;  // instances per launch (the per-instance table travels as a kernel argument)
struct BgLaunch { BgInst inst[BG_LAUNCH_MAX]; double mean[3]; int b0, pad; };
int bg_geometry(int H, int W, int bh, int bw, BgGeom *g);
int replace_bg_launch(dim_ctx *ctx, const BgLaunch &L, int nb, const float *obs, const float *mask, float *image,
                      uint8_t *comp, cudaStream_t st);
int mask_dilate_launch(dim_ctx *ctx, const float *in, const int *draws, int B, float *out, cudaStream_t st);

// icp.cu
constexpr int ICP_ROWS = 8;   // frame rows per association CTA
constexpr int ICP_SLOT = 30;  // doubles per CTA slot: A (21 upper entries), g (6), inliers, sum r^2, model pixels
struct IcpCall {  // dim_icp's arguments, checked
  const float *depth;  // [F,H,W] metres
  int F;
  const int32_t *frame_idx;
  const float *K9, *K_frames;  // exactly one non-null
  const int32_t *cls_idx;
  const double *pose_in;
  int B, n_iter;
  float zn, zf, max_dist;
  int min_points;
  double *poses_out;
  int32_t *inliers, *status;
  float *rms;
};
int icp_launch(dim_ctx *ctx, const IcpCall &c, cudaStream_t st);
int depth_u16_launch(const uint16_t *in, size_t n, float factor, float *out, cudaStream_t st);

// vsd.cu
constexpr int VSD_ROWS = 8;                     // frame rows per VSD pass CTA
constexpr int VSD_MAX_TAU = 16;
constexpr int VSD_SLOT = 2 + VSD_MAX_TAU;       // int32 per CTA slot: |union|, |inter|, c_tau
struct VsdCall {  // dim_pose_error_vsd's arguments, checked
  const float *depth;  // [F,H,W] metres
  int F;
  const int32_t *frame_idx;
  const float *K9, *K_frames;  // exactly one non-null
  const int32_t *cls_idx;
  const double *pose_est, *pose_gt;
  int B;
  float zn, zf, delta;
  const double *taus;  // host [n_tau]
  int n_tau;
  double *err;
  int32_t *status;  // nullable
};
int vsd_launch(dim_ctx *ctx, const VsdCall &c, cudaStream_t st);

// net.cu
int net_create(dim_ctx *ctx);
void net_destroy(dim_ctx *ctx);
int net_load(dim_ctx *ctx, const float *const *W, const float *const *Bv);
int net_alloc_weights(dim_ctx *ctx);
// net_pack_weights' `packs`: the bf16 hi packs (with fc7^T), the bf16x3 lo halves, the fp16 packs
enum : unsigned { PACK_HI = 1, PACK_LO = 2, PACK_F16 = 4 };
int net_pack_weights(dim_ctx *ctx, const float *const *w, cudaStream_t st, unsigned packs);
void net_input_geometry(dim_ctx *ctx, int *rows, int *cols, int *pad, __nv_bfloat16 **hi, __nv_bfloat16 **lo);
int net_forward(dim_ctx *ctx, int B, int precision, const float *zoom_factor, float *rot_out, float *trans_out,
                float *se3_out, cudaStream_t st, cudaEvent_t after_conv);
bool net_graph_safe(dim_ctx *ctx);
int net_set_input_depth(dim_ctx *ctx, bool enable);
bool net_input_depth(dim_ctx *ctx);
int net_set_input_mask(dim_ctx *ctx, bool enable);
bool net_input_mask(dim_ctx *ctx);
int net_layer_profile(dim_ctx *ctx, int enable, float *ms10);
int net_debug_activation(dim_ctx *ctx, int idx, int lo, void *host_dst, size_t bytes);
void net_layer_geometry(dim_ctx *ctx, int idx, int *out /*rows, cols, Cbuf, py, px, Ho, Wo, Cout*/);

// train.cu
int train_create(dim_ctx *ctx, int max_points);
void train_destroy(dim_ctx *ctx);
int train_load_params(dim_ctx *ctx, const float *flat_host, size_t n, cudaStream_t st);
int train_refresh_lo(dim_ctx *ctx, cudaStream_t st);
int train_refresh_f16(dim_ctx *ctx, cudaStream_t st);
void train_drop_maps(dim_ctx *ctx);
int train_get_params(dim_ctx *ctx, float *flat_host, size_t n, int which, cudaStream_t st);
size_t train_param_count(dim_ctx *ctx);
int train_param_info(int idx, const char **name, long long *w_numel, long long *b_numel, bool input_depth, bool input_mask);
int train_forward_backward(dim_ctx *ctx, const TrainIO &io, cudaStream_t st);
int train_sgd_update(dim_ctx *ctx, const float *grads, float lr, float momentum, float wd, float rescale, cudaStream_t st);
int train_set_precision(dim_ctx *ctx, int precision);
int train_get_precision(dim_ctx *ctx, int *precision);
int train_debug_tensor(dim_ctx *ctx, int id, void *host, size_t bytes);
int train_debug_phases(dim_ctx *ctx, float *ms7);
void train_debug_geometry(dim_ctx *ctx, int id, int *out /*Hp, Wp, py, px, C, H, W*/);
int train_debug_wgrad_slices(dim_ctx *ctx, int B, int *out36);

}  // namespace dim
