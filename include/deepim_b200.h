/*
 * deepim_b200.h -- C ABI of libdeepim_b200.so (hand-written sm_90a CUDA, no CPU fallback).
 *
 * Drop-in boundary for the mx-DeepIM render-and-compare hot path.  Each entry point names the
 * reference interface it replaces (paths relative to the mx-DeepIM repo).  The reference binds its
 * native/GPU pieces from Python (mx.operator.CustomOp classes in deepim/operator_py/, the Cython
 * wrapper lib/flow_c/gpu_flow.pyx, the glumpy renderer class); the matching binding here is the
 * ctypes stub shown in INTEGRATION.md and shipped as mx-deepim_b200/deepim_b200/_capi.py.
 *
 * Conventions
 *   - all tensor pointers are DEVICE pointers owned by the caller, contiguous, NCHW float32 unless
 *     noted; "host" in a parameter comment means a host pointer (small attribute arrays);
 *   - `stream` is a cudaStream_t passed as void*; every call is asynchronous on it and allocates
 *     nothing (all scratch is sized by dim_ctx_create); one context per device, not thread-safe;
 *   - return 0 on success, non-zero on error; dim_last_error() gives the message
 *     (the reference ops raise Python exceptions instead; the Python shims re-raise);
 *   - H, W are fixed per context (480 x 640 in every shipped config).
 */
#ifndef DEEPIM_B200_H_
#define DEEPIM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define DIM_API
#else
#define DIM_API __attribute__((visibility("default")))
#endif

typedef struct dim_ctx dim_ctx;

#define DIM_ABI_VERSION 4
DIM_API int32_t dim_abi_version(void);
DIM_API const char *dim_last_error(void);

/* Context: owns meshes, weights and all scratch.  max_verts/max_faces bound the largest mesh.
 * Replaces the per-process state of Render_Py.__init__ (lib/render_glumpy/render_py_multi.py:54-99)
 * and of the MXNet executor (deepim/core/tester.py:41-43). */
DIM_API int32_t dim_ctx_create(int32_t device, int32_t max_batch, int32_t height, int32_t width,
                               int32_t max_classes, int32_t max_verts, int32_t max_faces,
                               dim_ctx **out);
DIM_API void dim_ctx_destroy(dim_ctx *ctx);

/* Upload one class mesh (host pointers).  verts f32[V,3] metres, uvs f32[V,2], faces i32[F,3],
 * tex u8[Th,Tw,3] RGB with row 0 = v 0 (i.e. already flipped as render_py_multi.py:76 does).
 * Replaces data.objload + gloo.Program.bind + u_texture upload (render_py_multi.py:72-76). */
DIM_API int32_t dim_mesh_upload(dim_ctx *ctx, int32_t cls_idx, const float *verts_host,
                                const float *uvs_host, int32_t V, const int32_t *faces_host,
                                int32_t F, const uint8_t *tex_host, int32_t Th, int32_t Tw);

/* Rasterise B instances.  Replaces Render_Py.render (render_py_multi.py:101-129) plus the
 * post-render glue (deepim/core/tester.py:185-188,433-442; lib/utils/image.py:583-594).
 *   cls_idx i32[B] (device), pose f32[B,3,4] (device), K9 host f32[9], pixel_means_rgb host f64[3]
 *   trunc_u8: 1 = test path (uint8 truncation, tester.py:188), 0 = train path
 *   outputs (each may be NULL):
 *     out_image f32[B,3,H,W] RGB - means;  out_depth f32[B,1,H,W] metres;  out_mask f32[B,1,H,W]
 *     out_bgr f32[B,H,W,3] BGR in [0,255] (the Render_Py return layout);
 *     out_bbox i32[B,4] x0,x1,y0,y1 of out_mask (min/max nonzero col/row; -1 when empty). */
DIM_API int32_t dim_render(dim_ctx *ctx, const int32_t *cls_idx, const float *pose, int32_t B,
                           const float *K9_host, float znear, float zfar,
                           const double *pixel_means_rgb_host, int32_t trunc_u8, float *out_image,
                           float *out_depth, float *out_mask, float *out_bgr, int32_t *out_bbox,
                           void *stream);

/* ZoomMask forward (deepim/operator_py/zoom_mask.py:29-112).
 * in : mask_observed, mask_gt_observed, mask_rendered f32[B,1,H,W]; src_pose f32[B,3,4]; K9 host
 * out: 3 zoomed masks f32[B,1,H,W] (any may be NULL), zoom_factor f32[B,4],
 *      bbox i32[B,8] = observed x0,x1,y0,y1, rendered x0,x1,y0,y1 (may be NULL),
 *      status i32[B] (may be NULL): 1 where the observed mask is empty (the reference raises). */
DIM_API int32_t dim_zoom_mask_fwd(dim_ctx *ctx, const float *mask_observed,
                                  const float *mask_gt_observed, const float *mask_rendered,
                                  const float *src_pose, int32_t B, const float *K9_host,
                                  float *zoom_mask_observed, float *zoom_mask_gt_observed,
                                  float *zoom_mask_rendered, float *zoom_factor, int32_t *bbox,
                                  int32_t *status, void *stream);

/* ZoomImageWithFactor forward (zoom_image_with_factor.py:31-65). pixel_means_rgb host f32[3] is the
 * already-reversed attr (l.79-81).  images f32[B,3,H,W]. */
DIM_API int32_t dim_zoom_image_with_factor_fwd(dim_ctx *ctx, const float *zoom_factor,
                                               const float *image_observed,
                                               const float *image_rendered, int32_t B,
                                               const float *pixel_means_rgb_host,
                                               float *zoom_image_observed,
                                               float *zoom_image_rendered, void *stream);

/* Lit renderer (lib/render_glumpy/render_py_light_modelnet_multi.py:36-79 shader, 131-175 render): Lambert shading
 * colour = texel * ((1 - brightness_ratio) + brightness_ratio * clamp(cos(normal, light - position), 0, 1)) *
 * light_intensity, quantised to 8 bits like the framebuffer the reference reads back.  normals f32[V,3] (host) per
 * class; light_position / light_intensity f32[B,3] (device), position in the GL camera frame (x, -y, -z of the
 * OpenCV frame).  Outputs as dim_render (out_bgr holds the quantised colours as floats). */
DIM_API int32_t dim_mesh_upload_normals(dim_ctx *ctx, int32_t cls_idx, const float *normals_host, int32_t V);
DIM_API int32_t dim_render_lit(dim_ctx *ctx, const int32_t *cls_idx, const float *pose, int32_t B,
                               const float *K9_host, float znear, float zfar,
                               const double *pixel_means_rgb_host, const float *light_position,
                               const float *light_intensity, float brightness_ratio, float *out_image,
                               float *out_depth, float *out_mask, float *out_bgr, int32_t *out_bbox,
                               void *stream);

/* Data-preparation render (toolkit/LM6d_ds_1 .. ds_4, LM6d_0_gen_gt_observed.py): what the dataset files hold, from one
 * rasterisation of B instances.
 *   lit_bgr   u8[B,H,W,3]  Render_Py_Light colour (lib/render_glumpy/render_py_light.py get_fragment):
 *                          texel * ((1 - ratio) + (ratio * brightness) * light_intensity), brightness as dim_render_lit,
 *                          quantised to 8 bits.  The light colour scales only the diffuse term (dim_render_lit scales
 *                          both);
 *   bgr       u8[B,H,W,3]  unlit colour, Render_Py.render(...).astype('uint8');
 *   depth_u16 u16[B,H,W]   (uint16)(depth * depth_factor), truncated like numpy's astype(np.uint16);
 *   label     u8[B,H,W]    depth != 0.
 * Every output may be NULL.  light_position / light_intensity f32[B,3] and brightness_ratio f32[B] are device arrays,
 * given exactly when lit_bgr is (the call is refused otherwise); a lit call needs normals for every uploaded mesh
 * (dim_mesh_upload_normals). */
DIM_API int32_t dim_render_dataset(dim_ctx *ctx, const int32_t *cls_idx, const float *pose, int32_t B,
                                   const float *K9_host, float znear, float zfar, float depth_factor,
                                   const float *light_position, const float *light_intensity,
                                   const float *brightness_ratio, uint8_t *lit_bgr, uint8_t *bgr,
                                   uint16_t *depth_u16, uint8_t *label, void *stream);

/* ZoomImage forward (zoom_image.py:26-107, the INPUT_MASK: False front end): the two boxes come from the
 * images themselves, valid = sum_c(image + pixel_mean_c) > 0.01; centre / crop / sampling as ZoomMask +
 * ZoomImageWithFactor.  pixel_means_rgb_host = the op's (already reversed) pixel_means attr.
 * bbox i32[B,8] / status i32[B] as dim_zoom_mask_fwd (may be NULL). */
DIM_API int32_t dim_zoom_image_fwd(dim_ctx *ctx, const float *image_observed, const float *image_rendered,
                                   const float *src_pose, int32_t B, const float *K9_host,
                                   const float *pixel_means_rgb_host, float *zoom_image_observed,
                                   float *zoom_image_rendered, float *zoom_factor, int32_t *bbox,
                                   int32_t *status, void *stream);

/* GroupPicker (group_picker.py:22-60): forward out[b] = in[b, g*cg:(g+1)*cg] (g = group_idx[b], a float like the
 * NDArray the reference reads); backward = 1 scatters out_grad (in) into a zero [B,channels,...] gradient. */
DIM_API int32_t dim_group_picker(dim_ctx *ctx, const float *in, const float *group_idx, int32_t B,
                                 int32_t channels, int32_t group_num, int64_t elems_per_channel,
                                 int32_t backward, float *out, void *stream);

/* ZoomMaskWithFactor forward (zoom_mask_with_factor.py:29-64): mask f32[B,1,H,W]. */
DIM_API int32_t dim_zoom_mask_with_factor_fwd(dim_ctx *ctx, const float *zoom_factor,
                                              const float *mask, int32_t B, int32_t b_inv_zoom,
                                              float *zoom_mask, void *stream);

/* ZoomFlow forward (zoom_flow.py:28-71): flow f32[B,2,H,W]; flow_weights/zoom_flow_weights
 * f32[B,fw_channels,H,W] (1, or 2 as tiled by batch_updater_py_multi.py:293-296) used only when
 * b_inv_zoom == 0 (may be NULL). */
DIM_API int32_t dim_zoom_flow_fwd(dim_ctx *ctx, const float *zoom_factor, const float *flow,
                                  const float *flow_weights, int32_t fw_channels, int32_t B,
                                  int32_t b_inv_zoom, float *zoom_flow, float *zoom_flow_weights,
                                  void *stream);

/* ZoomDepth forward (zoom_depth.py:24-44): depth f32[B,1,H,W] x2. */
DIM_API int32_t dim_zoom_depth_fwd(dim_ctx *ctx, const float *zoom_factor,
                                   const float *depth_observed, const float *depth_rendered,
                                   int32_t B, float *zoom_depth_observed,
                                   float *zoom_depth_rendered, void *stream);

/* ZoomTrans forward / backward (zoom_trans.py:22-74): trans f32[B,3]. */
DIM_API int32_t dim_zoom_trans_fwd(dim_ctx *ctx, const float *zoom_factor, const float *trans_delta,
                                   int32_t B, int32_t b_inv_zoom, float *zoom_trans_delta,
                                   void *stream);
DIM_API int32_t dim_zoom_trans_bwd(dim_ctx *ctx, const float *zoom_factor, const float *out_grad,
                                   int32_t B, int32_t b_inv_zoom, int32_t b_zoom_grad,
                                   float *trans_grad, void *stream);

/* mask_observed := end-exclusive bbox rectangle of mask_rendered
 * (lib/pair_matching/data_pair.py:93-105).  bbox i32[B,4] as written by dim_render. */
DIM_API int32_t dim_update_mask_box(dim_ctx *ctx, const int32_t *bbox, int32_t B,
                                    float *mask_observed, void *stream);

/* SE(3) compose in float64 (lib/pair_matching/RT_transform.py:127-151).
 * pose_src f64[B,3,4], se3 f32[B,7] = (quat w,x,y,z un-normalised, trans), T_means/T_stds host
 * f64[3], rot_coord 0 MODEL / 1 CAMERA / 2 CAMERA_NEW; pose_out f64[B,3,4]. */
DIM_API int32_t dim_se3_compose(dim_ctx *ctx, const double *pose_src, const float *se3, int32_t B,
                                const double *T_means_host, const double *T_stds_host,
                                int32_t rot_coord, double *pose_out, void *stream);

/* Reprojection-flow labels (lib/flow_c/gpu_flow_kernel.cu:32-69 flow_kernel, gpu_flow.pyx:24-41).
 * depth_src, depth_tgt f32[B,1,H,W]; KT f32[B,3,4] = K.T_src->tgt; Kinv host f32[9];
 * flow f32[B,2,H,W] (dh,dw), valid f32[B,1,H,W]. */
DIM_API int32_t dim_flow_fwd(dim_ctx *ctx, const float *depth_src, const float *depth_tgt,
                             const float *KT, const float *Kinv_host, int32_t B, float *flow,
                             float *valid, void *stream);

/* Transform3D forward / backward (deepim/operator_py/transform3d.py:34-151).
 * point_cloud f32[B,3,N], rotation f32[B,4], translation f32[B,3], pose_src f32[B,3,4]. */
DIM_API int32_t dim_transform3d_fwd(dim_ctx *ctx, const float *point_cloud, const float *rotation,
                                    const float *translation, const float *pose_src, int32_t B,
                                    int32_t N, const float *T_means_host, const float *T_stds_host,
                                    int32_t rot_coord, float *out_points, void *stream);
DIM_API int32_t dim_transform3d_bwd(dim_ctx *ctx, const float *out_grad, const float *point_cloud,
                                    const float *rotation, const float *translation,
                                    const float *pose_src, int32_t B, int32_t N,
                                    const float *T_means_host, const float *T_stds_host,
                                    int32_t rot_coord, float *rot_grad, float *trans_grad,
                                    void *stream);

/* Lighting of the ModelNet / unseen-object configuration (config.dataset.dataset "ModelNet*": deepim/core/tester.py:114-133,
 * 146-185; lib/pair_matching/batch_updater_py_multi.py:35-52,187-229).  The `lighting` argument of dim_train_update,
 * dim_refine and dim_refine_host_async: NULL = the unlit renderer; otherwise every render of the call is the Lambert-lit
 * renderer of dim_render_lit.  The light follows the pose being rendered: in the GL camera frame
 *   light_position = float32(offset[0] + t_x, offset[1] - t_y, offset[2] - t_z)
 * computed from the float64 pose (the reference's hard-coded light index 2 gives offset = (0, 0.5, 0.5)).  The reference
 * draws light_intensity from U(0.9, 1.1)^3 afresh for every render; here the caller supplies the draws.
 *   intensity (non-NULL): device f32 [n_iter,B,3] for dim_refine (iteration it renders with intensity[it]), [B,3] for
 *              dim_train_update, HOST f32 [n_iter,B,3] for dim_refine_host_async (n_iter <= 8; copied to the
 *              context on `stream` before the call returns, so a pageable buffer may be reused at once).
 *   brightness_ratio: colour = texel * ((1 - ratio) + ratio * brightness) * intensity (the reference: 0.7).
 * Depth, masks, bboxes, zoom, labels and flow are those of the unlit calls; only the colours change.  Every uploaded mesh
 * must have normals (dim_mesh_upload_normals).  Lit loops share dim_refine_status and are captured / replayed as CUDA
 * graphs like unlit ones. */
typedef struct dim_lighting {
  const float *intensity; /* see above: device [n_iter,B,3] (refine) / [B,3] (train update); host for dim_refine_host_async */
  double offset[3];       /* light at zero translation, GL frame; the reference: (0, 0.5, 0.5) */
  float brightness_ratio; /* the reference: 0.7 */
} dim_lighting;

/* Train-time inter-iteration update (lib/pair_matching/batch_updater_py_multi.py:91-328,
 * batchUpdaterPyMulti.forward): compose the predicted delta onto src_pose, re-render WITHOUT uint8
 * truncation (float32 image - float32 means, l.184,234), recompute the labels rot (quaternion of
 * calc_RT_delta(..., "QUAT")), trans, the reprojection flow against depth_gt_observed and its weights
 * (valid tiled to 2 channels).  mask_observed / image_observed / tgt_pose stay fixed (not touched).
 *   in : cls_idx i32[B], src_pose/tgt_pose f32[B,3,4], rot_est f32[B,4], trans_est f32[B,3],
 *        depth_gt_observed f32[B,1,H,W] (may be NULL when flow == NULL); K9 / T_means / T_stds /
 *        pixel_means_rgb host f64
 *   out: image_rendered f32[B,3,H,W], depth_rendered/mask_rendered f32[B,1,H,W], src_pose_new f32[B,3,4],
 *        rot_label f32[B,4], trans_label f32[B,3], flow f32[B,2,H,W], flow_weights f32[B,2,H,W]
 *        (flow, flow_weights may be NULL together).
 *   lighting (nullable, see dim_lighting): the ModelNet re-render (l.187-235); the light follows the float64 refined pose,
 *        image_rendered = float32 quantised lit colours - float32 means; every other output is the unlit one. */
DIM_API int32_t dim_train_update(dim_ctx *ctx, const int32_t *cls_idx, const float *src_pose,
                                 const float *rot_est, const float *trans_est, const float *tgt_pose,
                                 const float *depth_gt_observed, int32_t B, const double *K9_host,
                                 float znear, float zfar, const double *pixel_means_rgb_host,
                                 const double *T_means_host, const double *T_stds_host,
                                 int32_t rot_coord, float *image_rendered, float *depth_rendered,
                                 float *mask_rendered, float *src_pose_new, float *rot_label,
                                 float *trans_label, float *flow, float *flow_weights,
                                 const dim_lighting *lighting, void *stream);

/* Network variants.  A context runs one of three networks, chosen before dim_net_load / dim_train_create (either switch
 * is an error afterwards); a context that never switches runs the mask network.
 *   - mask network (INPUT_MASK on): conv1 sees concat(image_observed/255, image_rendered/255, mask_observed,
 *     mask_rendered), flow_conv1_weight (64, 8, 7, 7).
 *   - RGB-D network (config.network.INPUT_DEPTH: deepIM_flownet.py:33-51, tester.py:437-438), dim_ctx_set_input_depth(ctx,
 *     1): the input gains two channels, in the order image_observed/255, image_rendered/255, depth_observed/255,
 *     depth_rendered/255, mask_observed, mask_rendered, so flow_conv1_weight is (64, 10, 7, 7).  The depths are metres,
 *     divided by 255 as the reference does; depth_rendered is each iteration's render depth (0 = background), zoomed with
 *     the iteration's zoom factor like every other input (ZoomDepth, zoom_depth.py:24-44).
 *   - image-only network (config.network.INPUT_MASK: False, the reference's default; deepIM_flownet.py:53-62,
 *     tester.py:439), dim_ctx_set_input_mask(ctx, 0): conv1 sees concat(image_observed/255, image_rendered/255), so
 *     flow_conv1_weight is (64, 6, 7, 7), and the test graph zooms with ZoomImage (zoom_image.py:26-107, the boxes of
 *     sum_c(image + mean) > 0.01) instead of ZoomMask + ZoomImageWithFactor.
 * dim_ctx_set_input_depth: enable = 1 switches to the RGB-D network, 0 back.  dim_ctx_set_input_mask: enable = 0 switches
 * to the image-only network, 1 back.  Depth input without the mask channels (INPUT_DEPTH without INPUT_MASK) is not
 * supported: each switch refuses it.
 * Every entry point follows the context's network, with these rules:
 *   - depth inputs (depth_frames of dim_refine, depth_frames_u16_host of dim_refine_host_async, zoom_depth_* of
 *     dim_net_fwd and dim_train_forward_backward) are non-NULL exactly on an RGB-D context; otherwise the call fails with a
 *     message naming the argument and dim_ctx_set_input_depth;
 *   - mask inputs (zoom_mask_* of dim_net_fwd and dim_train_forward_backward) are NULL exactly on an image-only context;
 *   - dim_net_load takes the network's flow_conv1 weight; the flat training vector is the network's table
 *     (dim_train_param_info) and dim_train_param_count reports its size.
 * On an image-only context dim_refine / dim_refine_host_async run the image-only chain: the observed box is computed once
 * per call, the rendered box of every iteration from the render's colours; the zoom factor is ZoomImage's (ZoomMask's
 * arithmetic with the observed-centre fallback for an empty render).  dim_refine_status: bit 0 = the observed image has no
 * valid pixel (the reference raises; the fallback factor (1,1,0,0) was used), bit 2 = the rendered image has none (the
 * zoom centres on the observed box, as the reference does), bit 1 unchanged.  dim_train_update is the same for every
 * network: with PRED_MASK the reference's training graph still zooms with ZoomMask and learns the mask; only the network
 * input loses the mask channels. */
DIM_API int32_t dim_ctx_set_input_depth(dim_ctx *ctx, int32_t enable);
DIM_API int32_t dim_ctx_set_input_mask(dim_ctx *ctx, int32_t enable);

/* FlowNetS weights (deepim/symbols/deepIM_flownet.py:63-116,716-717; MXNet layouts: Convolution
 * (Cout,Cin,kh,kw), FullyConnected (out,in)).  Host float32 pointers, 14 (weight,bias) pairs in the
 * order flow_conv1, conv2, conv3, conv3_1, conv4, conv4_1, conv5, conv5_1, conv6, conv6_1, fc6,
 * fc7, rot, trans.  Replaces load_param + Module.init_params (deepim/core/tester.py:41-43). */
DIM_API int32_t dim_net_load(dim_ctx *ctx, const float *const *weights_host,
                             const float *const *biases_host);

/* precision of the conv stack */
#define DIM_PREC_BF16 0   /* one bf16 wgmma pass, fp32 accumulate (throughput mode)            */
#define DIM_PREC_BF16X3 1 /* hi/lo split, 3 wgmma passes, ~fp32 accuracy (parity mode)         */
#define DIM_PREC_FP16 2   /* one fp16 wgmma pass (11 significant bits), fp32 accumulate, saturating stores:
                             the single-pass mode that meets the 1e-4 rot / 1e-3 trans se3 tolerance (headline mode) */

/* Encoder + fc + heads on already-zoomed blobs (get_convs, deepIM_flownet.py:53-116; heads
 * l.716-717): inputs f32 NCHW as the op surface produces them (zoomed depths f32 [B,1,H,W] in metres, zoomed masks
 * f32 [B,1,H,W]; NULL as the network variant says); rot f32[B,4] raw quaternion, trans f32[B,3] zoomed translation. */
DIM_API int32_t dim_net_fwd(dim_ctx *ctx, const float *zoom_image_observed,
                            const float *zoom_image_rendered, const float *zoom_depth_observed,
                            const float *zoom_depth_rendered, const float *zoom_mask_observed,
                            const float *zoom_mask_rendered, int32_t B, int32_t precision,
                            float *rot, float *trans, void *stream);

/* The fused test-time loop (deepim/core/tester.py:340-485 with FAST_TEST / UPDATE_MASK
 * box_rendered): n_iter x (render -> bbox+zoom -> FlowNetS -> ZoomTrans^-1 -> RT_transform),
 * everything on the device, no host sync.  Two entries run it: dim_refine on device buffers, dim_refine_host_async on host
 * buffers.  Both take B instances observing F frames, 1 <= B, F <= max_batch; each frame is uploaded (host entry) and
 * packed once per call, however many instances observe it.
 *   frame_idx i32[B] or NULL: instance b observes frame frame_idx[b] (several objects of one image, or several initial
 *     hypotheses of one object); its results equal those of a call with frame frame_idx[b] as frame b, bit for bit.
 *     NULL: instance b observes frame b, and F must equal B (the call is refused otherwise).
 *   K9_host f32[9] (one camera for every instance) or K_frames f32[F,9] (one camera per frame, row-major): exactly one is
 *     non-NULL (the call is refused otherwise).  K_frames is read through the frame map: instance b is rendered and zoomed
 *     with K_frames[frame_of(b)] -- the frame whose taps it observes; row b without a map.  One K serves both the render
 *     and the zoom centre K . t (the reference's per-pair `<observed>-K.txt`, tester.py:424-427, zooms with the config's K
 *     even when the pair has its own).  Instance b's results equal those of K9 = K_frames[frame_of(b)], bit for bit.
 *   cls_idx i32[B]; pose_init f64[B,3,4].
 *   lighting: nullable, see dim_lighting.  Image-only network: the observed box is computed once per frame.
 *
 * dim_refine: every pointer but K9_host / pixel_means_rgb_host is a device pointer.
 *   image_frames f32[F,3,H,W] RGB-mean (constant over iterations); depth_frames: RGB-D network only, f32 [F,1,H,W] in
 *   metres; lighting->intensity device [n_iter,B,3].
 *   frame_idx is not checked on the host: an index outside [0, F) makes the instance observe frame 0 (and use K_frames
 *   row 0) and sets status bit 3 (dim_refine_status) in every iteration; nothing is read outside the F frames.  K_frames
 *   is read as given (not checked).
 *   outputs: poses f64[n_iter,B,3,4], se3 f32[n_iter,B,7], zoom_factor f32[n_iter,B,4],
 *   bbox i32[n_iter,B,8]; any of the last three may be NULL.
 *   pose_override f64[n_iter,B,3,4] or NULL: when given, iteration `it` starts from
 *   pose_override[it] instead of the previous estimate (teacher forcing for parity tests).
 *   After one eager run of an argument set the chain is captured as a CUDA graph and replayed (keyed on every argument,
 *   the depth, intensity, frame_idx and K_frames pointers included).  The graph reads frame_idx and K_frames at replay:
 *   new indices or intrinsics written into the same buffers need no re-capture; another buffer is another graph.
 *
 * dim_refine_host_async: host buffers (what deepim/core/tester.py:pred_eval would call).  frames_u8_host u8[F,H,W,3] BGR
 *   (as cv2.imread returns; transformed on device as lib/utils/image.py:583-594), frame_idx_host / K_frames_host /
 *   cls_idx_host / pose_init_host on the host; poses_out_host f64[n_iter,B,3,4], se3_out_host f32[n_iter,B,7] (nullable);
 *   n_iter in [1, 8].
 *   depth_frames_u16_host: RGB-D network only, the host depth file values u16 [F,H,W], converted on the device as
 *   lib/utils/image.py:203,218 does: float32(u16) / float32(depth_factor) (LINEMOD: 1000; depth_factor is checked only
 *   when a depth is given).  lighting->intensity HOST [n_iter,B,3] (copied to the context on `stream` before the call
 *   returns, so a pageable buffer may be reused at once).
 *   Every class index, frame index and K_frames_host row is checked before anything is enqueued: a class index without a
 *   mesh, a frame index outside [0, F) or a row that is not a finite pinhole matrix [[fx,0,cx],[0,fy,cy],[0,0,1]] with
 *   fx, fy > 0 fails the call with a message naming the instance or frame.  K9_host is not checked.
 *   Returns right after enqueueing the copies and kernels on `stream` (no synchronisation): the host output buffers are
 *   valid once the stream has been synchronised.  Pinned buffers are recommended; they let a caller overlap the H2D copy
 *   of batch k+1 (second context / stream) with the compute of k. */
DIM_API int32_t dim_refine(dim_ctx *ctx, const float *image_frames, int32_t F, const int32_t *frame_idx,
                           const float *K9_host, const float *K_frames, const int32_t *cls_idx,
                           const double *pose_init, int32_t B, int32_t n_iter, float znear, float zfar,
                           const double *pixel_means_rgb_host, int32_t precision, const double *pose_override,
                           double *poses, float *se3, float *zoom_factor, int32_t *bbox,
                           const float *depth_frames, const dim_lighting *lighting, void *stream);
DIM_API int32_t dim_refine_host_async(dim_ctx *ctx, const uint8_t *frames_u8_host, int32_t F,
                                      const int32_t *frame_idx_host, const float *K9_host,
                                      const float *K_frames_host, const int32_t *cls_idx_host,
                                      const double *pose_init_host, int32_t B, int32_t n_iter, float znear,
                                      float zfar, const double *pixel_means_rgb_host, int32_t precision,
                                      double *poses_out_host, float *se3_out_host,
                                      const uint16_t *depth_frames_u16_host, float depth_factor,
                                      const dim_lighting *lighting, void *stream);

/* Per-iteration status of the LAST dim_refine / dim_refine_host_async call on this context, copied device -> host
 * asynchronously on `stream` (the stream that call ran on): [min(n_iter,8), B] int32.
 * 0 = ok; bit 0 = the rendered mask of that iteration was empty (the reference crashes there: np.min of an empty array,
 * zoom_mask.py:55-58; here the fallback zoom factor was used and the instance's pose is meaningless); bit 1 = class index
 * out of range or no mesh uploaded for that class (the reference indexes a python list and raises); bit 2 = image-only
 * network, empty render (see the network variants); bit 3 = dim_refine with a frame map only: the instance's frame index
 * lies outside [0, F), so it observed frame 0 instead (its pose is meaningless). */
DIM_API int32_t dim_refine_status(dim_ctx *ctx, int32_t B, int32_t n_iter, int32_t *status_host, void *stream);

/* Projective point-to-plane ICP against the observed depth: polishes B poses (typically dim_refine's last estimate) against
 * the depth sensor.  Not in the reference (its evaluation only reads ICP poses computed by another program); the contract
 * is oracle/icp.py, restated on the device in float64.  Per call the model surface is rendered once, at float32(pose_in),
 * by the refinement loop's rasteriser; each iteration associates every model pixel with the observed pixel it projects
 * to, builds the 6x6 point-to-plane normal equations of the inliers (|model depth - observed depth| < max_dist) and takes
 * one Gauss-Newton step.  The results are identical run to run (no atomics in any sum).
 *   depth_frames f32 [F,H,W] device, metres (0 = hole); frame_idx / F / K9_host / K_frames as dim_refine (a device index
 *   outside [0, F) means frame 0 and status bit 3; K_frames is read as given; K9_host must be a finite pinhole matrix).
 *   cls_idx i32[B], pose_in f64[B,3,4] device; 1 <= B, F <= max_batch; n_iter >= 1; max_dist > 0 (metres) also bounds the
 *   depth step between a model pixel and its neighbours (silhouette and self-occlusion edges); min_points >= 6.
 *   outputs (device): poses_out f64[n_iter,B,3,4] (the pose after each iteration), inliers i32[n_iter,B] and rms
 *   f32[n_iter,B] (sqrt(mean r^2) of the inliers, 0 without any), both measured before that iteration's update, and
 *   status i32[n_iter,B]: 0 = ok; bit 0 = no model pixel (empty render), bit 1 = bad class index, bit 3 = frame index out
 *   of range, bit 4 = fewer than min_points inliers or a singular system.  With bit 0 or 4 the pose is left unchanged.
 * Never reads the network: runs on every context variant.  A refused call enqueues nothing and leaves the outputs untouched.
 * The call overwrites the context's render scratch; refinement graphs captured before it replay unchanged after it.
 * With dim_profile_enable on, each call adds one record to dim_profile_read: ms4[0] = render, ms4[1] = association + solve. */
DIM_API int32_t dim_icp(dim_ctx *ctx, const float *depth_frames, int32_t F, const int32_t *frame_idx,
                        const float *K9_host, const float *K_frames, const int32_t *cls_idx,
                        const double *pose_in, int32_t B, int32_t n_iter, float znear, float zfar,
                        float max_dist, int32_t min_points, double *poses_out, int32_t *inliers,
                        float *rms, int32_t *status, void *stream);

/* The depth files' u16 values [F,H,W] (device) -> metres f32 [F,H,W] (device), as lib/utils/image.py:203,218 converts them:
 * float32(u16) / float32(depth_factor) (LINEMOD: 1000). */
DIM_API int32_t dim_depth_from_u16(dim_ctx *ctx, const uint16_t *depth_u16, int32_t F, float depth_factor,
                                   float *depth, void *stream);

/* Visible Surface Discrepancy (Hodan et al., "On Evaluation of 6D Object Pose Estimation", ECCVW 2016; the render-based
 * error of the reference's lib/utils/pose_error.py): per instance, the depth renders at float32(poses_est) and
 * float32(poses_gt) by the refinement loop's rasteriser, the distance images of them and of the observed depth
 * (lib/utils/misc.py depth_im_to_dist_im), the visibility masks V_gt and V_est (lib/utils/visibility.py, tolerance delta,
 * compared in float32), and for each tau the step cost e = (c_tau + |union| - |inter|) / |union|, c_tau = the pixels of
 * V_gt & V_est whose distances differ by >= tau; e = 1 when the union is empty.  The contract is oracle/vsd.py.  Every sum is
 * an integer count: the results are identical run to run and for any batch composition.
 *   depth_frames f32 [F,H,W] device, metres (0 = hole); frame_idx / F / K9_host / K_frames as dim_refine (a device index
 *   outside [0, F) means frame 0 and status bit 3; K9_host must be a finite pinhole matrix).
 *   cls_idx i32[B], poses_est / poses_gt f64[B,3,4] device; 1 <= B, F <= max_batch; delta > 0 (metres, finite);
 *   taus_host f64[n_tau] host, 1 <= n_tau <= 16, each > 0 and finite.
 *   outputs (device): err f64[B,n_tau]; status i32[B] (nullable): 0 = ok; bit 0 = empty union (e = 1), bit 1 = bad class
 *   index, bit 3 = frame index out of range.
 * Never reads the network: runs on every context variant.  A refused call enqueues nothing and leaves the outputs untouched.
 * The call overwrites the context's render scratch; refinement graphs captured before it replay unchanged after it.
 * With dim_profile_enable on, each call adds one record to dim_profile_read: ms4[0] = the two renders, ms4[1] = VSD pass. */
DIM_API int32_t dim_pose_error_vsd(dim_ctx *ctx, const float *depth_frames, int32_t F, const int32_t *frame_idx,
                                   const float *K9_host, const float *K_frames, const int32_t *cls_idx,
                                   const double *poses_est, const double *poses_gt, int32_t B, float znear, float zfar,
                                   float delta, const double *taus_host, int32_t n_tau, double *err, int32_t *status,
                                   void *stream);

/* BGR u8 HWC -> RGB-mean f32 CHW on device (lib/utils/image.py:583-594 transform). */
DIM_API int32_t dim_transform_image_u8(dim_ctx *ctx, const uint8_t *bgr_u8, int32_t B,
                                       const double *pixel_means_rgb_host, float *image,
                                       void *stream);

/* Train-time augmentation of the observed inputs (the shipped training config: LM6D_REFINE + LM6D_REFINE_SYN, MASK_DILATE).
 * The caller supplies every random draw (deepim_b200/augment.py draws them in the reference's order).
 *
 * Background bank: BGR u8 photos [h,w,3] of any size (h, w in [1, 16384]), uploaded once per context like meshes.
 *   Capacity: indices 0 .. DIM_BG_MAX-1; each dim_bg_upload allocates h*w*3 bytes of device memory, held until the context
 *   is destroyed; uploading to an index already used replaces its photo (frees the old one; synchronises the device).
 *   A photo whose resized crop (below) does not fit the context's H x W canvas is refused at upload.
 * dim_bg_geometry: host only, no context -- the crop and resize of image.py:108-145 + resize (image.py:552-572) in float64:
 *   out4 = crop_h, crop_w, dst_h, dst_w; *scale = cv2.resize's fx = fy.  The crop is the photo's top-left crop_h x crop_w
 *   (its H:W aspect), resized to dst_h x dst_w and placed at the canvas's top-left corner, black elsewhere.  A crop scaled
 *   by exactly 1/2 with an odd side is refused (cv2 takes its INTER_AREA border path there, not reproduced).
 * dim_replace_background (image.py:96-157): per instance b,
 *   composite[b] = mask[b] != 0 ? observed_bgr[b] : background;  image_observed[b] = transform(composite[b])
 *   with transform the float64 mean subtraction of dim_transform_image_u8.
 *   observed_bgr f32 [B,H,W,3] BGR in [0,255] as dim_render's out_bgr writes it: that is the observed image the device
 *     pipeline already has, so no conversion pass is needed; values are clamped to [0,255] and truncated to u8 as numpy's
 *     store into the reference's uint8 canvas does (dim_render's truncating renders are whole numbers already);
 *   mask f32 [B,1,H,W] (mask_gt_observed; != 0 keeps the observed pixel);
 *   bg_index_host HOST i32 [B]: bank index, or -1 = keep the observed image (image_observed = transform(observed));
 *   image_observed f32 [B,3,H,W] RGB - means; composite_u8 u8 [B,H,W,3] BGR (nullable).
 *   The bilinear resize is OpenCV 4.x INTER_LINEAR on 8-bit images, bit for bit (pinned against cv2 4.13; augment.cu).
 *   Refused: B outside [1, max_batch], an index >= 0 that names no uploaded photo (or any index >= 0 on an empty bank).
 * dim_mask_dilate (lib/utils/mask_dilate.py:19-47): mask_in / mask_out f32 [B,1,H,W]; draws DEVICE i32 [B,5] = direction,
 *   then the thickness of the down, up, right and left shift (<= 0: that side is skipped).  Each shift tests the ORIGINAL
 *   mask, so a box grows into a cross; nonzero inputs stay as they are except values > 1, which become 1.  In place
 *   (mask_in == mask_out) is refused. */
#define DIM_BG_MAX 65536
DIM_API int32_t dim_bg_upload(dim_ctx *ctx, int32_t idx, const uint8_t *bgr_u8_host, int32_t h, int32_t w);
DIM_API int32_t dim_bg_geometry(int32_t H, int32_t W, int32_t bh, int32_t bw, int32_t *out4, double *scale);
DIM_API int32_t dim_replace_background(dim_ctx *ctx, const float *observed_bgr, const float *mask,
                                       const int32_t *bg_index_host, int32_t B, const double *pixel_means_rgb_host,
                                       float *image_observed, uint8_t *composite_u8, void *stream);
DIM_API int32_t dim_mask_dilate(dim_ctx *ctx, const float *mask_in, const int32_t *draws, int32_t B, float *mask_out,
                                void *stream);

/* Test hooks (not part of the drop-in surface): copy the bf16 NHWC activation buffer feeding conv
 * layer idx (10 = fc6 input) to the host, and its geometry
 * out8 = rows, cols, C, py, px, Ho, Wo, Cout. */
DIM_API int32_t dim_debug_activation(dim_ctx *ctx, int32_t idx, int32_t lo, void *host_dst,
                                     uint64_t bytes);
DIM_API int32_t dim_debug_layer_geometry(dim_ctx *ctx, int32_t idx, int32_t *out8);
/* tuning hooks (not part of the drop-in surface).
 * dim_debug_set_option: run-time switch.  Key "graph": 1 (default) = replay the refinement chain as a CUDA graph,
 *   0 = enqueue it launch by launch.  Key "sms": the SM count the library sizes its launches for (the persistent conv
 *   grids, conv1's row runs, the training step's parity-class streams and weight-gradient K slices): 1 ... the device's
 *   count, or 0 = the device's count (the default); other values are refused.  It changes no device setting: the
 *   kernels simply run on fewer CTAs, which lets the tests exercise the schedules of smaller parts (H100 PCIe: 114 SMs).
 *   Every key drops the captured graphs; the "sms" key also the training step's cached launch descriptors.  Any other
 *   key is an error.
 * dim_debug_layer_profile: enable = 1 records CUDA events around each conv layer of every dim_net_fwd / dim_refine
 *   iteration; ms10 (nullable) receives the 10 layer times of the LAST forward pass; enable = 0 stops. */
DIM_API int32_t dim_debug_set_option(dim_ctx *ctx, const char *key, int32_t value);
DIM_API int32_t dim_debug_layer_profile(dim_ctx *ctx, int32_t enable, float *ms10);
/* dim_debug_graph_count: how many refinement chains this context holds captured as CUDA graphs (-1: NULL ctx). */
DIM_API int32_t dim_debug_graph_count(dim_ctx *ctx);

/* Stage profiling of dim_refine with CUDA events on the launching stream (used by bench.py for the
 * live roofline numbers).  enable=1 starts recording; dim_profile_read synchronises the device and
 * returns accumulated milliseconds since the last read as ms[4] = render, bbox+zoom, conv tower,
 * fc+head+compose, and the number of recorded iterations. */
DIM_API int32_t dim_profile_enable(dim_ctx *ctx, int32_t enable);
DIM_API int32_t dim_profile_read(dim_ctx *ctx, float *ms4, int32_t *iterations);

/* ADD / ADI pose error (lib/utils/pose_error.py:72-108; LM6D_REFINE.evaluate_pose_add l.418-424 picks ADI for the
 * symmetric classes): poses f64[M,3,4] (device), points f64[N,3] model points (device), err f64[M].
 * symmetric = 0: mean point distance; 1: mean distance from every GT-transformed point to the nearest
 * estimate-transformed point (brute force, float64). */
DIM_API int32_t dim_pose_error(dim_ctx *ctx, const double *poses_est, const double *poses_gt, int32_t M,
                               const double *points, int32_t N, int32_t symmetric, double *err,
                               void *stream);

/* Average 2D re-projection error and rotation / translation distances of pose pairs (float64, device pointers):
 * err3[m] = { arp_2d (pixels; lib/utils/pose_error.py:55-69), rotation distance in degrees, translation distance in metres
 * (lib/pair_matching/RT_transform.py:162-173 calc_rt_dist_m) } -- the inputs of LM6D_REFINE.evaluate_pose (5 cm 5 deg,
 * lib/dataset/LM6D_REFINE.py:278-371) and evaluate_pose_arp_2d (Proj. 2D, l.514-). K9_dev: 9 doubles on the device. */
DIM_API int32_t dim_pose_error_2d(dim_ctx *ctx, const double *poses_est, const double *poses_gt, int32_t M, const double *points,
                                  int32_t N, const double *K9_dev, double *err3, void *stream);

/* End-point error of a predicted flow (deepim/core/tester.py:573-589 calc_EPE_one_pair; the non-FAST_TEST evaluation):
 * flows [B,2,H,W], visible / bg [B,1,H,W] float32 device; out6 [B,6] float64 device =
 * { sum |gt - pred| over all pixels, pixel count, sum over visible == 1, sum(visible), sum over visible | bg, count }. */
DIM_API int32_t dim_flow_epe(dim_ctx *ctx, const float *flow_pred, const float *flow_gt, const float *visible, const float *bg,
                             int32_t B, double *out6, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Training step of the refiner network (train graph: deepim/symbols/deepIM_flownet.py:121-365 decoder,
 * flow / mask / point-matching losses; optimiser: deepim/train.py:296-304 SGD-momentum, one update per inner
 * iteration as deepim/core/module.py:1131-1137).  Replaces Module.forward_backward + Module.update for this
 * network; the zoom front of the train symbol (ZoomMask / ZoomImageWithFactor / ZoomFlow, symbol:391-489) is
 * the dim_zoom_* calls above, the inter-iteration batch update is dim_train_update.
 *
 * Parameters live in ONE flat fp32 vector in MXNet layouts: for each of the 22 trainable tensors in the order
 * returned by dim_train_param_info (flow_conv1 ... conv6_1, fc6, fc7, rot, trans, Convolution1, deconv5,
 * upsample_flow6to5, Convolution2, deconv4, upsample_flow5to4, Convolution3, mask_conv3) weight then bias,
 * followed by the frozen bilinear upsampling_weight (2,1,32,32) and mask_upsampling_weight (1,1,32,32):
 * 57 749 164 floats for the mask network; the RGB-D network's flow_conv1 (64, 10, 7, 7) adds 6 272, the image-only
 * network's (64, 6, 7, 7) removes 6 272, every other entry is the same.  One tensor is permuted: fc6_weight is stored
 * (256, h*10+w, c) -- the NHWC order of the conv6_1 activation it multiplies -- instead of MXNet's (256, c*80 + h*10 + w)
 * (the Python host permutes on load / get; element-wise consumers such as the all-reduce and SGD do not care).  Gradients
 * use the same layout (that is the buffer a data-parallel caller all-reduces with NCCL between dim_train_forward_backward
 * and dim_train_sgd_update; kvstore replacement, deepim/core/module.py:616-635).
 * dim_train_param_info needs no context: entry idx of the table of the network (input_depth, input_mask) as the Network
 * variants above; input_depth = 1 with input_mask = 0 is refused.  Non-zero past the last entry. */
DIM_API int32_t dim_train_create(dim_ctx *ctx, int32_t max_points);
DIM_API int64_t dim_train_param_count(dim_ctx *ctx);
DIM_API int32_t dim_train_param_info(int32_t input_depth, int32_t input_mask, int32_t idx, const char **name,
                                     int64_t *weight_numel, int64_t *bias_numel);
/* flat_host: host pointer.  Also (re)loads the inference network of this context. */
DIM_API int32_t dim_train_load_params(dim_ctx *ctx, const float *flat_host, int64_t n, void *stream);
/* which = 0: parameters, 1: momentum.  Synchronises the stream. */
DIM_API int32_t dim_train_get_params(dim_ctx *ctx, float *flat_host, int64_t n, int32_t which,
                                     void *stream);
/* Device pointers, fp32 NCHW: zoomed images (B,3,H,W), zoomed masks (B,1,H,W), zoom_factor (B,4), zoomed flow
 * label (B,2,H,W) and weights (B,2,H,W), zoomed GT mask (B,1,H,W), src_pose (B,3,4), point clouds (B,3,N).
 * RGB-D network: zoom_depth_observed / zoom_depth_rendered (B,1,H,W), metres (the train-time update's depth_rendered,
 * zoomed with the pair's zoom factor; deepIM_flownet.py:33-51, batch_updater l.269); conv1 has no data gradient, so only
 * flow_conv1_weight's gradient widens.  Depth and mask inputs are NULL as the network variant says.
 * Outputs: rot_est_norm (B,4) = L2Normalization(rot), trans_est (B,3) = invZoomTrans, flow_est (B,2,H,W)
 * (= flow_est_crop * NORMALIZE_FLOW, nullable), mask_prob (B,1,H,W) (nullable), losses4 = [sum flow_loss,
 * sum point_matching_loss, sum mask BCE, weighted objective], grads (flat, see above; NULL = forward only:
 * the non-FAST_TEST outputs of the test graph, symbol:624-713).
 * With grads == NULL the labels (zoom_flow ... point clouds, losses4) may all be NULL: pure test-time forward of
 * the full graph; rot_raw (B,4, nullable) is the un-normalised quaternion the test graph concatenates into se3.
 * bucket_events (nullable): n_buckets cudaEvent_t handles; event k is recorded (on an internal stream) as soon as
 * the gradients of every tensor with table index >= bucket_first_tensor[k] are complete, so a data-parallel
 * caller can start the NCCL all-reduce of that slice of `grads` while the rest of the backward pass still runs.
 * All work is joined back into `stream` before the call's stream order ends. */
DIM_API int32_t dim_train_forward_backward(
    dim_ctx *ctx, const float *zoom_image_observed, const float *zoom_image_rendered,
    const float *zoom_mask_observed, const float *zoom_mask_rendered, const float *zoom_factor,
    const float *zoom_flow, const float *zoom_flow_weights, const float *zoom_mask_gt_observed,
    const float *src_pose, const float *point_cloud_model, const float *point_cloud_weights,
    const float *point_cloud_observed, int32_t B, int32_t N, float *rot_est_norm, float *trans_est,
    float *flow_est, float *mask_prob, float *losses4, float *grads, float *rot_raw,
    void *const *bucket_events, const int32_t *bucket_first_tensor, int32_t n_buckets,
    const float *zoom_depth_observed, const float *zoom_depth_rendered, void *stream);
/* Loss weights / normalisers of the training step and the pose parameterisation shared with the refinement loop: the
 * values the reference reads from its yaml (experiments/deepim/cfgs/...: train.LW_FLOW / LW_MASK / LW_PM, NUM_3D_SAMPLE,
 * NORMALIZE_3D_POINT, NORMALIZE_FLOW, network.TRANS_MEANS / TRANS_STDS, ROT_COORD).  Defaults = the shipped LM6d config
 * (0.25, 0.03, 0.1, 3000, 0.1, 20, means 0, stds 1, CAMERA).  The MakeLoss grad_scale of the point-matching loss is
 * lw_pm / num_3d_sample whatever the number of points passed per call (deepIM_flownet.py:330-336).
 * dim_train_set_config applies to dim_train_forward_backward of this context; trans_means / trans_stds / rot_coord also
 * drive dim_refine / dim_refine_host_async (RT_transform with T_means / T_stds / rot_coord, tester.py:452-461) and may be set
 * without dim_train_create (the other fields are then stored and used once a training state exists). */
typedef struct dim_train_config {
  float lw_flow, lw_mask, lw_pm;
  float num_3d_sample;
  float normalize_3d_point;
  float normalize_flow;
  float trans_means[3], trans_stds[3];
  int32_t rot_coord; /* 0 = MODEL, 1 = CAMERA */
} dim_train_config;
DIM_API int32_t dim_train_set_config(dim_ctx *ctx, const dim_train_config *cfg);
DIM_API int32_t dim_train_get_config(dim_ctx *ctx, dim_train_config *cfg);
/* mom = momentum*mom - lr*(rescale_grad*grad + wd*w); w += mom  (wd on *_weight only; the two bilinear kernels
 * are frozen), then refreshes every bf16 operand pack of the context from the new master weights. */
DIM_API int32_t dim_train_sgd_update(dim_ctx *ctx, const float *grads, float lr, float momentum, float wd,
                                     float rescale_grad, void *stream);
/* Precision of this context's training step: DIM_PREC_BF16 (default; bf16 activations and activation gradients) or
 * DIM_PREC_BF16X3 (every activation, activation gradient and operand pack a bf16 hi / lo pair, three tensor-core passes:
 * gradients near the fp32 reference, about 2^-16 relative per stored value).  Gradients, master weights and momentum are
 * fp32 in both.  Applies to dim_train_forward_backward, with and without gradients, and to the operand refresh of
 * dim_train_sgd_update.  Any other value is refused (DIM_PREC_FP16 included).  Needs dim_train_create.  The first switch to
 * DIM_PREC_BF16X3 allocates the lo halves; every switch to it synchronises the device and refreshes them from the master
 * weights.  Switching back to DIM_PREC_BF16 leaves the bf16 step exactly as it was. */
DIM_API int32_t dim_train_set_precision(dim_ctx *ctx, int32_t precision);
DIM_API int32_t dim_train_get_precision(dim_ctx *ctx, int32_t *precision);
/* Test hooks: intermediates of the training step and their geometry out7 = Hp, Wp, py, px, C, H, W (ids in train.cu):
 * 0-9 the fp32 flow / mask maps, their gradients, h6 and dh6; 10-15 and 20-29 the bf16 decoder, gradient and gz buffers
 * (100 + one of these ids = its lo half after a DIM_PREC_BF16X3 step); 30-41 the fp32 pose heads and losses (h7, rot_raw,
 * ztrans, rot_n, trans_est, pts_est, dpts, drot_n, dtrans, drot, dh7, dfull), which have no lo half and zero geometry. */
DIM_API int32_t dim_train_debug_tensor(dim_ctx *ctx, int32_t id, void *host_dst, uint64_t bytes);
DIM_API int32_t dim_train_debug_geometry(dim_ctx *ctx, int32_t id, int32_t *out7);
/* Test hook: the K slicing of the 12 weight gradients (flow_conv1, conv2 ... conv6_1, deconv5, deconv4) of a B-image step
 * at the current SM count (dim_debug_set_option "sms") and precision: out36[3 g], [3 g + 1], [3 g + 2] = slices, pixel
 * blocks per slice (the K range one fp32 accumulator sums; 64 pixels a block), pixel blocks in all. */
DIM_API int32_t dim_train_debug_wgrad_slices(dim_ctx *ctx, int32_t B, int32_t *out36);
/* ms7 = device time of the phases of the last dim_train_forward_backward (with gradients) on the caller's stream:
 * encoder fwd, decoder fwd, losses + pose heads, fc/head backward, decoder backward, encoder data-gradient chain,
 * wait for the weight-gradient stream.  Synchronises the device. */
DIM_API int32_t dim_train_debug_phases(dim_ctx *ctx, float *ms7);

/* number of kernel launches issued by this library since the counter was last reset */
DIM_API int64_t dim_launch_count(int32_t reset);

#ifdef __cplusplus
}
#endif
#endif /* DEEPIM_B200_H_ */
