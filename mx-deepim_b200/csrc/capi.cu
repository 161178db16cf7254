// capi.cu -- the extern "C" surface declared in include/deepim_b200.h.
#include <stdarg.h>
#include <string.h>

#include <cmath>

#include "launch.cuh"

namespace dim {

static thread_local char g_err[1024] = "";
long long g_launches = 0;

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int prof_begin(dim_ctx *ctx, cudaStream_t st, cudaEvent_t **ev) {
  *ev = nullptr;
  if (!ctx->prof) return 0;
  while (ctx->prof_events.size() < ctx->prof_used + 5) {
    cudaEvent_t e;
    DIM_CHECK(cudaEventCreate(&e));
    ctx->prof_events.push_back(e);
  }
  *ev = &ctx->prof_events[ctx->prof_used];
  ctx->prof_used += 5;
  DIM_CHECK(cudaEventRecord((*ev)[0], st));
  return 0;
}

}  // namespace dim

using namespace dim;

// captured refinement graphs bake in launch dimensions and kernel choices: anything that changes them drops the graphs
static void drop_graphs(dim_ctx *ctx) {
  if (ctx->graphs.empty()) return;
  cudaDeviceSynchronize();
  for (auto &g : ctx->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
  ctx->graphs.clear();
}

extern "C" {

DIM_API int32_t dim_abi_version(void) { return DIM_ABI_VERSION; }
DIM_API const char *dim_last_error(void) { return g_err; }
DIM_API int64_t dim_launch_count(int32_t reset) {
  long long v = g_launches;
  if (reset) g_launches = 0;
  return v;
}

DIM_API int32_t dim_ctx_create(int32_t device, int32_t max_batch, int32_t H, int32_t W, int32_t max_classes,
                               int32_t max_verts, int32_t max_faces, dim_ctx **out) {
  DIM_REQUIRE(out != nullptr, "dim_ctx_create: out is NULL");
  DIM_REQUIRE(max_batch >= 1 && H >= 16 && W >= 16 && (W % 4) == 0, "dim_ctx_create: bad sizes");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    set_error("dim_ctx_create: no CUDA device available (%s); this library has no CPU fallback",
              cudaGetErrorString(e));
    return 10;
  }
  DIM_CHECK(cudaSetDevice(device));
  cudaDeviceProp prop;
  DIM_CHECK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("dim_ctx_create: device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major,
              prop.minor);
    return 11;
  }
  dim_ctx *ctx = new dim_ctx();
  ctx->device = device; ctx->max_batch = max_batch; ctx->H = H; ctx->W = W;
  ctx->max_classes = max_classes; ctx->max_verts = max_verts; ctx->max_faces = max_faces;
  ctx->num_sms = ctx->device_sms = prop.multiProcessorCount;
  const size_t P = (size_t)H * W, Bm = (size_t)max_batch;
  int rc = 0;
  rc |= dev_alloc(ctx, &ctx->meshes, (size_t)max_classes);
  rc |= dev_alloc(ctx, &ctx->pverts, Bm * (size_t)max_verts);
  rc |= dev_alloc(ctx, &ctx->vis, Bm * P);
  rc |= dev_alloc(ctx, &ctx->vbox, Bm * 4);
  rc |= dev_alloc(ctx, &ctx->bbox8, Bm * 8);
  rc |= dev_alloc(ctx, &ctx->cls_flag, Bm);
  rc |= dev_alloc(ctx, &ctx->status_hist, 8 * Bm);
  rc |= dev_alloc(ctx, &ctx->zoom_factor, Bm * 4);
  rc |= dev_alloc(ctx, &ctx->mask_rendered, Bm * P);
  rc |= dev_alloc(ctx, &ctx->bbox_ren, Bm * 4);
  rc |= dev_alloc(ctx, &ctx->pose_cur, Bm * 12);
  rc |= dev_alloc(ctx, &ctx->pose_cur_f32, Bm * 12);
  rc |= dev_alloc(ctx, &ctx->se3_cur, Bm * 7);
  rc |= dev_alloc(ctx, &ctx->ren4, Bm * P);
  rc |= dev_alloc(ctx, &ctx->obs4, Bm * P);
  rc |= dev_alloc(ctx, &ctx->image_observed_u8, Bm * 3 * P);
  rc |= dev_alloc(ctx, &ctx->cls_dev, Bm);
  rc |= dev_alloc(ctx, &ctx->frame_dev, Bm);
  rc |= dev_alloc(ctx, &ctx->K_dev, Bm * 9);
  rc |= dev_alloc(ctx, &ctx->poses_dev, 8 * Bm * 12);
  rc |= dev_alloc(ctx, &ctx->se3_hist_dev, 8 * Bm * 7);
  rc |= dev_alloc(ctx, &ctx->light_pos, Bm * 3);
  rc |= dev_alloc(ctx, &ctx->lit_intensity, 8 * Bm * 3);
  rc |= dev_alloc(ctx, &ctx->icp_partial, Bm * (size_t)cdiv(H, ICP_ROWS) * ICP_SLOT);
  rc |= dev_alloc(ctx, &ctx->vsd_partial, Bm * (size_t)cdiv(H, VSD_ROWS) * VSD_SLOT);
  rc |= dev_alloc(ctx, &ctx->vsd_box, Bm * 4);
  rc |= dev_alloc(ctx, &ctx->vsd_diam, Bm);
  rc |= dev_alloc(ctx, &ctx->sym_partial, Bm * SYM_SLOTS * 2);
  if (rc) { dim_ctx_destroy(ctx); return 12; }
  ctx->meshes_host.assign(max_classes, MeshDev{nullptr, nullptr, nullptr, nullptr, 0, 0, 0, 0, nullptr, nullptr});
  DIM_CHECK(cudaMemset(ctx->meshes, 0, sizeof(MeshDev) * max_classes));
  DIM_CHECK(cudaMemset(ctx->vis, 0xFF, sizeof(unsigned long long) * Bm * P));  // all pixels empty
  DIM_CHECK(cudaMemset(ctx->pverts, 0, sizeof(PVert) * Bm * max_verts));
  DIM_CHECK(cudaMemset(ctx->cls_flag, 0, sizeof(int) * Bm));
  DIM_CHECK(cudaMemset(ctx->status_hist, 0, sizeof(int) * 8 * Bm));
  if (net_create(ctx)) { dim_ctx_destroy(ctx); return 13; }
  DIM_CHECK(cudaDeviceSynchronize());
  *out = ctx;
  return 0;
}

DIM_API void dim_ctx_destroy(dim_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  train_destroy(ctx);
  net_destroy(ctx);
  for (auto &g : ctx->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
  for (cudaEvent_t e : ctx->prof_events) cudaEventDestroy(e);
  for (void *p : ctx->owned) cudaFree(p);
  for (auto &e : ctx->bg) if (e.data) cudaFree(e.data);
  delete ctx;
}

DIM_API int32_t dim_mesh_upload(dim_ctx *ctx, int32_t cls, const float *verts, const float *uvs, int32_t V,
                                const int32_t *faces, int32_t F, const uint8_t *tex, int32_t Th, int32_t Tw) {
  DIM_REQUIRE(ctx && cls >= 0 && cls < ctx->max_classes, "dim_mesh_upload: bad class index");
  DIM_REQUIRE(V > 0 && V <= ctx->max_verts && F > 0 && F <= ctx->max_faces, "dim_mesh_upload: mesh exceeds ctx limits");
  drop_graphs(ctx);  // the render launch grid follows the largest uploaded mesh
  for (int32_t i = 0; i < 3 * F; ++i) DIM_REQUIRE(faces[i] >= 0 && faces[i] < V, "dim_mesh_upload: face index out of range");
  MeshDev m;
  float *dv, *du; int *df; uint8_t *dt;
  if (dev_alloc(ctx, &dv, (size_t)3 * V) || dev_alloc(ctx, &du, (size_t)2 * V) || dev_alloc(ctx, &df, (size_t)3 * F) ||
      dev_alloc(ctx, &dt, (size_t)3 * Th * Tw))
    return 12;
  DIM_CHECK(cudaMemcpy(dv, verts, sizeof(float) * 3 * V, cudaMemcpyHostToDevice));
  DIM_CHECK(cudaMemcpy(du, uvs, sizeof(float) * 2 * V, cudaMemcpyHostToDevice));
  DIM_CHECK(cudaMemcpy(df, faces, sizeof(int) * 3 * F, cudaMemcpyHostToDevice));
  DIM_CHECK(cudaMemcpy(dt, tex, (size_t)3 * Th * Tw, cudaMemcpyHostToDevice));
  m.verts = dv; m.uvs = du; m.faces = df; m.tex = dt; m.V = V; m.F = F; m.Th = Th; m.Tw = Tw; m.normals = nullptr;
  m.colours = nullptr;
  ctx->meshes_host[cls] = m;
  DIM_CHECK(cudaMemcpy(ctx->meshes + cls, &m, sizeof(MeshDev), cudaMemcpyHostToDevice));
  return 0;
}

// vertex-coloured mesh: the fragment colour interpolates the winner triangle's vertex colours (raster.cu, fragment_colour).
// Every check runs before anything is allocated or changed, so a refused call leaves the class's previous mesh in place.
DIM_API int32_t dim_mesh_upload_colours(dim_ctx *ctx, int32_t cls, const float *verts, const float *colours, int32_t V,
                                        const int32_t *faces, int32_t F) {
  DIM_REQUIRE(ctx && cls >= 0 && cls < ctx->max_classes, "dim_mesh_upload_colours: bad class index");
  DIM_REQUIRE(verts && colours && faces, "dim_mesh_upload_colours: NULL argument");
  DIM_REQUIRE(V > 0 && V <= ctx->max_verts && F > 0 && F <= ctx->max_faces, "dim_mesh_upload_colours: mesh exceeds ctx limits");
  for (int32_t i = 0; i < 3 * F; ++i)
    DIM_REQUIRE(faces[i] >= 0 && faces[i] < V, "dim_mesh_upload_colours: face index out of range");
  std::vector<float4> c4((size_t)V);
  for (int32_t v = 0; v < V; ++v) {
    const float *c = colours + 3 * (size_t)v;
    for (int e = 0; e < 3; ++e)
      if (!(c[e] >= 0.f && c[e] <= 1.f)) {  // NaN fails both comparisons
        set_error("dim_mesh_upload_colours: the colour of vertex %d is not finite or lies outside [0, 1]", v);
        return 2;
      }
    c4[v] = make_float4(c[0], c[1], c[2], 0.f);
  }
  drop_graphs(ctx);  // the render launch grid follows the largest uploaded mesh
  MeshDev m{};
  float *dv; int *df; float4 *dc;
  if (dev_alloc(ctx, &dv, (size_t)3 * V) || dev_alloc(ctx, &df, (size_t)3 * F) || dev_alloc(ctx, &dc, (size_t)V)) return 12;
  DIM_CHECK(cudaMemcpy(dv, verts, sizeof(float) * 3 * V, cudaMemcpyHostToDevice));
  DIM_CHECK(cudaMemcpy(df, faces, sizeof(int) * 3 * F, cudaMemcpyHostToDevice));
  DIM_CHECK(cudaMemcpy(dc, c4.data(), sizeof(float4) * V, cudaMemcpyHostToDevice));
  m.verts = dv; m.faces = df; m.colours = dc; m.V = V; m.F = F;
  ctx->meshes_host[cls] = m;
  DIM_CHECK(cudaMemcpy(ctx->meshes + cls, &m, sizeof(MeshDev), cudaMemcpyHostToDevice));
  return 0;
}

DIM_API int32_t dim_render(dim_ctx *ctx, const int32_t *cls_idx, const float *pose, int32_t B, const float *K9,
                           float zn, float zf, const double *means, int32_t trunc_u8, float *out_image,
                           float *out_depth, float *out_mask, float *out_bgr, int32_t *out_bbox, void *stream) {
  DIM_REQUIRE(ctx && cls_idx && pose && K9, "dim_render: NULL argument");
  return render_launch(ctx, cls_idx, pose, B, zn, zf, means,
                       {.cams = frame_cams(K9), .out_image = out_image, .out_depth = out_depth, .out_mask = out_mask,
                        .out_bgr = out_bgr, .out_bbox = out_bbox, .trunc_u8 = trunc_u8},
                       (cudaStream_t)stream);
}

// lit renderer (lib/render_glumpy/render_py_light_modelnet_multi.py)
DIM_API int32_t dim_mesh_upload_normals(dim_ctx *ctx, int32_t cls, const float *normals, int32_t V) {
  DIM_REQUIRE(ctx && normals && cls >= 0 && cls < ctx->max_classes, "dim_mesh_upload_normals: bad argument");
  MeshDev &m = ctx->meshes_host[cls];
  DIM_REQUIRE(m.V > 0 && m.V == V, "dim_mesh_upload_normals: upload the mesh first; V must match");
  float *dn;
  if (dev_alloc(ctx, &dn, (size_t)3 * V)) return 12;
  DIM_CHECK(cudaMemcpy(dn, normals, sizeof(float) * 3 * V, cudaMemcpyHostToDevice));
  m.normals = dn;
  DIM_CHECK(cudaMemcpy(ctx->meshes + cls, &m, sizeof(MeshDev), cudaMemcpyHostToDevice));
  return 0;
}
// the lit renderer shades with per-vertex normals: every uploaded mesh must have them
static int normals_check(dim_ctx *ctx, const char *fn) {
  for (auto &m : ctx->meshes_host)
    if (m.V > 0 && m.normals == nullptr) {
      set_error("%s: a mesh has no normals (dim_mesh_upload_normals)", fn);
      return 2;
    }
  return 0;
}
// lighting of the loop / update entry points: NULL = unlit; else its intensities are given and every uploaded mesh has normals
static int lit_check(dim_ctx *ctx, const dim_lighting *lit, const char *fn) {
  if (!lit) return 0;
  if (!lit->intensity) {
    set_error("%s: NULL lighting->intensity", fn);
    return 2;
  }
  return normals_check(ctx, fn);
}
static LitParams lit_params(const float *light_pos, const float *intensity, float ratio) {
  return LitParams{light_pos, intensity, (float)(1.0 - (double)ratio), ratio};
}

// depth inputs are given exactly when the context's network is RGB-D: never run conv1 on the wrong channels.
// d1: the second depth of a pair (the single-depth entries pass d0 twice); args names them in the message.
static int depth_check(dim_ctx *ctx, const void *d0, const void *d1, const char *fn, const char *args) {
  const bool rgbd = net_input_depth(ctx);
  if (rgbd ? (d0 && d1) : (!d0 && !d1)) return 0;
  if (rgbd)
    set_error("%s: this context's network takes depth input (dim_ctx_set_input_depth): %s must not be NULL", fn, args);
  else
    set_error("%s: this context's network takes no depth input (dim_ctx_set_input_depth): pass %s = NULL", fn, args);
  return 2;
}

DIM_API int32_t dim_render_lit(dim_ctx *ctx, const int32_t *cls_idx, const float *pose, int32_t B, const float *K9, float zn,
                               float zf, const double *means, const float *light_pos, const float *light_int,
                               float brightness_ratio, float *out_image, float *out_depth, float *out_mask, float *out_bgr,
                               int32_t *out_bbox, void *stream) {
  DIM_REQUIRE(ctx && cls_idx && pose && K9 && light_pos && light_int, "dim_render_lit: NULL argument");
  if (int rc = normals_check(ctx, "dim_render_lit")) return rc;
  const LitParams lit = lit_params(light_pos, light_int, brightness_ratio);
  return render_launch(ctx, cls_idx, pose, B, zn, zf, means,
                       {.cams = frame_cams(K9), .out_image = out_image, .out_depth = out_depth, .out_mask = out_mask,
                        .out_bgr = out_bgr, .out_bbox = out_bbox, .trunc_u8 = 1, .lit = &lit},
                       (cudaStream_t)stream);
}

// data-preparation render (toolkit/LM6d_ds_1, ds_2, ds_4, LM6d_0): Render_Py_Light and Render_Py outputs of one pass
DIM_API int32_t dim_render_dataset(dim_ctx *ctx, const int32_t *cls_idx, const float *pose, int32_t B, const float *K9,
                                   float zn, float zf, float depth_factor, const float *light_position,
                                   const float *light_intensity, const float *brightness_ratio, uint8_t *lit_bgr,
                                   uint8_t *bgr, uint16_t *depth_u16, uint8_t *label, void *stream) {
  DIM_REQUIRE(ctx && cls_idx && pose && K9, "dim_render_dataset: NULL argument");
  const char *lit_args[3] = {"light_position", "light_intensity", "brightness_ratio"};
  const void *lit_ptrs[3] = {light_position, light_intensity, brightness_ratio};
  for (int k = 0; k < 3; ++k)
    if ((lit_ptrs[k] != nullptr) != (lit_bgr != nullptr)) {
      set_error(lit_bgr ? "dim_render_dataset: lit_bgr needs %s (NULL given)"
                        : "dim_render_dataset: %s is given but lit_bgr is NULL (the light is used only for lit_bgr)",
                lit_args[k]);
      return 2;
    }
  if (lit_bgr)
    if (int rc = normals_check(ctx, "dim_render_dataset")) return rc;
  const DatasetOut o{lit_bgr, bgr, depth_u16, label, brightness_ratio, depth_factor};
  return render_dataset_launch(ctx, cls_idx, pose, B, K9, zn, zf, light_position, light_intensity, o, (cudaStream_t)stream);
}

DIM_API int32_t dim_zoom_mask_fwd(dim_ctx *ctx, const float *mo, const float *mgt, const float *mr,
                                  const float *src_pose, int32_t B, const float *K9, float *zmo, float *zmgt,
                                  float *zmr, float *zoom_factor, int32_t *bbox, int32_t *status, void *stream) {
  DIM_REQUIRE(ctx && mo && mgt && mr && src_pose && K9 && zoom_factor, "dim_zoom_mask_fwd: NULL argument");
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch, "dim_zoom_mask_fwd: batch exceeds max_batch");
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = zoom_factor_launch(ctx, mgt, mr, 1, src_pose, B, K9, zoom_factor, bbox, status, st)) return rc;
  if (zmo) if (int rc = zoom_gather_launch(ctx, 1, mo, zmo, zoom_factor, B, 1, 0, nullptr, st)) return rc;
  if (zmgt) if (int rc = zoom_gather_launch(ctx, 1, mgt, zmgt, zoom_factor, B, 1, 0, nullptr, st)) return rc;
  // rendered mask is binarised at 0.2 before sampling (zoom_mask.py:39-42)
  if (zmr) if (int rc = zoom_gather_launch(ctx, 2, mr, zmr, zoom_factor, B, 1, 0, nullptr, st)) return rc;
  return 0;
}

DIM_API int32_t dim_zoom_image_with_factor_fwd(dim_ctx *ctx, const float *zoom_factor, const float *io,
                                               const float *ir, int32_t B, const float *means, float *zio,
                                               float *zir, void *stream) {
  DIM_REQUIRE(ctx && zoom_factor && io && ir && means && zio && zir, "dim_zoom_image_with_factor_fwd: NULL argument");
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch, "batch exceeds max_batch");
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = zoom_gather_launch(ctx, 3, io, zio, zoom_factor, B, 3, 0, means, st)) return rc;
  return zoom_gather_launch(ctx, 3, ir, zir, zoom_factor, B, 3, 0, means, st);
}

// ZoomImage (zoom_image.py:26-107): bbox from the images themselves (INPUT_MASK: False graphs)
DIM_API int32_t dim_zoom_image_fwd(dim_ctx *ctx, const float *io, const float *ir, const float *src_pose, int32_t B,
                                   const float *K9, const float *means, float *zio, float *zir, float *zoom_factor,
                                   int32_t *bbox, int32_t *status, void *stream) {
  DIM_REQUIRE(ctx && io && ir && src_pose && K9 && means && zio && zir && zoom_factor, "dim_zoom_image_fwd: NULL argument");
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch, "dim_zoom_image_fwd: batch exceeds max_batch");
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = zoom_factor_launch(ctx, io, ir, 3, src_pose, B, K9, zoom_factor, bbox, status, st, means)) return rc;
  if (int rc = zoom_gather_launch(ctx, 3, io, zio, zoom_factor, B, 3, 0, means, st)) return rc;
  return zoom_gather_launch(ctx, 3, ir, zir, zoom_factor, B, 3, 0, means, st);
}

DIM_API int32_t dim_group_picker(dim_ctx *ctx, const float *in, const float *group_idx, int32_t B, int32_t channels,
                                 int32_t group_num, int64_t elems_per_channel, int32_t backward, float *out, void *stream) {
  DIM_REQUIRE(ctx && in && group_idx && out, "dim_group_picker: NULL argument");
  DIM_REQUIRE(group_num >= 1 && channels % group_num == 0 && elems_per_channel >= 1, "dim_group_picker: channels must divide into groups");
  return group_pick_launch(in, group_idx, B, channels, group_num, (size_t)elems_per_channel, out, backward, (cudaStream_t)stream);
}

DIM_API int32_t dim_zoom_mask_with_factor_fwd(dim_ctx *ctx, const float *zoom_factor, const float *mask, int32_t B,
                                              int32_t inv, float *out, void *stream) {
  DIM_REQUIRE(ctx && zoom_factor && mask && out, "dim_zoom_mask_with_factor_fwd: NULL argument");
  return zoom_gather_launch(ctx, 2, mask, out, zoom_factor, B, 1, inv, nullptr, (cudaStream_t)stream);
}

DIM_API int32_t dim_zoom_flow_fwd(dim_ctx *ctx, const float *zoom_factor, const float *flow, const float *fw,
                                  int32_t fw_channels, int32_t B, int32_t inv, float *zflow, float *zfw, void *stream) {
  DIM_REQUIRE(ctx && zoom_factor && flow && zflow, "dim_zoom_flow_fwd: NULL argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = zoom_gather_launch(ctx, inv ? 4 : 6, flow, zflow, zoom_factor, B, 2, inv, nullptr, st)) return rc;
  if (!inv && fw && zfw) {
    DIM_REQUIRE(fw_channels == 1 || fw_channels == 2, "dim_zoom_flow_fwd: flow_weights has 1 or 2 channels");
    return zoom_gather_launch(ctx, 5, fw, zfw, zoom_factor, B, fw_channels, 0, nullptr, st);
  }
  return 0;
}

DIM_API int32_t dim_zoom_depth_fwd(dim_ctx *ctx, const float *zoom_factor, const float *dobs, const float *dren,
                                   int32_t B, float *zobs, float *zren, void *stream) {
  DIM_REQUIRE(ctx && zoom_factor && dobs && dren && zobs && zren, "dim_zoom_depth_fwd: NULL argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = zoom_gather_launch(ctx, 0, dobs, zobs, zoom_factor, B, 1, 0, nullptr, st)) return rc;
  return zoom_gather_launch(ctx, 0, dren, zren, zoom_factor, B, 1, 0, nullptr, st);
}

DIM_API int32_t dim_zoom_trans_fwd(dim_ctx *ctx, const float *zoom_factor, const float *trans, int32_t B, int32_t inv,
                                   float *out, void *stream) {
  DIM_REQUIRE(ctx && zoom_factor && trans && out, "dim_zoom_trans_fwd: NULL argument");
  return zoom_trans_launch(zoom_factor, trans, B, inv ? 1 : 0, 1, out, (cudaStream_t)stream);
}
DIM_API int32_t dim_zoom_trans_bwd(dim_ctx *ctx, const float *zoom_factor, const float *og, int32_t B, int32_t inv,
                                   int32_t zoom_grad, float *out, void *stream) {
  DIM_REQUIRE(ctx && zoom_factor && og && out, "dim_zoom_trans_bwd: NULL argument");
  return zoom_trans_launch(zoom_factor, og, B, inv ? 1 : 0, zoom_grad ? 1 : 0, out, (cudaStream_t)stream);
}

DIM_API int32_t dim_update_mask_box(dim_ctx *ctx, const int32_t *bbox, int32_t B, float *mask, void *stream) {
  DIM_REQUIRE(ctx && bbox && mask, "dim_update_mask_box: NULL argument");
  return box_mask_launch(ctx, bbox, B, mask, (cudaStream_t)stream);
}

DIM_API int32_t dim_se3_compose(dim_ctx *ctx, const double *pose_src, const float *se3, int32_t B, const double *Tm,
                                const double *Ts, int32_t rot_coord, double *pose_out, void *stream) {
  DIM_REQUIRE(ctx && pose_src && se3 && Tm && Ts && pose_out, "dim_se3_compose: NULL argument");
  DIM_REQUIRE(rot_coord >= 0 && rot_coord <= 2, "dim_se3_compose: unknown rot_coord");
  return se3_compose_launch(pose_src, se3, B, Tm, Ts, rot_coord, pose_out, nullptr, (cudaStream_t)stream);
}

DIM_API int32_t dim_flow_fwd(dim_ctx *ctx, const float *ds, const float *dt, const float *KT, const float *Kinv,
                             int32_t B, float *flow, float *valid, void *stream) {
  DIM_REQUIRE(ctx && ds && dt && KT && Kinv && flow && valid, "dim_flow_fwd: NULL argument");
  return flow_launch(ctx, ds, dt, KT, Kinv, B, flow, valid, nullptr, (cudaStream_t)stream);
}

DIM_API int32_t dim_transform3d_fwd(dim_ctx *ctx, const float *pc, const float *rot, const float *tr,
                                    const float *ps, int32_t B, int32_t N, const float *Tm, const float *Ts,
                                    int32_t rot_coord, float *out, void *stream) {
  DIM_REQUIRE(ctx && pc && rot && tr && ps && Tm && Ts && out, "dim_transform3d_fwd: NULL argument");
  return transform3d_fwd_launch(pc, rot, tr, ps, B, N, Tm, Ts, rot_coord, out, (cudaStream_t)stream);
}
DIM_API int32_t dim_transform3d_bwd(dim_ctx *ctx, const float *og, const float *pc, const float *rot, const float *tr,
                                    const float *ps, int32_t B, int32_t N, const float *Tm, const float *Ts,
                                    int32_t rot_coord, float *rg, float *tg, void *stream) {
  DIM_REQUIRE(ctx && og && pc && rot && tr && ps && Tm && Ts && rg && tg, "dim_transform3d_bwd: NULL argument");
  return transform3d_bwd_launch(og, pc, rot, tr, ps, B, N, Tm, Ts, rot_coord, rg, tg, (cudaStream_t)stream);
}

DIM_API int32_t dim_ctx_set_input_depth(dim_ctx *ctx, int32_t enable) {
  DIM_REQUIRE(ctx != nullptr, "dim_ctx_set_input_depth: NULL context");
  if (net_input_depth(ctx) == (enable != 0)) return 0;
  DIM_REQUIRE(train_param_count(ctx) == 0, "dim_ctx_set_input_depth: call it before dim_train_create (this context trains)");
  DIM_REQUIRE(net_input_mask(ctx), "dim_ctx_set_input_depth: input_depth with input_mask = 0 (depth input without the mask "
                                   "channels, INPUT_DEPTH without INPUT_MASK) is not supported");
  drop_graphs(ctx);
  if (enable && !ctx->depth_u16)
    if (dev_alloc(ctx, &ctx->depth_u16, (size_t)ctx->max_batch * ctx->H * ctx->W)) return 12;
  return net_set_input_depth(ctx, enable != 0);
}

DIM_API int32_t dim_ctx_set_input_mask(dim_ctx *ctx, int32_t enable) {
  DIM_REQUIRE(ctx != nullptr, "dim_ctx_set_input_mask: NULL context");
  if (net_input_mask(ctx) == (enable != 0)) return 0;
  DIM_REQUIRE(train_param_count(ctx) == 0, "dim_ctx_set_input_mask: call it before dim_train_create (this context trains)");
  DIM_REQUIRE(!net_input_depth(ctx), "dim_ctx_set_input_mask: input_mask = 0 with input_depth (depth input without the mask "
                                     "channels, INPUT_DEPTH without INPUT_MASK) is not supported");
  drop_graphs(ctx);
  if (!enable && !ctx->bbox_obs)
    if (dev_alloc(ctx, &ctx->bbox_obs, (size_t)ctx->max_batch * 4)) return 12;
  return net_set_input_mask(ctx, enable != 0);
}

DIM_API int32_t dim_net_load(dim_ctx *ctx, const float *const *W, const float *const *Bv) {
  DIM_REQUIRE(ctx && W && Bv, "dim_net_load: NULL argument");
  drop_graphs(ctx);
  return net_load(ctx, W, Bv);
}

DIM_API int32_t dim_net_fwd(dim_ctx *ctx, const float *zio, const float *zir, const float *zdo, const float *zdr,
                            const float *zmo, const float *zmr, int32_t B, int32_t precision, float *rot, float *trans,
                            void *stream) {
  DIM_REQUIRE(ctx && zio && zir && rot && trans, "dim_net_fwd: NULL argument");
  if (int rc = depth_check(ctx, zdo, zdr, "dim_net_fwd", "zoom_depth_observed / zoom_depth_rendered")) return rc;
  if (net_input_mask(ctx)) {
    DIM_REQUIRE(zmo && zmr, "dim_net_fwd: NULL argument");
  } else {
    DIM_REQUIRE(!zmo && !zmr, "dim_net_fwd: this context's network takes no mask input (dim_ctx_set_input_mask): pass "
                              "zoom_mask_observed = zoom_mask_rendered = NULL");
  }
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch, "dim_net_fwd: batch exceeds max_batch");
  cudaStream_t st = (cudaStream_t)stream;
  int rows, cols, pad; __nv_bfloat16 *hi, *lo;
  net_input_geometry(ctx, &rows, &cols, &pad, &hi, &lo);
  __nv_bfloat16 *lo_or_null = precision == DIM_PREC_BF16X3 ? lo : nullptr;
  const int f16 = precision == DIM_PREC_FP16;
  if (int rc = zdo ? pack_nhwc10_launch(ctx, zio, zir, zdo, zdr, zmo, zmr, B, rows, cols, pad, hi, lo_or_null, st, f16)
                   : pack_nhwc8_launch(ctx, zio, zir, zmo, zmr, B, rows, cols, pad, hi, lo_or_null, st, f16))
    return rc;
  return net_forward(ctx, B, precision, nullptr, rot, trans, nullptr, st, nullptr);
}

DIM_API int32_t dim_transform_image_u8(dim_ctx *ctx, const uint8_t *bgr, int32_t B, const double *means, float *image,
                                       void *stream) {
  DIM_REQUIRE(ctx && bgr && means && image, "dim_transform_image_u8: NULL argument");
  return transform_u8_launch(ctx, bgr, B, means, image, (cudaStream_t)stream);
}

// train-time augmentation of the observed inputs (augment.cu)
DIM_API int32_t dim_bg_upload(dim_ctx *ctx, int32_t idx, const uint8_t *bgr, int32_t h, int32_t w) {
  DIM_REQUIRE(ctx && bgr, "dim_bg_upload: NULL argument");
  DIM_REQUIRE(idx >= 0 && idx < DIM_BG_MAX, "dim_bg_upload: bank index outside [0, DIM_BG_MAX)");
  DIM_REQUIRE(h >= 1 && w >= 1 && h <= 16384 && w <= 16384, "dim_bg_upload: image size outside [1, 16384]");
  BgGeom g;
  if (int rc = bg_geometry(ctx->H, ctx->W, h, w, &g)) return rc;
  if ((size_t)idx >= ctx->bg.size()) ctx->bg.resize(idx + 1);
  dim_ctx::BgImage &e = ctx->bg[idx];
  if (e.data) {  // replacing a photo: cudaFree waits for the device, so no enqueued replacement still reads it
    DIM_CHECK(cudaFree(e.data));
    e = dim_ctx::BgImage();
  }
  uint8_t *d = nullptr;
  DIM_CHECK(cudaMalloc(&d, (size_t)h * w * 3));
  e.data = d; e.h = h; e.w = w;
  DIM_CHECK(cudaMemcpy(d, bgr, (size_t)h * w * 3, cudaMemcpyHostToDevice));
  return 0;
}

DIM_API int32_t dim_bg_geometry(int32_t H, int32_t W, int32_t bh, int32_t bw, int32_t *out4, double *scale) {
  DIM_REQUIRE(out4 && scale, "dim_bg_geometry: NULL argument");
  DIM_REQUIRE(H >= 1 && W >= 1 && bh >= 1 && bw >= 1, "dim_bg_geometry: bad sizes");
  BgGeom g;
  if (int rc = bg_geometry(H, W, bh, bw, &g)) return rc;
  out4[0] = g.crop_h; out4[1] = g.crop_w; out4[2] = g.dst_h; out4[3] = g.dst_w;
  *scale = g.scale;
  return 0;
}

DIM_API int32_t dim_replace_background(dim_ctx *ctx, const float *observed_bgr, const float *mask,
                                       const int32_t *bg_index_host, int32_t B, const double *means,
                                       float *image_observed, uint8_t *composite_u8, void *stream) {
  DIM_REQUIRE(ctx && observed_bgr && mask && bg_index_host && means && image_observed,
              "dim_replace_background: NULL argument");
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch, "dim_replace_background: B outside [1, max_batch]");
  BgLaunch L;
  memset(&L, 0, sizeof(L));
  for (int k = 0; k < 3; ++k) L.mean[k] = means[k];
  for (int b0 = 0; b0 < B; b0 += BG_LAUNCH_MAX) {  // validate every index before the first launch
    const int nb = B - b0 < BG_LAUNCH_MAX ? B - b0 : BG_LAUNCH_MAX;
    for (int i = 0; i < nb; ++i) {
      const int idx = bg_index_host[b0 + i];
      if (idx < 0) continue;
      if (ctx->bg.empty()) {
        set_error("dim_replace_background: instance %d names photo %d but the background bank is empty", b0 + i, idx);
        return 2;
      }
      if ((size_t)idx >= ctx->bg.size() || !ctx->bg[idx].data) {
        set_error("dim_replace_background: instance %d names photo %d, which was not uploaded", b0 + i, idx);
        return 2;
      }
      BgGeom g;
      if (int rc = bg_geometry(ctx->H, ctx->W, ctx->bg[idx].h, ctx->bg[idx].w, &g)) return rc;
    }
  }
  for (int b0 = 0; b0 < B; b0 += BG_LAUNCH_MAX) {
    const int nb = B - b0 < BG_LAUNCH_MAX ? B - b0 : BG_LAUNCH_MAX;
    L.b0 = b0;
    for (int i = 0; i < nb; ++i) {
      BgInst &in = L.inst[i];
      in = BgInst{};
      const int idx = bg_index_host[b0 + i];
      if (idx < 0) continue;
      const dim_ctx::BgImage &e = ctx->bg[idx];
      BgGeom g;
      bg_geometry(ctx->H, ctx->W, e.h, e.w, &g);
      in.data = e.data; in.inv_scale = 1.0 / g.scale; in.stride = e.w;
      in.crop_h = g.crop_h; in.crop_w = g.crop_w; in.dst_h = g.dst_h; in.dst_w = g.dst_w;
    }
    if (int rc = replace_bg_launch(ctx, L, nb, observed_bgr, mask, image_observed, composite_u8, (cudaStream_t)stream))
      return rc;
  }
  return 0;
}

DIM_API int32_t dim_mask_dilate(dim_ctx *ctx, const float *mask_in, const int32_t *draws, int32_t B, float *mask_out,
                                void *stream) {
  DIM_REQUIRE(ctx && mask_in && draws && mask_out, "dim_mask_dilate: NULL argument");
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch, "dim_mask_dilate: B outside [1, max_batch]");
  DIM_REQUIRE(mask_in != mask_out, "dim_mask_dilate: in place (mask_in == mask_out) is not supported");
  return mask_dilate_launch(ctx, mask_in, draws, B, mask_out, (cudaStream_t)stream);
}

static int refine_core(dim_ctx *ctx, const RefineArgs &a, cudaStream_t st) {
  const double Tm[3] = {ctx->cfg.trans_means[0], ctx->cfg.trans_means[1], ctx->cfg.trans_means[2]};
  const double Ts[3] = {ctx->cfg.trans_stds[0], ctx->cfg.trans_stds[1], ctx->cfg.trans_stds[2]};
  const float means_f[3] = {(float)a.means[0], (float)a.means[1], (float)a.means[2]};
  int rows, cols, pad; __nv_bfloat16 *hi, *lo;
  net_input_geometry(ctx, &rows, &cols, &pad, &hi, &lo);
  const bool depth = net_input_depth(ctx);  // RGB-D network: ren4.w = depth, obs4.w = depth_observed
  // image-only network (ZoomImage): both boxes come from the colours; the observed one once per call and frame
  const bool mask = net_input_mask(ctx);
  if (!mask)
    if (int rc = obs_colour_box_launch(ctx, a.obs4, a.cams.n_frames, ctx->bbox_obs, st)) return rc;
  const double *pose_src = a.pose_init;
  for (int it = 0; it < a.n_iter; ++it) {
    DimNvtxRange r_it("dim_refine iteration");
    cudaEvent_t *ev;
    if (int rc = prof_begin(ctx, st, &ev)) return rc;
    if (a.pose_override) pose_src = a.pose_override + (size_t)it * a.B * 12;
    // src_pose blob is float32 (nd.array), the host pose stays float64 (tester.py:391); the lit chain also derives the
    // light of this iteration's render from the float64 pose
    if (a.lit) {
      if (int rc = pose_light_launch(pose_src, ctx->pose_cur_f32, ctx->light_pos, a.B, a.offset, st)) return rc;
    } else if (int rc = f64_to_f32_launch(pose_src, ctx->pose_cur_f32, a.B * 12, st)) {
      return rc;
    }
    // render at the current pose (tester.py:427-442) straight into the pixel-interleaved
    // (R,G,B,mask) image the zoom kernel samples; mask_observed := box(mask_rendered) is analytic
    {
      DimNvtxRange r("render");
      const LitParams lp = a.lit ? lit_params(ctx->light_pos, a.intensity + (size_t)it * a.B * 3, a.brightness_ratio)
                                 : LitParams{nullptr, nullptr, 0.f, 0.f};
      if (int rc = render_launch(ctx, a.cls_idx, ctx->pose_cur_f32, a.B, a.zn, a.zf, a.means,
                                 {.cams = a.cams, .out_ren4 = ctx->ren4, .trunc_u8 = 1, .lit = a.lit ? &lp : nullptr,
                                  .ren4_depth = depth, .colour_box = !mask},
                                 st))
        return rc;
    }
    if (ev) DIM_CHECK(cudaEventRecord(ev[1], st));
    float *zf_it = a.zoom_factor ? a.zoom_factor + (size_t)it * a.B * 4 : ctx->zoom_factor;
    int *bbox_it = a.bbox ? a.bbox + (size_t)it * a.B * 8 : nullptr;
    // per-iteration status (bit 0: rendered / observed mask empty -> fallback zoom factor; bit 1: bad class index;
    // image-only network: bit 0 = observed image empty, bit 2 = rendered image empty -> zoom centred on the observed box;
    // bit 3: frame index out of range -> frame 0 observed)
    {
      DimNvtxRange r("bbox + zoom");
      int *status_it = ctx->status_hist + (size_t)(it < 8 ? it : 7) * a.B;
      if (mask) {
        if (int rc = zoom_factor_from_ren_launch(ctx, ctx->bbox_ren, ctx->pose_cur_f32, a.B, a.cams, zf_it, bbox_it, status_it,
                                                 st))
          return rc;
      } else if (int rc = zoom_factor_from_boxes_launch(ctx, ctx->bbox_obs, ctx->bbox_ren, ctx->pose_cur_f32, a.B, a.cams,
                                                        zf_it, bbox_it, status_it, st)) {
        return rc;
      }
      if (int rc = zoom_fused_launch(ctx, a.obs4, ctx->ren4, zf_it, means_f, a.B, rows, cols, pad, hi,
                                     a.precision == DIM_PREC_BF16X3 ? lo : nullptr, st, a.precision == DIM_PREC_FP16, a.means,
                                     depth, mask, a.cams))
        return rc;
    }
    if (ev) DIM_CHECK(cudaEventRecord(ev[2], st));
    float *se3_it = a.se3 ? a.se3 + (size_t)it * a.B * 7 : ctx->se3_cur;
    {
      DimNvtxRange r("FlowNetS tower + heads");
      if (int rc = net_forward(ctx, a.B, a.precision, zf_it, nullptr, nullptr, se3_it, st, ev ? ev[3] : nullptr)) return rc;
    }
    double *pose_out = a.poses + (size_t)it * a.B * 12;
    {
      DimNvtxRange r("SE(3) compose");
      if (int rc = se3_compose_launch(pose_src, se3_it, a.B, Tm, Ts, ctx->cfg.rot_coord, pose_out, nullptr, st)) return rc;
    }
    if (ev) DIM_CHECK(cudaEventRecord(ev[4], st));
    pose_src = pose_out;
  }
  return 0;
}

// The 4-iteration chain is ~90 kernel launches whose arguments do not change from call to call when the caller reuses
// its buffers (PoseRefiner does; so does bench.py).  After one eager run of an argument set the chain is captured into a
// CUDA graph (stream capture, thread-local mode) and replayed with one cudaGraphLaunch: the data-dependent parts of the
// loop are already branch-free on the device.  Disabled while stage / layer profiling is on or the context trains.
static int refine_graphed(dim_ctx *ctx, const RefineArgs &a, cudaStream_t st) {
  // the legacy default stream (and the per-thread default stream handle) cannot be captured
  const bool capturable = st != nullptr && st != cudaStreamLegacy && st != cudaStreamPerThread;
  if (!ctx->use_graph || ctx->prof || !capturable || !net_graph_safe(ctx)) return refine_core(ctx, a, st);
  dim_ctx::RefineGraph *g = nullptr;
  for (auto &e : ctx->graphs)
    if (memcmp(&e.key, &a, sizeof(RefineArgs)) == 0) { g = &e; break; }
  if (g && g->exec) {
    DIM_CHECK(cudaGraphLaunch(g->exec, st));
    g_launches += g->kernels;
    return 0;
  }
  if (!g) {  // first sight of this argument set: eager run (also builds tensor maps, sets function attributes)
    if (ctx->graphs.size() >= 32) ctx->graphs.erase(ctx->graphs.begin());
    ctx->graphs.push_back(dim_ctx::RefineGraph{a, nullptr, 0});
    return refine_core(ctx, a, st);
  }
  const long long before = g_launches;
  DIM_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  const int rc = refine_core(ctx, a, st);
  cudaGraph_t graph = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(st, &graph);
  if (rc != 0 || ce != cudaSuccess || graph == nullptr) {
    if (graph) cudaGraphDestroy(graph);
    if (rc == 0) set_error("dim_refine: stream capture failed: %s", cudaGetErrorString(ce));
    cudaGetLastError();
    return rc ? rc : 1;
  }
  const long long kernels = g_launches - before;
  g_launches = before;
  cudaGraphExec_t exec = nullptr;
  const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ie != cudaSuccess) { set_error("dim_refine: cudaGraphInstantiate failed: %s", cudaGetErrorString(ie)); return 1; }
  g->exec = exec;
  g->kernels = kernels;
  DIM_CHECK(cudaGraphLaunch(exec, st));
  g_launches += kernels;
  return 0;
}

// the loop's host values; the caller sets the pointers (lit: nullptr = unlit)
static RefineArgs refine_args(int32_t B, int32_t n_iter, const FrameCams &cams, float zn, float zf, const double *means,
                              int32_t precision, const dim_lighting *lit) {
  RefineArgs a{};
  a.B = B; a.n_iter = n_iter; a.precision = precision; a.zn = zn; a.zf = zf;
  a.cams = cams;
  memcpy(a.means, means, sizeof(a.means));
  if (lit) {
    a.lit = 1;
    a.intensity = lit->intensity;
    memcpy(a.offset, lit->offset, sizeof(a.offset));
    a.brightness_ratio = lit->brightness_ratio;
  }
  return a;
}

static int refuse(const char *fn, const char *msg) {
  set_error("%s: %s", fn, msg);
  return 2;
}

// the frame batch of every entry that works against observed frames: exactly one of K9_host and the per-frame cameras
// (K_frames_arg names them), B and F in [1, max_batch], and F == B without a frame map (instance b then observes frame b)
static int frames_check(dim_ctx *ctx, const char *fn, const float *K9_host, const void *K_frames, const char *K_frames_arg,
                        int32_t B, int32_t F, const int32_t *frame_idx) {
  if (!K9_host == !K_frames) {
    set_error("%s: exactly one of K9_host and %s must be non-NULL", fn, K_frames_arg);
    return 2;
  }
  if (B < 1 || B > ctx->max_batch) return refuse(fn, "batch exceeds max_batch");
  if (F < 1 || F > ctx->max_batch) return refuse(fn, "frame count F outside [1, max_batch]");
  if (!frame_idx && F != B) return refuse(fn, "frame_idx is NULL (instance b observes frame b): F must equal B");
  return 0;
}

// why the host intrinsics K (row-major 3x3) are not a finite pinhole matrix [[fx, 0, cx], [0, fy, cy], [0, 0, 1]] with
// fx, fy > 0, or nullptr when they are
static const char *pinhole_defect(const float *K) {
  for (int k = 0; k < 9; ++k)
    if (!std::isfinite(K[k])) return "a value is not finite";
  if (!(K[0] > 0.f && K[4] > 0.f)) return "fx and fy must be > 0";
  if (K[1] != 0.f || K[3] != 0.f) return "K[0][1] (skew) and K[1][0] must be 0";
  if (K[6] != 0.f || K[7] != 0.f || K[8] != 1.f) return "the last row must be (0, 0, 1)";
  return nullptr;
}

// K9_host, when given, is a finite pinhole matrix
static int pinhole_check(const char *fn, const float *K9_host) {
  if (K9_host)
    if (const char *why = pinhole_defect(K9_host)) {
      set_error("%s: K9_host is not a finite pinhole matrix [[fx,0,cx],[0,fy,cy],[0,0,1]]: %s", fn, why);
      return 2;
    }
  return 0;
}

// the argument checks both loop entries share; fn names the entry in every message.  host: dim_refine_host_async (its
// argument names, n_iter <= 8).
static int refine_check(dim_ctx *ctx, const char *fn, bool host, const void *frames, int32_t F, const int32_t *frame_idx,
                        const float *K9, const float *K_frames, const int32_t *cls_idx, const double *pose_init, int32_t B,
                        int32_t n_iter, const double *means, const void *poses, const void *depth,
                        const dim_lighting *lighting) {
  if (!(ctx && frames && cls_idx && pose_init && means && poses)) return refuse(fn, "NULL argument");
  if (int rc = frames_check(ctx, fn, K9, K_frames, host ? "K_frames_host" : "K_frames", B, F, frame_idx)) return rc;
  if (int rc = depth_check(ctx, depth, depth, fn, host ? "depth_frames_u16_host" : "depth_frames")) return rc;
  if (int rc = lit_check(ctx, lighting, fn)) return rc;
  if (host ? (n_iter < 1 || n_iter > 8) : n_iter < 1)
    return refuse(fn, host ? "n_iter must be in [1,8]" : "n_iter must be >= 1");
  return 0;
}

DIM_API int32_t dim_refine(dim_ctx *ctx, const float *image_frames, int32_t F, const int32_t *frame_idx, const float *K9,
                           const float *K_frames, const int32_t *cls_idx, const double *pose_init, int32_t B, int32_t n_iter,
                           float zn, float zf, const double *means, int32_t precision, const double *pose_override,
                           double *poses, float *se3, float *zoom_factor, int32_t *bbox, const float *depth_frames,
                           const dim_lighting *lighting, void *stream) {
  if (int rc = refine_check(ctx, "dim_refine", false, image_frames, F, frame_idx, K9, K_frames, cls_idx, pose_init, B, n_iter,
                            means, poses, depth_frames, lighting))
    return rc;
  cudaStream_t st = (cudaStream_t)stream;
  RefineArgs a = refine_args(B, n_iter, frame_cams(K9, K_frames, frame_idx, F), zn, zf, means, precision, lighting);
  a.obs4 = ctx->obs4; a.cls_idx = cls_idx; a.pose_init = pose_init; a.pose_override = pose_override;
  a.poses = poses; a.se3 = se3; a.zoom_factor = zoom_factor; a.bbox = bbox;
  // the F observed frames (and their depths) are packed into obs4 outside the graph.  The graph never reads the depth, so
  // a replay is correct whatever the key holds; keying on it only costs one capture per distinct depth buffer
  a.depth_observed = depth_frames;
  if (int rc = pack_obs4_launch(ctx, image_frames, F, ctx->obs4, a.means, st)) return rc;
  if (depth_frames)
    if (int rc = obs4_depth_launch(ctx, ctx->obs4, F, depth_frames, nullptr, 0.f, st)) return rc;
  return refine_graphed(ctx, a, st);
}

// dim_refine_host_async once its scalar arguments are checked: the class and frame indices (and intrinsics) are checked
// here, before anything is enqueued.  frame_host nullptr = instance b observes frame b (F == B).  K_host: nullptr = K9 for
// every instance; else host [F,9], one camera per frame (K9 nullptr)
static int refine_host_enqueue(dim_ctx *ctx, const char *fn, const uint8_t *frames_u8, int32_t F, const int32_t *frame_host,
                               const float *K_host, const int32_t *cls_host, const double *pose_host, int32_t B,
                               int32_t n_iter, const float *K9, float zn, float zf, const double *means, int32_t precision,
                               double *poses_out, float *se3_out, const uint16_t *depth_u16, float depth_factor,
                               const dim_lighting *lighting, cudaStream_t st) {
  for (int32_t i = 0; i < B; ++i) {  // the class indices are on the host here: fail loudly (the reference indexes a python list)
    const int32_t c = cls_host[i];
    if (c < 0 || c >= ctx->max_classes || ctx->meshes_host[c].V <= 0) {
      set_error("%s: instance %d has class index %d: out of range [0,%d) or no mesh uploaded for it", fn, (int)i, (int)c,
                (int)ctx->max_classes);
      return 2;
    }
  }
  if (frame_host)  // so are the frame indices: nothing is enqueued when one is out of range
    for (int32_t i = 0; i < B; ++i)
      if (frame_host[i] < 0 || frame_host[i] >= F) {
        set_error("%s: instance %d has frame index %d: out of range [0,%d)", fn, (int)i, (int)frame_host[i], (int)F);
        return 2;
      }
  if (K_host)  // and the cameras
    for (int32_t f = 0; f < F; ++f)
      if (const char *why = pinhole_defect(K_host + 9 * f)) {
        set_error("%s: frame %d has intrinsics that are not a finite pinhole matrix [[fx,0,cx],[0,fy,cy],[0,0,1]]: %s", fn,
                  (int)f, why);
        return 2;
      }
  const size_t P = (size_t)ctx->H * ctx->W;
  DIM_CHECK(cudaMemcpyAsync(ctx->image_observed_u8, frames_u8, (size_t)F * 3 * P, cudaMemcpyHostToDevice, st));
  DIM_CHECK(cudaMemcpyAsync(ctx->cls_dev, cls_host, sizeof(int) * B, cudaMemcpyHostToDevice, st));
  DIM_CHECK(cudaMemcpyAsync(ctx->pose_cur, pose_host, sizeof(double) * B * 12, cudaMemcpyHostToDevice, st));
  if (frame_host) DIM_CHECK(cudaMemcpyAsync(ctx->frame_dev, frame_host, sizeof(int) * B, cudaMemcpyHostToDevice, st));
  if (K_host) DIM_CHECK(cudaMemcpyAsync(ctx->K_dev, K_host, sizeof(float) * 9 * F, cudaMemcpyHostToDevice, st));
  RefineArgs a = refine_args(B, n_iter,
                             frame_cams(K9, K_host ? ctx->K_dev : nullptr, frame_host ? ctx->frame_dev : nullptr, F), zn, zf,
                             means, precision, lighting);
  a.obs4 = ctx->obs4; a.cls_idx = ctx->cls_dev; a.pose_init = ctx->pose_cur; a.poses = ctx->poses_dev;
  a.se3 = ctx->se3_hist_dev;
  if (lighting) {  // the intensities move to the context's buffer (a fixed address: graphs)
    a.intensity = ctx->lit_intensity;
    DIM_CHECK(cudaMemcpyAsync(ctx->lit_intensity, lighting->intensity, sizeof(float) * (size_t)n_iter * B * 3,
                              cudaMemcpyHostToDevice, st));
  }
  if (int rc = transform_u8_obs4_launch(ctx, ctx->image_observed_u8, F, means, ctx->obs4, st)) return rc;
  if (depth_u16) {  // the converted depth lands in obs4 outside the graph, like the image
    DIM_CHECK(cudaMemcpyAsync(ctx->depth_u16, depth_u16, sizeof(uint16_t) * F * P, cudaMemcpyHostToDevice, st));
    if (int rc = obs4_depth_launch(ctx, ctx->obs4, F, nullptr, ctx->depth_u16, depth_factor, st)) return rc;
  }
  if (int rc = refine_graphed(ctx, a, st)) return rc;
  DIM_CHECK(cudaMemcpyAsync(poses_out, ctx->poses_dev, sizeof(double) * (size_t)n_iter * B * 12, cudaMemcpyDeviceToHost, st));
  if (se3_out)
    DIM_CHECK(cudaMemcpyAsync(se3_out, ctx->se3_hist_dev, sizeof(float) * (size_t)n_iter * B * 7, cudaMemcpyDeviceToHost, st));
  return 0;
}

// lighting: the caller's lighting with HOST intensities [n_iter,B,3]; depth_u16: the caller's host depth file values [F,H,W]
DIM_API int32_t dim_refine_host_async(dim_ctx *ctx, const uint8_t *frames_u8, int32_t F, const int32_t *frame_host,
                                      const float *K9, const float *K_host, const int32_t *cls_host, const double *pose_host,
                                      int32_t B, int32_t n_iter, float zn, float zf, const double *means, int32_t precision,
                                      double *poses_out, float *se3_out, const uint16_t *depth_u16, float depth_factor,
                                      const dim_lighting *lighting, void *stream) {
  const char *fn = "dim_refine_host_async";
  if (int rc = refine_check(ctx, fn, true, frames_u8, F, frame_host, K9, K_host, cls_host, pose_host, B, n_iter, means,
                            poses_out, depth_u16, lighting))
    return rc;
  if (depth_u16 && !(depth_factor > 0.f && depth_factor < 3.0e38f)) return refuse(fn, "depth_factor must be positive and finite");
  return refine_host_enqueue(ctx, fn, frames_u8, F, frame_host, K_host, cls_host, pose_host, B, n_iter, K9, zn, zf, means,
                             precision, poses_out, se3_out, depth_u16, depth_factor, lighting, (cudaStream_t)stream);
}

// projective point-to-plane ICP against the observed depth (icp.cu; the contract is oracle/icp.py).  Refused calls enqueue
// nothing.  The call writes ren4, vbox, bbox_ren, cls_flag and pose_cur_f32, which every refinement iteration rewrites
// before reading, so refinement graphs captured before it replay unchanged.
DIM_API int32_t dim_icp(dim_ctx *ctx, const float *depth_frames, int32_t F, const int32_t *frame_idx, const float *K9_host,
                        const float *K_frames, const int32_t *cls_idx, const double *pose_in, int32_t B, int32_t n_iter,
                        float znear, float zfar, float max_dist, int32_t min_points, double *poses_out, int32_t *inliers,
                        float *rms, int32_t *status, void *stream) {
  const char *fn = "dim_icp";
  if (!(ctx && depth_frames && cls_idx && pose_in && poses_out && inliers && rms && status)) return refuse(fn, "NULL argument");
  if (int rc = frames_check(ctx, fn, K9_host, K_frames, "K_frames", B, F, frame_idx)) return rc;
  if (n_iter < 1) return refuse(fn, "n_iter must be >= 1");
  if (!(max_dist > 0.f && max_dist < 3.0e38f)) return refuse(fn, "max_dist must be positive and finite");
  if (min_points < 6) return refuse(fn, "min_points must be >= 6 (six pose parameters)");
  if (int rc = pinhole_check(fn, K9_host)) return rc;
  const IcpCall c{depth_frames, frame_cams(K9_host, K_frames, frame_idx, F), cls_idx, pose_in, B, n_iter, znear, zfar,
                  max_dist, min_points, poses_out, inliers, status, rms};
  return icp_launch(ctx, c, (cudaStream_t)stream);
}

// Visible Surface Discrepancy (vsd.cu; the contract is oracle/vsd.py).  Refused calls enqueue nothing and leave the outputs
// untouched.  The call writes ren4, vbox, bbox_ren, cls_flag, pose_cur_f32 and mask_rendered, which every refinement
// iteration (and dim_train_update, for mask_rendered) rewrites before reading, so graphs captured before it replay unchanged.
static int32_t pose_error_vsd(const char *fn, dim_ctx *ctx, const float *depth_frames, int32_t F, const int32_t *frame_idx,
                              const float *K9_host, const float *K_frames, const int32_t *cls_idx, const double *poses_est,
                              const double *poses_gt, int32_t B, float znear, float zfar, float delta, const double *taus_host,
                              int32_t n_tau, int32_t visib_mode, const double *diam_host, double *err, int32_t *status,
                              cudaStream_t st) {
  if (!(ctx && depth_frames && cls_idx && poses_est && poses_gt && taus_host && err)) return refuse(fn, "NULL argument");
  if (int rc = frames_check(ctx, fn, K9_host, K_frames, "K_frames", B, F, frame_idx)) return rc;
  if (n_tau < 1 || n_tau > VSD_MAX_TAU) return refuse(fn, "n_tau must be in [1,16]");
  if (!(delta > 0.f && delta < 3.0e38f)) return refuse(fn, "delta must be positive and finite");
  for (int32_t k = 0; k < n_tau; ++k)
    if (!(taus_host[k] > 0.0 && taus_host[k] < 1.0e308)) return refuse(fn, "every tau must be positive and finite");
  if (int rc = pinhole_check(fn, K9_host)) return rc;
  if (visib_mode != 0 && visib_mode != 1) return refuse(fn, "visib_mode must be 0 (SIXD 2017) or 1 (BOP 2019)");
  if (diam_host) {
    for (int32_t b = 0; b < B; ++b)
      if (!(diam_host[b] > 0.0 && diam_host[b] < 1.0e308)) return refuse(fn, "every diameter must be positive and finite");
    DIM_CHECK(cudaMemcpyAsync(ctx->vsd_diam, diam_host, sizeof(double) * B, cudaMemcpyHostToDevice, st));
  }
  const VsdCall c{depth_frames, frame_cams(K9_host, K_frames, frame_idx, F), cls_idx, poses_est, poses_gt, B, znear, zfar,
                  delta, taus_host, n_tau, err, status, visib_mode, diam_host ? ctx->vsd_diam : nullptr};
  return vsd_launch(ctx, c, st);
}

DIM_API int32_t dim_pose_error_vsd(dim_ctx *ctx, const float *depth_frames, int32_t F, const int32_t *frame_idx,
                                   const float *K9_host, const float *K_frames, const int32_t *cls_idx, const double *poses_est,
                                   const double *poses_gt, int32_t B, float znear, float zfar, float delta,
                                   const double *taus_host, int32_t n_tau, double *err, int32_t *status, void *stream) {
  return pose_error_vsd("dim_pose_error_vsd", ctx, depth_frames, F, frame_idx, K9_host, K_frames, cls_idx, poses_est,
                        poses_gt, B, znear, zfar, delta, taus_host, n_tau, 0, nullptr, err, status, (cudaStream_t)stream);
}

DIM_API int32_t dim_pose_error_vsd_ex(dim_ctx *ctx, const float *depth_frames, int32_t F, const int32_t *frame_idx,
                                      const float *K9_host, const float *K_frames, const int32_t *cls_idx,
                                      const double *poses_est, const double *poses_gt, int32_t B, float znear, float zfar,
                                      float delta, const double *taus_host, int32_t n_tau, int32_t visib_mode,
                                      const double *diam_host, double *err, int32_t *status, void *stream) {
  return pose_error_vsd("dim_pose_error_vsd_ex", ctx, depth_frames, F, frame_idx, K9_host, K_frames, cls_idx, poses_est,
                        poses_gt, B, znear, zfar, delta, taus_host, n_tau, visib_mode, diam_host, err, status,
                        (cudaStream_t)stream);
}

// BOP 2019 MSSD / MSPD over a symmetry set (bop.cu; the contract is oracle/bop.py).  Refused calls enqueue nothing and leave
// the outputs untouched.  The call writes only sym_partial, which nothing else reads.
DIM_API int32_t dim_pose_error_sym(dim_ctx *ctx, const double *poses_est, const double *poses_gt, int32_t M,
                                   const double *points, int32_t N, const double *syms, int32_t S, const double *K_inst,
                                   double *err2, int32_t *sym_idx2, void *stream) {
  const char *fn = "dim_pose_error_sym";
  if (!(ctx && poses_est && poses_gt && points && syms && K_inst && err2)) return refuse(fn, "NULL argument");
  if (M < 1 || M > ctx->max_batch) return refuse(fn, "M must be in [1, max_batch]");
  if (N < 1) return refuse(fn, "N must be >= 1");
  if (S < 1 || S > SYM_MAX) return refuse(fn, "S must be in [1,4096]");
  return sym_launch(ctx, SymCall{poses_est, poses_gt, M, points, N, syms, S, K_inst, err2, sym_idx2}, (cudaStream_t)stream);
}

DIM_API int32_t dim_depth_from_u16(dim_ctx *ctx, const uint16_t *depth_u16, int32_t F, float depth_factor, float *depth,
                                   void *stream) {
  const char *fn = "dim_depth_from_u16";
  if (!(ctx && depth_u16 && depth)) return refuse(fn, "NULL argument");
  if (F < 1) return refuse(fn, "F must be >= 1");
  if (!(depth_factor > 0.f && depth_factor < 3.0e38f)) return refuse(fn, "depth_factor must be positive and finite");
  return depth_u16_launch(depth_u16, (size_t)F * ctx->H * ctx->W, depth_factor, depth, (cudaStream_t)stream);
}

// status of the LAST dim_refine / dim_refine_host_async call on this context: [min(n_iter, 8), B] int32, device -> host
// (asynchronous on `stream`, which must be the stream that call ran on).  0 = ok; bit 0 = the rendered mask of that iteration
// was empty (object left the frustum: the reference crashes in ZoomMask, np.min of an empty array; here the fallback zoom
// factor (1,1,0,0) was used and the pose of that instance is meaningless); bit 1 = class index out of range or no mesh
// uploaded for it; bit 3 = dim_refine with a frame map: frame index out of range (frame 0 used).
DIM_API int32_t dim_refine_status(dim_ctx *ctx, int32_t B, int32_t n_iter, int32_t *status_host, void *stream) {
  DIM_REQUIRE(ctx && status_host && B >= 1 && B <= ctx->max_batch && n_iter >= 1, "dim_refine_status: bad argument");
  const int n = n_iter < 8 ? n_iter : 8;
  DIM_CHECK(cudaMemcpyAsync(status_host, ctx->status_hist, sizeof(int) * (size_t)n * B, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return 0;
}

// lighting: nullptr = the unlit re-render
DIM_API int32_t dim_train_update(dim_ctx *ctx, const int32_t *cls_idx, const float *src_pose, const float *rot_est,
                                 const float *trans_est, const float *tgt_pose, const float *depth_gt_observed, int32_t B,
                                 const double *K9, float zn, float zf, const double *means, const double *Tm, const double *Ts,
                                 int32_t rot_coord, float *image_rendered, float *depth_rendered, float *mask_rendered,
                                 float *src_pose_new, float *rot_label, float *trans_label, float *flow, float *flow_weights,
                                 const dim_lighting *lit, void *stream) {
  DIM_REQUIRE(ctx && cls_idx && src_pose && rot_est && trans_est && tgt_pose && K9 && means && Tm && Ts,
              "dim_train_update: NULL argument");
  DIM_REQUIRE(image_rendered && depth_rendered && mask_rendered && src_pose_new && rot_label && trans_label,
              "dim_train_update: NULL output");
  if (int rc = lit_check(ctx, lit, "dim_train_update")) return rc;
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch, "dim_train_update: batch exceeds max_batch");
  DIM_REQUIRE(rot_coord >= 0 && rot_coord <= 2, "dim_train_update: unknown rot_coord");
  cudaStream_t st = (cudaStream_t)stream;
  float *KT = ctx->pose_cur_f32;  // [B,12] scratch
  if (int rc = train_pose_launch(src_pose, rot_est, trans_est, tgt_pose, B, Tm, Ts, rot_coord, K9, src_pose_new,
                                 rot_label, trans_label, KT, st, lit ? ctx->light_pos : nullptr, lit ? lit->offset : nullptr))
    return rc;
  const float K9f[9] = {(float)K9[0], (float)K9[1], (float)K9[2], (float)K9[3], (float)K9[4],
                        (float)K9[5], (float)K9[6], (float)K9[7], (float)K9[8]};
  // no uint8 truncation on the train path (batch_updater_py_multi.py:184,234); the lit colours are already 8-bit quantised
  const LitParams lp = lit ? lit_params(ctx->light_pos, lit->intensity, lit->brightness_ratio) : LitParams{nullptr, nullptr, 0.f, 0.f};
  if (int rc = render_launch(ctx, cls_idx, src_pose_new, B, zn, zf, means,
                             {.cams = frame_cams(K9f), .out_image = image_rendered, .out_depth = depth_rendered,
                              .out_mask = mask_rendered, .trunc_u8 = 0, .lit = lit ? &lp : nullptr},
                             st))
    return rc;
  if (flow && flow_weights) {
    DIM_REQUIRE(depth_gt_observed != nullptr, "dim_train_update: flow labels need depth_gt_observed");
    // Kinv = inverse of K (np.linalg.inv, l.60) in float64, cast to float32 (l.292)
    const double a = K9[0], b_ = K9[1], c = K9[2], d = K9[3], e = K9[4], f = K9[5], g = K9[6], h = K9[7], i = K9[8];
    const double det = a * (e * i - f * h) - b_ * (d * i - f * g) + c * (d * h - e * g);
    const float Kinv[9] = {(float)((e * i - f * h) / det), (float)((c * h - b_ * i) / det), (float)((b_ * f - c * e) / det),
                           (float)((f * g - d * i) / det), (float)((a * i - c * g) / det), (float)((c * d - a * f) / det),
                           (float)((d * h - e * g) / det), (float)((b_ * g - a * h) / det), (float)((a * e - b_ * d) / det)};
    const size_t P = (size_t)ctx->H * ctx->W;
    // flow_weights = tile(valid, [1,2,1,1]) (l.296): the kernel writes both copies
    if (int rc = flow_launch(ctx, depth_rendered, depth_gt_observed, KT, Kinv, B, flow, ctx->mask_rendered,
                             nullptr, st))
      return rc;
    // interleave valid into the two weight planes per instance
    for (int pl = 0; pl < 2; ++pl)
      DIM_CHECK(cudaMemcpy2DAsync(flow_weights + pl * P, 2 * P * sizeof(float), ctx->mask_rendered, P * sizeof(float),
                                  P * sizeof(float), B, cudaMemcpyDeviceToDevice, st));
  }
  return 0;
}

DIM_API int32_t dim_profile_enable(dim_ctx *ctx, int32_t enable) {
  DIM_REQUIRE(ctx, "dim_profile_enable: NULL ctx");
  DIM_CHECK(cudaDeviceSynchronize());
  ctx->prof = enable != 0;
  ctx->prof_used = 0;
  return 0;
}
DIM_API int32_t dim_profile_read(dim_ctx *ctx, float *ms4, int32_t *iterations) {
  DIM_REQUIRE(ctx && ms4, "dim_profile_read: NULL argument");
  DIM_CHECK(cudaDeviceSynchronize());
  for (int k = 0; k < 4; ++k) ms4[k] = 0.f;
  const size_t n = ctx->prof_used / 5;
  for (size_t i = 0; i < n; ++i)
    for (int k = 0; k < 4; ++k) {
      float ms = 0.f;
      DIM_CHECK(cudaEventElapsedTime(&ms, ctx->prof_events[5 * i + k], ctx->prof_events[5 * i + k + 1]));
      ms4[k] += ms;
    }
  if (iterations) *iterations = (int32_t)n;
  ctx->prof_used = 0;
  return 0;
}

// ---- test hooks (not part of the drop-in surface; used by tests/ to look inside the conv tower)
DIM_API int32_t dim_debug_activation(dim_ctx *ctx, int32_t idx, int32_t lo, void *host_dst, uint64_t bytes) {
  return net_debug_activation(ctx, idx, lo, host_dst, (size_t)bytes);
}
DIM_API int32_t dim_debug_layer_geometry(dim_ctx *ctx, int32_t idx, int32_t *out8) {
  DIM_REQUIRE(ctx && out8 && idx >= 0 && idx <= 10, "dim_debug_layer_geometry: bad argument");
  net_layer_geometry(ctx, idx, out8);
  return 0;
}


DIM_API int32_t dim_debug_set_option(dim_ctx *ctx, const char *key, int32_t value) {
  DIM_REQUIRE(ctx && key, "dim_debug_set_option: NULL argument");
  drop_graphs(ctx);  // captured graphs hold the old kernel choice
  if (!strcmp(key, "graph")) { ctx->use_graph = value != 0; return 0; }
  if (!strcmp(key, "sms")) {
    // the SM count the launch schedules are sized for: the persistent conv grids, conv1's row runs, the training step's
    // parity-class streams and weight-gradient K slices.  The device is not touched.
    if (value < 0 || value > ctx->device_sms) {
      set_error("dim_debug_set_option: \"sms\" must be in [1, %d] (the device's SM count), or 0 for the device's count; got %d",
                ctx->device_sms, value);
      return 2;
    }
    ctx->num_sms = value ? value : ctx->device_sms;
    train_drop_maps(ctx);  // the cached training launch descriptors hold the old weight-gradient K-slice counts
    return 0;
  }
  set_error("dim_debug_set_option: unknown key '%s'", key);
  return 2;
}
DIM_API int32_t dim_debug_graph_count(dim_ctx *ctx) {
  if (!ctx) return -1;
  int32_t n = 0;
  for (const auto &g : ctx->graphs) n += g.exec != nullptr;
  return n;
}
DIM_API int32_t dim_debug_train_update(dim_ctx *ctx, int32_t B, float *kt_host, float *light_host) {
  DIM_REQUIRE(ctx && kt_host, "dim_debug_train_update: NULL argument");
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch, "dim_debug_train_update: batch exceeds max_batch");
  DIM_CHECK(cudaDeviceSynchronize());
  DIM_CHECK(cudaMemcpy(kt_host, ctx->pose_cur_f32, (size_t)B * 12 * sizeof(float), cudaMemcpyDeviceToHost));
  if (light_host) DIM_CHECK(cudaMemcpy(light_host, ctx->light_pos, (size_t)B * 3 * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}
DIM_API int32_t dim_debug_layer_profile(dim_ctx *ctx, int32_t enable, float *ms10) {
  DIM_REQUIRE(ctx, "dim_debug_layer_profile: NULL ctx");
  return net_layer_profile(ctx, enable, ms10);
}

// ADD / ADI (lib/utils/pose_error.py:72-108)
DIM_API int32_t dim_pose_error(dim_ctx *ctx, const double *poses_est, const double *poses_gt, int32_t M, const double *points,
                               int32_t N, int32_t symmetric, double *err, void *stream) {
  DIM_REQUIRE(ctx && poses_est && poses_gt && points && err && M >= 1 && N >= 1, "dim_pose_error: bad argument");
  return pose_error_launch(poses_est, poses_gt, M, points, N, symmetric, err, (cudaStream_t)stream);
}

// flow end-point error sums (deepim/core/tester.py:573-589)
DIM_API int32_t dim_flow_epe(dim_ctx *ctx, const float *flow_pred, const float *flow_gt, const float *visible, const float *bg,
                             int32_t B, double *out6, void *stream) {
  DIM_REQUIRE(ctx && flow_pred && flow_gt && visible && bg && out6 && B >= 1, "dim_flow_epe: bad argument");
  return epe_launch(flow_pred, flow_gt, visible, bg, B, ctx->H * ctx->W, out6, (cudaStream_t)stream);
}

// Proj. 2D / (rot, trans) distances (lib/utils/pose_error.py:55-69, lib/pair_matching/RT_transform.py:162-173)
DIM_API int32_t dim_pose_error_2d(dim_ctx *ctx, const double *poses_est, const double *poses_gt, int32_t M, const double *points,
                                  int32_t N, const double *K9_dev, double *err3, void *stream) {
  DIM_REQUIRE(ctx && poses_est && poses_gt && points && K9_dev && err3 && M >= 1 && N >= 1, "dim_pose_error_2d: bad argument");
  return pose_error2d_launch(poses_est, poses_gt, M, points, N, K9_dev, err3, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------ training step
DIM_API int32_t dim_train_create(dim_ctx *ctx, int32_t max_points) {
  DIM_REQUIRE(ctx && max_points >= 1, "dim_train_create: bad argument");
  return train_create(ctx, max_points);
}
DIM_API int64_t dim_train_param_count(dim_ctx *ctx) { return ctx ? (int64_t)train_param_count(ctx) : 0; }
DIM_API int32_t dim_train_param_info(int32_t input_depth, int32_t input_mask, int32_t idx, const char **name, int64_t *w_numel,
                                     int64_t *b_numel) {
  DIM_REQUIRE(name && w_numel && b_numel, "dim_train_param_info: NULL argument");
  DIM_REQUIRE(!input_depth || input_mask, "dim_train_param_info: input_depth with input_mask = 0 (depth input without the mask "
                                          "channels, INPUT_DEPTH without INPUT_MASK) is not supported");
  long long w = 0, b = 0;
  if (train_param_info(idx, name, &w, &b, input_depth != 0, input_mask != 0)) return 2;
  *w_numel = w; *b_numel = b;
  return 0;
}
DIM_API int32_t dim_train_load_params(dim_ctx *ctx, const float *flat_host, int64_t n, void *stream) {
  DIM_REQUIRE(ctx && flat_host && n > 0, "dim_train_load_params: bad argument");
  return train_load_params(ctx, flat_host, (size_t)n, (cudaStream_t)stream);
}
DIM_API int32_t dim_train_get_params(dim_ctx *ctx, float *flat_host, int64_t n, int32_t which, void *stream) {
  DIM_REQUIRE(ctx && flat_host && n > 0, "dim_train_get_params: bad argument");
  return train_get_params(ctx, flat_host, (size_t)n, which, (cudaStream_t)stream);
}
DIM_API int32_t dim_train_forward_backward(dim_ctx *ctx, const float *zio, const float *zir, const float *zmo, const float *zmr,
                                           const float *zoom_factor, const float *zflow, const float *zfw, const float *zmask_gt,
                                           const float *src_pose, const float *pc_model, const float *pc_weights,
                                           const float *pc_observed, int32_t B, int32_t N, float *rot_est_norm, float *trans_est,
                                           float *flow_est, float *mask_prob, float *losses4, float *grads, float *rot_raw,
                                           void *const *bucket_events, const int32_t *bucket_first_tensor, int32_t n_buckets,
                                           const float *zdo, const float *zdr, void *stream) {
  DIM_REQUIRE(ctx && zio && zir && zoom_factor, "dim_train_forward_backward: NULL argument");
  if (int rc = depth_check(ctx, zdo, zdr, "dim_train_forward_backward", "zoom_depth_observed / zoom_depth_rendered")) return rc;
  if (net_input_mask(ctx)) {
    DIM_REQUIRE(zmo && zmr, "dim_train_forward_backward: NULL argument");
  } else {
    DIM_REQUIRE(!zmo && !zmr, "dim_train_forward_backward: this context's network takes no mask input "
                              "(dim_ctx_set_input_mask): pass zoom_mask_observed = zoom_mask_rendered = NULL");
  }
  TrainIO io{zio, zir, zmo, zmr, zoom_factor, zflow, zfw, zmask_gt, src_pose, pc_model, pc_weights, pc_observed, B, N,
             rot_est_norm, trans_est, flow_est, mask_prob, losses4, grads, rot_raw, bucket_events, bucket_first_tensor,
             (bucket_events && bucket_first_tensor) ? n_buckets : 0, zdo, zdr};
  return train_forward_backward(ctx, io, (cudaStream_t)stream);
}
DIM_API int32_t dim_train_set_config(dim_ctx *ctx, const dim_train_config *cfg) {
  DIM_REQUIRE(ctx && cfg, "dim_train_set_config: NULL argument");
  DIM_REQUIRE(cfg->rot_coord == 0 || cfg->rot_coord == 1, "dim_train_set_config: rot_coord must be 0 (MODEL) or 1 (CAMERA)");
  DIM_REQUIRE(cfg->num_3d_sample > 0.f && cfg->normalize_3d_point > 0.f && cfg->normalize_flow > 0.f,
              "dim_train_set_config: num_3d_sample, normalize_3d_point and normalize_flow must be positive");
  for (int i = 0; i < 3; ++i) DIM_REQUIRE(cfg->trans_stds[i] != 0.f, "dim_train_set_config: trans_stds must be non-zero");
  ctx->cfg = *cfg;
  drop_graphs(ctx);  // the captured refinement chains carry trans_means / trans_stds / rot_coord as kernel arguments
  return 0;
}
DIM_API int32_t dim_train_get_config(dim_ctx *ctx, dim_train_config *cfg) {
  DIM_REQUIRE(ctx && cfg, "dim_train_get_config: NULL argument");
  *cfg = ctx->cfg;
  return 0;
}
DIM_API int32_t dim_train_sgd_update(dim_ctx *ctx, const float *grads, float lr, float momentum, float wd, float rescale_grad,
                                     void *stream) {
  DIM_REQUIRE(ctx && grads, "dim_train_sgd_update: NULL argument");
  return train_sgd_update(ctx, grads, lr, momentum, wd, rescale_grad, (cudaStream_t)stream);
}
DIM_API int32_t dim_train_set_precision(dim_ctx *ctx, int32_t precision) {
  DIM_REQUIRE(ctx, "dim_train_set_precision: NULL context");
  return train_set_precision(ctx, precision);
}
DIM_API int32_t dim_train_get_precision(dim_ctx *ctx, int32_t *precision) {
  DIM_REQUIRE(ctx && precision, "dim_train_get_precision: NULL argument");
  int p = 0;
  if (int rc = train_get_precision(ctx, &p)) return rc;
  *precision = p;
  return 0;
}
DIM_API int32_t dim_train_debug_tensor(dim_ctx *ctx, int32_t id, void *host_dst, uint64_t bytes) {
  DIM_REQUIRE(ctx && host_dst, "dim_train_debug_tensor: NULL argument");
  return train_debug_tensor(ctx, id, host_dst, (size_t)bytes);
}
DIM_API int32_t dim_train_debug_phases(dim_ctx *ctx, float *ms7) {
  DIM_REQUIRE(ctx && ms7, "dim_train_debug_phases: NULL argument");
  return train_debug_phases(ctx, ms7);
}
DIM_API int32_t dim_train_debug_geometry(dim_ctx *ctx, int32_t id, int32_t *out7) {
  DIM_REQUIRE(ctx && out7, "dim_train_debug_geometry: NULL argument");
  train_debug_geometry(ctx, id, out7);
  return 0;
}
DIM_API int32_t dim_train_debug_wgrad_slices(dim_ctx *ctx, int32_t B, int32_t *out36) {
  DIM_REQUIRE(ctx && out36, "dim_train_debug_wgrad_slices: NULL argument");
  return train_debug_wgrad_slices(ctx, B, out36);
}
}  // extern "C"
