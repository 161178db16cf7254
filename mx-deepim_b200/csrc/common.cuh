// common.cuh -- context, error handling and launch bookkeeping shared by all translation units.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>

#include <nvtx3/nvToolsExt.h>  // header-only; no-ops unless a profiler injects itself

#include "../../include/deepim_b200.h"

// NVTX range for the host-side enqueue of one stage (Nsight Systems timelines: SURVEY 5 "tracing"): scoped push / pop
struct DimNvtxRange {
  bool open = true;
  explicit DimNvtxRange(const char *name) { nvtxRangePushA(name); }
  void end() {  // close before the scope does (ranges must nest: end inner ranges first)
    if (open) { nvtxRangePop(); open = false; }
  }
  ~DimNvtxRange() { end(); }
  DimNvtxRange(const DimNvtxRange &) = delete;
  DimNvtxRange &operator=(const DimNvtxRange &) = delete;
};

namespace dim {

void set_error(const char *fmt, ...);
extern long long g_launches;

#define DIM_CHECK(expr)                                                                  \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      dim::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return 1;                                                                          \
    }                                                                                    \
  } while (0)

#define DIM_LAUNCH_CHECK()                                                               \
  do {                                                                                   \
    ++dim::g_launches;                                                                   \
    cudaError_t _e = cudaGetLastError();                                                 \
    if (_e != cudaSuccess) {                                                             \
      dim::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return 1;                                                                          \
    }                                                                                    \
  } while (0)

#define DIM_REQUIRE(cond, msg)                                        \
  do {                                                                \
    if (!(cond)) {                                                    \
      dim::set_error("%s:%d: %s", __FILE__, __LINE__, msg);           \
      return 2;                                                       \
    }                                                                 \
  } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------------------------- rasteriser
struct PVert {  // projected vertex, 24 B
  int X, Y;     // 24.8 fixed-point screen position
  float iz;     // 1/Zc
  float uz, vz; // u/Zc, v/Zc
  int ok;
};

struct MeshDev {
  const float *verts;   // [V,3]
  const float *uvs;     // [V,2]
  const int *faces;     // [F,3]
  const uint8_t *tex;   // [Th,Tw,3]
  int V, F, Th, Tw;
  const float *normals; // [V,3] per-vertex normals (lit renderer only; nullptr otherwise)
};

struct NetState;  // net_state.cuh

// The observed frame of instance b in the fused loop (dim_refine's frame map): frame_idx[b], or frame 0 when that lies outside
// [0, n_frames) -- a bad index never reads outside the packed frames (or the per-frame intrinsics); the zoom factor flags it
// as status bit 3.  frame_idx == nullptr: instance b observes frame b (no frame map).
__device__ __forceinline__ int frame_of(const int32_t *frame_idx, int n_frames, int b) {
  if (!frame_idx) return b;
  const int f = __ldg(frame_idx + b);
  return (f >= 0 && f < n_frames) ? f : 0;
}
__device__ __forceinline__ bool frame_bad(const int32_t *frame_idx, int n_frames, int b) {
  if (!frame_idx) return false;
  const int f = __ldg(frame_idx + b);
  return f < 0 || f >= n_frames;
}

// Everything the fused refinement loop reads from its caller, and the key of its CUDA graphs, compared byte for byte (so
// no padding).  Not in the key, because drop_graphs discards every graph when they change: ctx->cfg (trans means / stds,
// rot_coord), mesh uploads, network weights and the "graph" option.
struct RefineArgs {
  const float4 *obs4;        // n_frames observed frames
  const int32_t *frame_idx;  // device [B]: the frame instance b observes (read at replay); nullptr = frame b (no frame map)
  const float *K_frames;     // device [n_frames,9]: the camera of every frame (read at replay; K9 is then all zero);
                             // nullptr = K9 for every instance
  const int32_t *cls_idx;
  const double *pose_init, *pose_override;  // pose_override: nullable [n_iter,B,3,4] source pose of every iteration
  double *poses;
  float *se3, *zoom_factor;  // nullable: the context's scratch
  int32_t *bbox;             // nullable
  const float *intensity;    // lit: device [n_iter,B,3]; unlit: nullptr
  const float *depth_observed;  // RGB-D network, dim_refine: the caller's device depth; otherwise nullptr
  double means[3], offset[3];  // offset: the light's (lit only)
  float K9[9], zn, zf, brightness_ratio;
  int32_t B, n_iter, precision, lit;
  int32_t n_frames;  // frames in obs4 (dim_refine: B)
  int32_t zero;      // always 0: fills what would otherwise be tail padding
};
static_assert(sizeof(RefineArgs) == 12 * sizeof(void *) + 6 * sizeof(double) + 12 * sizeof(float) + 6 * sizeof(int32_t),
              "RefineArgs must have no padding: its bytes are the graph key");

}  // namespace dim

struct dim_ctx {
  int device = 0, max_batch = 0, H = 0, W = 0, max_classes = 0, max_verts = 0, max_faces = 0;
  int num_sms = 132;         // the SM count every launch decision uses (dim_debug_set_option "sms"; 0 restores device_sms)
  int device_sms = 132;      // the device's multiProcessorCount
  // meshes
  std::vector<dim::MeshDev> meshes_host;
  dim::MeshDev *meshes = nullptr;  // device table [max_classes]
  std::vector<void *> owned;       // device allocations to free
  // raster scratch
  dim::PVert *pverts = nullptr;          // [max_batch, max_verts]
  unsigned long long *vis = nullptr;     // [max_batch, H*W]
  int *vbox = nullptr;                   // [max_batch,4] screen bbox of projected vertices
  // zoom scratch
  int *bbox8 = nullptr;      // [max_batch, 8]
  int *cls_flag = nullptr;   // [max_batch] rasteriser: 2 = class index out of range / mesh missing (raster.cu mesh_for)
  int *status_hist = nullptr;  // [8, max_batch] per-iteration status of the last fused refinement (dim_refine_status)
  float *zoom_factor = nullptr;  // [max_batch,4]
  // refine-loop state
  float *mask_rendered = nullptr;  // [max_batch,H,W] scratch of dim_train_update (flow validity)
  int *bbox_ren = nullptr;   // [max_batch,4]
  double *pose_cur = nullptr;  // [max_batch,3,4]
  float *pose_cur_f32 = nullptr;
  float *se3_cur = nullptr;  // [max_batch,7]
  float4 *ren4 = nullptr, *obs4 = nullptr;  // [max_batch,H,W] pixel-interleaved images of the fused loop
  uint8_t *image_observed_u8 = nullptr;
  int *cls_dev = nullptr;
  int *frame_dev = nullptr;     // [max_batch] dim_refine_host_async: the caller's frame index of every instance
  float *K_dev = nullptr;       // [max_batch,9] dim_refine_host_async: the caller's intrinsics of every frame
  double *poses_dev = nullptr;  // [8, max_batch, 12]
  float *se3_hist_dev = nullptr;
  float *light_pos = nullptr;      // [max_batch,3] lit chain / lit train update: light of the pose being rendered
  float *lit_intensity = nullptr;  // [8, max_batch, 3] lit dim_refine_host_async: the caller's light intensities on the device
  uint16_t *depth_u16 = nullptr;   // [max_batch,H,W] RGB-D dim_refine_host_async: the caller's depth file values
  int *bbox_obs = nullptr;         // [max_batch,4] image-only network: the observed image's colour-valid box (ZoomImage)
  double *icp_partial = nullptr;   // [max_batch, H / ICP_ROWS, ICP_SLOT] dim_icp: one reduction slot per association CTA
  int32_t *vsd_partial = nullptr;  // [max_batch, H / VSD_ROWS, VSD_SLOT] dim_pose_error_vsd: one count slot per pass CTA
  int *vsd_box = nullptr;          // [max_batch,4] dim_pose_error_vsd: the ground-truth render's vertex box
  // background bank of dim_replace_background (dim_bg_upload): BGR u8 photos, each allocated at its upload
  struct BgImage { uint8_t *data = nullptr; int h = 0, w = 0; };
  std::vector<BgImage> bg;
  dim::NetState *net = nullptr;
  // CUDA graphs of the fused refinement chain (capi.cu refine_graphed): one executable graph per distinct argument set
  struct RefineGraph {
    dim::RefineArgs key;
    cudaGraphExec_t exec = nullptr;  // nullptr: seen once (eager warm-up run), captured on the next call
    long long kernels = 0;           // kernel nodes (dim_launch_count bookkeeping)
  };
  std::vector<RefineGraph> graphs;
  bool use_graph = true;
  // loss weights / normalisers / pose parameterisation (dim_train_set_config); defaults = the shipped LM6d config
  dim_train_config cfg = {0.25f, 0.03f, 0.1f, 3000.f, 0.1f, 20.f, {0.f, 0.f, 0.f}, {1.f, 1.f, 1.f}, 1};
  // stage profiling (dim_profile_enable)
  bool prof = false;
  std::vector<cudaEvent_t> prof_events;  // 5 per recorded iteration
  size_t prof_used = 0;
};

// device allocation owned by the context (freed by dim_ctx_destroy)
template <typename T>
static int dev_alloc(dim_ctx *ctx, T **p, size_t n, bool zero = false) {
  void *q = nullptr;
  DIM_CHECK(cudaMalloc(&q, n * sizeof(T)));
  if (zero) DIM_CHECK(cudaMemset(q, 0, n * sizeof(T)));
  ctx->owned.push_back(q);
  *p = reinterpret_cast<T *>(q);
  return 0;
}
