// net_state.cuh -- state of the FlowNetS network shared by net.cu (inference) and train.cu (training step).
#pragma once
#include <map>

#include "conv_igemm.cuh"

namespace dim {

// FlowNetS tower: name, Cout, Cin, k, stride, pad (deepIM_flownet.py:63-107)
struct LayerSpec {
  const char *name;
  int Cout, Cin, k, stride, pad;
};
static const LayerSpec kLayers[10] = {
    {"flow_conv1", 64, 8, 7, 2, 3},  {"conv2", 128, 64, 5, 2, 2},   {"conv3", 256, 128, 5, 2, 2},
    {"conv3_1", 256, 256, 3, 1, 1},  {"conv4", 512, 256, 3, 2, 1},  {"conv4_1", 512, 512, 3, 1, 1},
    {"conv5", 512, 512, 3, 2, 1},    {"conv5_1", 512, 512, 3, 1, 1}, {"conv6", 1024, 512, 3, 2, 1},
    {"conv6_1", 1024, 1024, 3, 1, 1}};

struct LayerGeom {
  // logical
  int Cin, Cout, k, stride, pad, Hin, Win, Ho, Wo;
  // input buffer: [B, rows, cols, Cbuf] bf16 (conv1: space-to-depth, Cbuf = 32)
  int rows, cols, Cbuf, py, px;  // py/px: where the producer writes pixel (0,0) (pre-s2d for conv1)
  // implicit GEMM view
  int KH, KW, stride_eff, Ceff, Hq;
  int BLOCK_N, BLOCK_K, BW, BH, n_col_tiles, kblocks;
};

struct TensorMaps {
  ConvKParams kp[10];
};

// conv1 operand K order inside one (dh, dw) tap of the space-to-depth form: the four 8-channel chunks (ph, pw) sit at
// ph*16 + pw*8 -- the order of the input strip's chunk planes -- except for dw = 3, where the two pw = 0 chunks come first
// (the pw = 1 half is kw = 7, outside the filter): the kernels feed that K step from chunk planes 0 and 2 and drop the other.
__host__ __device__ inline int conv1_kslot(int dw, int ph, int pw) { return dw == 3 ? pw * 16 + ph * 8 : ph * 16 + pw * 8; }

// one element of an operand pack from its fp32 weight: hi = bf16(v); lo = bf16(v - hi) (the bf16x3 residual) and f16 =
// half(v), each only where its destination is given
__device__ __forceinline__ void store_split(__nv_bfloat16 *hi, __nv_bfloat16 *lo, size_t i, float v,
                                            __nv_bfloat16 *f16 = nullptr) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  if (hi) hi[i] = h;
  if (lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
  if (f16) reinterpret_cast<__half *>(f16)[i] = __float2half_rn(v);  // inf only for |w| > 65504
}

struct NetState {
  LayerGeom g[10];
  __nv_bfloat16 *w_hi[10] = {}, *w_lo[10] = {};
  __nv_bfloat16 *w_f16[10] = {};  // the same packs as IEEE half (DIM_PREC_FP16; 16-bit payload, typed like the others)
  float *bias[10] = {};
  __nv_bfloat16 *act_hi[11] = {}, *act_lo[11] = {};  // act[i] = input of layer i, act[10] = fc6 input
  size_t act_elems_per_image[11] = {};
  // fc
  __nv_bfloat16 *fc6_w_hi = nullptr, *fc6_w_lo = nullptr;  // [256][81920] in (h,w,c) order
  __nv_bfloat16 *fc6_w_f16 = nullptr;
  bool train_aliased = false;  // dim_train_load_params made biases / head parameters alias the fp32 master vector
  bool f16_stale = false;  // training updated the weights: the fp16 packs are packed lazily from the master (train_refresh_f16)
  float *fc6_b = nullptr, *fc7_wT = nullptr, *fc7_b = nullptr, *rot_w = nullptr, *rot_b = nullptr,
        *trans_w = nullptr, *trans_b = nullptr;
  float *fc6_partial = nullptr;  // [FC6_SPLITS][max_batch][256]
  cudaEvent_t *layer_events = nullptr;  // tuning hook: 11 events around the conv layers of the last forward
  bool loaded = false, net_ok = false;
  // RGB-D network (dim_ctx_set_input_depth): flow_conv1 takes 10 channels and its space-to-depth input has 64 channels
  // (conv1_rgbd_kernel); the 8-channel network's conv1 input buffers are kept for switching back
  bool input_depth = false;
  __nv_bfloat16 *act0_rgb_hi = nullptr, *act0_rgb_lo = nullptr, *act0_rgbd_hi = nullptr, *act0_rgbd_lo = nullptr;
  // image-only network (dim_ctx_set_input_mask(ctx, 0)): flow_conv1 takes 6 channels; conv1_kernel and its 8-lane input are
  // unchanged, the weight pack carries zero columns for lanes 6-7 and every producer writes zeros there
  bool input_mask = true;
  float *save_h6 = nullptr, *save_h7 = nullptr;  // training: fc6 / fc7 activations kept for the backward pass ([B][256])
  cudaEvent_t repack_done = nullptr;  // training: the operand packs are refreshed on an internal stream after an update;
                                      // every consumer (net_forward) orders itself behind this event.  A lazy refresh in
                                      // net_forward moves it to the caller's stream, so that the next update's SGD waits
                                      // until that refresh has read the master too
  bool lo_stale = false;  // training updated the weights without refreshing the bf16 'lo' halves (bf16x3 mode refreshes lazily)
  // per batch size (+ kF16MapKey for the fp16 operand maps).  Tensor maps and layer parameters only: the launch schedule
  // comes from dim_ctx::num_sms at every net_forward, so a change of the SM count leaves these valid
  std::map<int, TensorMaps> maps;
  int max_batch = 0;
};

static constexpr int FC6_K = 1024 * 8 * 10;
static constexpr int FC6_KC = 256;
static constexpr int FC6_SPLITS = FC6_K / FC6_KC;  // 320


// net.cu (only net.cu and train.cu build tensor maps)
int encode_map(CUtensorMap *m, void *base, int rank, const uint64_t *dims, const uint64_t *strides_bytes,
               const uint32_t *box, int block_k /*64: SW128, 32: SW64, 0: no swizzle*/);
static constexpr int kF16MapKey = 1 << 20;

}  // namespace dim
