// raster.cu -- CUDA triangle rasteriser (compiled with -fmad=false: the float32 sequences must match
// the oracle bit for bit).
//
// Replaces lib/render_glumpy/render_py_multi.py (glumpy/OpenGL): Render_Py.render l.101-129, the GLSL
// programs l.22-52, my_compute_calib_proj l.134-151, _get_view_mtx l.153-160, and the post-render
// glue of deepim/core/tester.py:185-188,433-442 + lib/utils/image.py:583-594.
//
// Pipeline per call (all instances of the batch at once, HBM-bound):
//   raster_init      : reset per-instance boxes
//   raster_vertex    : one thread per (instance, vertex): pose * v, pinhole projection with the
//                      reference's pixel-centre convention (pixel (i,j) samples image point (j,i)),
//                      24.8 fixed-point snap; warp-reduced screen box of the instance
//   raster_coverage  : one thread per (instance, triangle): int64 edge functions, antisymmetric
//                      tie rule, perspective 1/Z, 64-bit atomicMin of (Z bits << 32 | tri id) into a
//                      visibility buffer.  Triangles with large boxes are swept by the whole warp.
//   raster_resolve   : one thread per 4 pixels: winner triangle -> perspective-correct UV -> nearest
//                      texel -> writes RGB-mean / depth / mask (/ BGR) with 16-byte stores, resets
//                      the visibility buffer, reduces the mask bbox.
// Algorithmic HBM bytes per instance: 16 B/px written (RGB + depth, SURVEY 8(d)); this version also
// writes the mask plane (4 B/px) and touches the visibility buffer only inside the vertex box.  In the fused
// refinement loop the only output is the pixel-interleaved (R,G,B,mask) image and it is written only inside the
// projected-vertex box: the zoom kernel knows the box and substitutes the background constant outside it.
#include "launch.cuh"

namespace dim {

static constexpr unsigned long long VIS_EMPTY = ~0ull;

struct RasterParams {
  const MeshDev *meshes;
  const int *cls;
  const float *pose;  // [B,3,4] f32
  PVert *pverts;
  unsigned long long *vis;
  int *vbox;      // [B,4]
  int *bbox_ren;  // [B,4]
  int max_verts, max_faces, H, W;
  int num_classes;  // size of the mesh table: class indices are range-checked on the device (mesh_for)
  int *cls_flag;    // [B] 0 ok / 2 = class index out of range or no mesh uploaded for it (renders nothing); nullable
  float fx, fy, cx, cy, zn, zf;
  const float *K_frames;     // fused loop, nullable: [n_frames,9] intrinsics; instance b projects with row frame_of(b) of them
  const int32_t *frame_idx;  // instead of fx, fy, cx, cy (RefineArgs)
  int n_frames;
  double mean[3];
  float bg[3];  // (float)(0.0 - mean)
  int trunc_u8;
  float *out_image, *out_depth, *out_mask, *out_bgr;
  float4 *out_ren4;  // [B,H,W] ((R-mean)+mean, (G-mean)+mean, (B-mean)+mean, mask): the fused loop's layout -- the "+ mean" is
                     // the zoom sampler's first float32 step (zoom_image_with_factor.py:44), applied here once per pixel
  int ren4_box_only; // 1: out_ren4 is written only inside the projected-vertex box (vbox); every pixel outside it is background
                     //    by construction and the only consumer (zoom_fused_nhwc8_kernel) substitutes the constant itself
  // lit renderer (render_py_light_modelnet_multi.py): per-instance light position / intensity, a0 + a1 * brightness
  int lit;
  const float *light_pos, *light_int;
  float a0, a1;
};

// class index -> mesh, range-checked: an out-of-range index (e.g. LINEMOD's 1-based class id) or a class whose mesh was never
// uploaded renders nothing instead of reading out of bounds; raster_vertex_kernel flags the instance in cls_flag
__device__ __forceinline__ MeshDev mesh_for(const RasterParams &p, int b) {
  const int c = p.cls[b];
  if (c < 0 || c >= p.num_classes) {
    MeshDev e;
    e.verts = nullptr; e.uvs = nullptr; e.faces = nullptr; e.tex = nullptr; e.V = e.F = e.Th = e.Tw = 0; e.normals = nullptr;
    return e;
  }
  return p.meshes[c];
}

__global__ void raster_init_kernel(int *vbox, int *bbox_ren, int B, int H, int W) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  vbox[4 * b + 0] = 0x7fffffff;
  vbox[4 * b + 1] = -0x7fffffff;
  vbox[4 * b + 2] = 0x7fffffff;
  vbox[4 * b + 3] = -0x7fffffff;
  bbox_ren[4 * b + 0] = W;
  bbox_ren[4 * b + 1] = -1;
  bbox_ren[4 * b + 2] = H;
  bbox_ren[4 * b + 3] = -1;
}

__global__ void __launch_bounds__(256) raster_vertex_kernel(RasterParams p) {
  const int b = blockIdx.y;
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  const MeshDev m = mesh_for(p, b);
  if (p.cls_flag && v == 0) p.cls_flag[b] = m.V > 0 ? 0 : 2;
  const float *pose = p.pose + 12 * b;
  int ok = 0, X = 0, Y = 0;
  float fx = p.fx, fy = p.fy, cx = p.cx, cy = p.cy;
  if (p.K_frames) {
    const float *k = p.K_frames + 9 * frame_of(p.frame_idx, p.n_frames, b);
    fx = __ldg(k + 0); cx = __ldg(k + 2); fy = __ldg(k + 4); cy = __ldg(k + 5);
  }
  if (v < m.V) {
    float x = m.verts[3 * v], y = m.verts[3 * v + 1], z = m.verts[3 * v + 2];
    float xc = ((pose[0] * x + pose[1] * y) + pose[2] * z) + pose[3];
    float yc = ((pose[4] * x + pose[5] * y) + pose[6] * z) + pose[7];
    float zc = ((pose[8] * x + pose[9] * y) + pose[10] * z) + pose[11];
    ok = zc > 1e-6f;
    float sx = 0.f, sy = 0.f, iz = 0.f;
    if (ok) {
      sx = (fx * xc) / zc + cx;
      sy = (fy * yc) / zc + cy;
      ok = (fabsf(sx) <= 1e6f) && (fabsf(sy) <= 1e6f);
      iz = 1.0f / zc;
    }
    PVert o;
    o.ok = ok;
    if (ok) {
      X = __float2int_rn(sx * 256.0f);
      Y = __float2int_rn(sy * 256.0f);
      o.X = X;
      o.Y = Y;
      o.iz = iz;
      o.uz = m.uvs[2 * v] * iz;
      o.vz = m.uvs[2 * v + 1] * iz;
    } else {
      o.X = o.Y = 0;
      o.iz = o.uz = o.vz = 0.f;
    }
    p.pverts[(size_t)b * p.max_verts + v] = o;
  }
  // conservative screen box of the instance (pixel units)
  int x0 = ok ? (X >> 8) : 0x7fffffff, x1 = ok ? ((X + 255) >> 8) : -0x7fffffff;
  int y0 = ok ? (Y >> 8) : 0x7fffffff, y1 = ok ? ((Y + 255) >> 8) : -0x7fffffff;
  x0 = __reduce_min_sync(0xffffffffu, x0);
  x1 = __reduce_max_sync(0xffffffffu, x1);
  y0 = __reduce_min_sync(0xffffffffu, y0);
  y1 = __reduce_max_sync(0xffffffffu, y1);
  if ((threadIdx.x & 31) == 0 && x1 >= x0) {
    atomicMin(&p.vbox[4 * b + 0], x0);
    atomicMax(&p.vbox[4 * b + 1], x1);
    atomicMin(&p.vbox[4 * b + 2], y0);
    atomicMax(&p.vbox[4 * b + 3], y1);
  }
}

__device__ __forceinline__ long long edge_fn(int ax, int ay, int bx, int by, int px, int py) {
  return (long long)(bx - ax) * (long long)(py - ay) - (long long)(by - ay) * (long long)(px - ax);
}
// pixel centre exactly on edge a->b belongs to the triangle iff dy>0 or (dy==0 and dx<0)
__device__ __forceinline__ bool edge_owns(int ax, int ay, int bx, int by) {
  int dx = bx - ax, dy = by - ay;
  return (dy > 0) || (dy == 0 && dx < 0);
}

struct TriSetup {
  int ax, ay, bx, by, cx, cy;
  float aiz, biz, ciz;
  long long area;
};

// returns false for degenerate / culled triangles; orients to positive area (swaps b,c)
__device__ __forceinline__ bool tri_setup(const PVert &A, PVert &Bv, PVert &Cv, TriSetup &t) {
  if (!(A.ok && Bv.ok && Cv.ok)) return false;
  long long area = edge_fn(A.X, A.Y, Bv.X, Bv.Y, Cv.X, Cv.Y);
  if (area == 0) return false;
  if (area < 0) {
    PVert tmp = Bv;
    Bv = Cv;
    Cv = tmp;
    area = -area;
  }
  t.ax = A.X; t.ay = A.Y; t.bx = Bv.X; t.by = Bv.Y; t.cx = Cv.X; t.cy = Cv.Y;
  t.aiz = A.iz; t.biz = Bv.iz; t.ciz = Cv.iz;
  t.area = area;
  return true;
}

__device__ __forceinline__ bool tri_fragment(const TriSetup &t, int i, int j, float zn, float zf,
                                             float &b0, float &b1, float &b2, float &iz, float &z) {
  int px = j << 8, py = i << 8;
  long long w0 = edge_fn(t.bx, t.by, t.cx, t.cy, px, py);
  long long w1 = edge_fn(t.cx, t.cy, t.ax, t.ay, px, py);
  long long w2 = edge_fn(t.ax, t.ay, t.bx, t.by, px, py);
  if (w0 < 0 || w1 < 0 || w2 < 0) return false;
  if (w0 == 0 && !edge_owns(t.bx, t.by, t.cx, t.cy)) return false;
  if (w1 == 0 && !edge_owns(t.cx, t.cy, t.ax, t.ay)) return false;
  if (w2 == 0 && !edge_owns(t.ax, t.ay, t.bx, t.by)) return false;
  float fa = (float)t.area;
  b0 = (float)w0 / fa;
  b1 = (float)w1 / fa;
  b2 = (float)w2 / fa;
  iz = (b0 * t.aiz + b1 * t.biz) + b2 * t.ciz;
  z = 1.0f / iz;
  return (z >= zn && z <= zf);
}

__device__ __forceinline__ void tri_box(const TriSetup &t, int H, int W, int &j0, int &j1, int &i0, int &i1) {
  int minX = min(t.ax, min(t.bx, t.cx)), maxX = max(t.ax, max(t.bx, t.cx));
  int minY = min(t.ay, min(t.by, t.cy)), maxY = max(t.ay, max(t.by, t.cy));
  j0 = max((minX + 255) >> 8, 0);
  j1 = min(maxX >> 8, W - 1);
  i0 = max((minY + 255) >> 8, 0);
  i1 = min(maxY >> 8, H - 1);
}

static constexpr int SMALL_TRI_PIXELS = 48;

__global__ void __launch_bounds__(128) raster_coverage_kernel(RasterParams p) {
  const int b = blockIdx.y;
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const MeshDev m = mesh_for(p, b);
  const PVert *pv = p.pverts + (size_t)b * p.max_verts;
  unsigned long long *vis = p.vis + (size_t)b * p.H * p.W;

  TriSetup t;
  bool valid = false;
  int j0 = 0, j1 = -1, i0 = 0, i1 = -1;
  if (f < m.F) {
    PVert A = pv[m.faces[3 * f]], Bv = pv[m.faces[3 * f + 1]], Cv = pv[m.faces[3 * f + 2]];
    valid = tri_setup(A, Bv, Cv, t);
    if (valid) {
      tri_box(t, p.H, p.W, j0, j1, i0, i1);
      valid = (j1 >= j0) && (i1 >= i0);
    }
  }
  const int bw = valid ? (j1 - j0 + 1) : 0, bh = valid ? (i1 - i0 + 1) : 0;
  const bool big = valid && (bw * bh > SMALL_TRI_PIXELS);
  if (valid && !big) {
    for (int i = i0; i <= i1; ++i)
      for (int j = j0; j <= j1; ++j) {
        float b0, b1, b2, iz, z;
        if (tri_fragment(t, i, j, p.zn, p.zf, b0, b1, b2, iz, z)) {
          unsigned long long key = ((unsigned long long)__float_as_uint(z) << 32) | (unsigned)f;
          atomicMin(&vis[(size_t)i * p.W + j], key);
        }
      }
  }
  // large triangles: the whole warp sweeps the box of one triangle at a time
  unsigned bigmask = __ballot_sync(0xffffffffu, big);
  while (bigmask) {
    const int src = __ffs(bigmask) - 1;
    bigmask &= bigmask - 1;
    TriSetup s;
    s.ax = __shfl_sync(0xffffffffu, t.ax, src);
    s.ay = __shfl_sync(0xffffffffu, t.ay, src);
    s.bx = __shfl_sync(0xffffffffu, t.bx, src);
    s.by = __shfl_sync(0xffffffffu, t.by, src);
    s.cx = __shfl_sync(0xffffffffu, t.cx, src);
    s.cy = __shfl_sync(0xffffffffu, t.cy, src);
    s.aiz = __shfl_sync(0xffffffffu, t.aiz, src);
    s.biz = __shfl_sync(0xffffffffu, t.biz, src);
    s.ciz = __shfl_sync(0xffffffffu, t.ciz, src);
    s.area = __shfl_sync(0xffffffffu, t.area, src);
    const int sj0 = __shfl_sync(0xffffffffu, j0, src), sj1 = __shfl_sync(0xffffffffu, j1, src);
    const int si0 = __shfl_sync(0xffffffffu, i0, src), si1 = __shfl_sync(0xffffffffu, i1, src);
    const int sf = __shfl_sync(0xffffffffu, f, src);
    const int sw = sj1 - sj0 + 1, n = sw * (si1 - si0 + 1);
    for (int k = lane; k < n; k += 32) {
      int i = si0 + k / sw, j = sj0 + k % sw;
      float b0, b1, b2, iz, z;
      if (tri_fragment(s, i, j, p.zn, p.zf, b0, b1, b2, iz, z)) {
        unsigned long long key = ((unsigned long long)__float_as_uint(z) << 32) | (unsigned)sf;
        atomicMin(&vis[(size_t)i * p.W + j], key);
      }
    }
  }
}

// colour chain of the reference: u8 texel -> GL float (c/255) -> "*255" (render_py_multi.py:124)
// -> optional uint8 truncation (deepim/core/tester.py:188)
__device__ __forceinline__ float colour_of(unsigned char c, int trunc_u8) {
  float f = ((float)c / 255.0f) * 255.0f;
  if (trunc_u8) f = (float)(unsigned char)f;
  return f;
}

// The two lit renderers of the reference share the Lambert term and differ in where the light colour enters:
//   SHADE_MODELNET  (render_py_light_modelnet_multi.py)  colour_c = texel_c * ((a0 + a1 * brightness) * I_c)
//   SHADE_PY_LIGHT  (render_py_light.py, get_fragment)   colour_c = texel_c * (a0 + (a1 * brightness) * I_c)
// with a0 = 1 - ratio, a1 = ratio; the fragment (b0, b1, b2, iz) is winner triangle f of instance b.  Returns the colours
// quantised like the 8-bit framebuffer the reference reads back.
enum Shade { SHADE_MODELNET, SHADE_PY_LIGHT };

template <Shade S>
__device__ __forceinline__ void shade_lit(const RasterParams &p, const MeshDev &m, const PVert *pv, int b, int f, float b0,
                                          float b1, float b2, float iz, const PVert &A, const PVert &Bv, const PVert &Cv,
                                          const unsigned char *tp, float a0, float a1, float q[3]) {
  // Lambert shading, same float32 sequence as the CPU checker (see DESIGN.md "lit renderer")
  const int iA = m.faces[3 * f];
  int iB = m.faces[3 * f + 1], iC = m.faces[3 * f + 2];
  if (edge_fn(pv[iA].X, pv[iA].Y, pv[iB].X, pv[iB].Y, pv[iC].X, pv[iC].Y) < 0) { const int tmp = iB; iB = iC; iC = tmp; }
  const float w0 = b0 * A.iz, w1 = b1 * Bv.iz, w2 = b2 * Cv.iz;
  const float *ps = p.pose + 12 * b;
  float pm[3], nm[3], pc[3], nc[3];
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    pm[e] = ((w0 * m.verts[3 * iA + e] + w1 * m.verts[3 * iB + e]) + w2 * m.verts[3 * iC + e]) / iz;
    nm[e] = ((w0 * m.normals[3 * iA + e] + w1 * m.normals[3 * iB + e]) + w2 * m.normals[3 * iC + e]) / iz;
  }
#pragma unroll
  for (int rr = 0; rr < 3; ++rr) {
    pc[rr] = ((ps[4 * rr] * pm[0] + ps[4 * rr + 1] * pm[1]) + ps[4 * rr + 2] * pm[2]) + ps[4 * rr + 3];
    nc[rr] = (ps[4 * rr] * nm[0] + ps[4 * rr + 1] * nm[1]) + ps[4 * rr + 2] * nm[2];
  }
  const float *lp = p.light_pos + 3 * b, *li = p.light_int + 3 * b;
  const float s0 = lp[0] - pc[0], s1 = lp[1] - (0.f - pc[1]), s2 = lp[2] - (0.f - pc[2]);
  const float g0 = nc[0], g1 = 0.f - nc[1], g2 = 0.f - nc[2];
  const float dot = (g0 * s0 + g1 * s1) + g2 * s2;
  const float ls = sqrtf((s0 * s0 + s1 * s1) + s2 * s2), ln = sqrtf((g0 * g0 + g1 * g1) + g2 * g2);
  const float den = ls * ln;
  float br = 0.f;
  if (den > 0.f) br = dot / den;
  br = br < 1.f ? br : 1.f;
  br = br > 0.f ? br : 0.f;
  const float scale = S == SHADE_MODELNET ? a0 + a1 * br : a1 * br;
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    float col = S == SHADE_MODELNET ? ((float)tp[e] / 255.0f) * (scale * li[e]) : ((float)tp[e] / 255.0f) * (a0 + scale * li[e]);
    col = col < 1.f ? col : 1.f;
    col = col > 0.f ? col : 0.f;
    q[e] = rintf(col * 255.0f);
  }
}

// LIT is a compile-time switch: the unlit instantiation (the refinement loop's renderer) carries none of the shading code.
// REN4_DEPTH (the RGB-D network's loop): the w lane of out_ren4 holds the depth instead of the 0/1 mask; the zoom kernel
// samples it as depth_rendered and re-derives the mask as depth > 0.2, which is how the mask is made here.
// COLOUR_BOX (the image-only network's loop): bbox_ren is ZoomImage's rendered box (zoom_image.py:35-37), the pixels whose
// ((x + y) + z) > 0.01f over the ren4 colours (image + mean): the float32 expression of zoom.cu's img_mode bbox, on the
// very values ren4 holds.  Uncovered pixels hold background + mean = 0 and never pass, so only covered ones are tested.
template <bool LIT, bool REN4_DEPTH = false, bool COLOUR_BOX = false>
__global__ void __launch_bounds__(256) raster_resolve_kernel(RasterParams p) {
  const int b = blockIdx.y;
  const int W4 = p.W >> 2;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in_range = q < W4 * p.H;
  const int i = in_range ? q / W4 : 0, j4 = in_range ? (q % W4) << 2 : 0;
  const size_t P = (size_t)p.H * p.W;
  const int vx0 = p.vbox[4 * b + 0], vx1 = p.vbox[4 * b + 1], vy0 = p.vbox[4 * b + 2], vy1 = p.vbox[4 * b + 3];
  unsigned long long *vis = p.vis + (size_t)b * P + (size_t)i * p.W + j4;

  float r[4], g[4], bl[4], d[4], mk[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    r[k] = p.bg[0]; g[k] = p.bg[1]; bl[k] = p.bg[2]; d[k] = 0.f; mk[k] = 0.f;
  }
  float raw[4][3];
#pragma unroll
  for (int k = 0; k < 4; ++k) raw[k][0] = raw[k][1] = raw[k][2] = 0.f;

  int mx0 = 0x7fffffff, mx1 = -1, my0 = 0x7fffffff, my1 = -1;
  const bool in_box = in_range && i >= vy0 && i <= vy1 && j4 + 3 >= vx0 && j4 <= vx1;
  if (in_box) {
    ulonglong2 k01 = *reinterpret_cast<const ulonglong2 *>(vis);
    ulonglong2 k23 = *reinterpret_cast<const ulonglong2 *>(vis + 2);
    unsigned long long keys[4] = {k01.x, k01.y, k23.x, k23.y};
    bool any = false;
    const MeshDev m = mesh_for(p, b);
    const PVert *pv = p.pverts + (size_t)b * p.max_verts;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (keys[k] == VIS_EMPTY) continue;
      any = true;
      const int f = (int)(unsigned)(keys[k] & 0xffffffffull);
      PVert A = pv[m.faces[3 * f]], Bv = pv[m.faces[3 * f + 1]], Cv = pv[m.faces[3 * f + 2]];
      TriSetup t;
      tri_setup(A, Bv, Cv, t);
      float b0 = 0.f, b1 = 0.f, b2 = 0.f, iz = 1.f, z = 0.f;
      tri_fragment(t, i, j4 + k, p.zn, p.zf, b0, b1, b2, iz, z);
      float un = (b0 * A.uz + b1 * Bv.uz) + b2 * Cv.uz;
      float vn = (b0 * A.vz + b1 * Bv.vz) + b2 * Cv.vz;
      float u = un / iz, v = vn / iz;
      int tx = (int)floorf(u * (float)m.Tw), ty = (int)floorf(v * (float)m.Th);
      tx = min(max(tx, 0), m.Tw - 1);
      ty = min(max(ty, 0), m.Th - 1);
      const unsigned char *tp = m.tex + ((size_t)ty * m.Tw + tx) * 3;
      float c0, c1, c2;
      if (LIT) {
        float q[3];
        shade_lit<SHADE_MODELNET>(p, m, pv, b, f, b0, b1, b2, iz, A, Bv, Cv, tp, p.a0, p.a1, q);
        c0 = q[0]; c1 = q[1]; c2 = q[2];
      } else {
        c0 = colour_of(tp[0], p.trunc_u8); c1 = colour_of(tp[1], p.trunc_u8); c2 = colour_of(tp[2], p.trunc_u8);
      }
      raw[k][0] = c0; raw[k][1] = c1; raw[k][2] = c2;
      // image.transform works in float64 and nd.array casts to float32 (lib/utils/image.py:583-594)
      if (p.trunc_u8) {
        r[k] = (float)((double)c0 - p.mean[0]);
        g[k] = (float)((double)c1 - p.mean[1]);
        bl[k] = (float)((double)c2 - p.mean[2]);
      } else {  // train path (batch_updater_py_multi.py:234-235): float32 image -= float32 pixel_means
        r[k] = c0 - (float)p.mean[0];
        g[k] = c1 - (float)p.mean[1];
        bl[k] = c2 - (float)p.mean[2];
      }
      d[k] = z;
      if (z > 0.2f) mk[k] = 1.f;  // mask = depth > 0.2 (deepim/core/tester.py:440)
      bool in_bbox = z > 0.2f;
      if (COLOUR_BOX)
        in_bbox = ((r[k] + (float)p.mean[0]) + (g[k] + (float)p.mean[1])) + (bl[k] + (float)p.mean[2]) > 0.01f;
      if (in_bbox) {
        mx0 = min(mx0, j4 + k);
        mx1 = max(mx1, j4 + k);
        my0 = i;
        my1 = i;
      }
    }
    if (any) {  // hand the visibility buffer back empty for the next render
      *reinterpret_cast<ulonglong2 *>(vis) = make_ulonglong2(VIS_EMPTY, VIS_EMPTY);
      *reinterpret_cast<ulonglong2 *>(vis + 2) = make_ulonglong2(VIS_EMPTY, VIS_EMPTY);
    }
  }
  if (in_range) {
    const size_t o = (size_t)i * p.W + j4;
    if (p.out_image) {
      float *img = p.out_image + (size_t)b * 3 * P;
      *reinterpret_cast<float4 *>(img + o) = make_float4(r[0], r[1], r[2], r[3]);
      *reinterpret_cast<float4 *>(img + P + o) = make_float4(g[0], g[1], g[2], g[3]);
      *reinterpret_cast<float4 *>(img + 2 * P + o) = make_float4(bl[0], bl[1], bl[2], bl[3]);
    }
    if (p.out_ren4 && (in_box || !p.ren4_box_only)) {
      float4 *o4 = p.out_ren4 + (size_t)b * P + o;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        o4[k] = make_float4(r[k] + (float)p.mean[0], g[k] + (float)p.mean[1], bl[k] + (float)p.mean[2], REN4_DEPTH ? d[k] : mk[k]);
    }
    if (p.out_depth) *reinterpret_cast<float4 *>(p.out_depth + (size_t)b * P + o) = make_float4(d[0], d[1], d[2], d[3]);
    if (p.out_mask) *reinterpret_cast<float4 *>(p.out_mask + (size_t)b * P + o) = make_float4(mk[0], mk[1], mk[2], mk[3]);
    if (p.out_bgr) {  // Render_Py layout [H,W,3] BGR: 12 floats = 3 float4
      float *o3 = p.out_bgr + ((size_t)b * P + o) * 3;
      *reinterpret_cast<float4 *>(o3) = make_float4(raw[0][2], raw[0][1], raw[0][0], raw[1][2]);
      *reinterpret_cast<float4 *>(o3 + 4) = make_float4(raw[1][1], raw[1][0], raw[2][2], raw[2][1]);
      *reinterpret_cast<float4 *>(o3 + 8) = make_float4(raw[2][0], raw[3][2], raw[3][1], raw[3][0]);
    }
  }
  // mask bbox (min/max nonzero col/row), warp-reduced
  mx0 = __reduce_min_sync(0xffffffffu, mx0);
  mx1 = __reduce_max_sync(0xffffffffu, mx1);
  my0 = __reduce_min_sync(0xffffffffu, my0);
  my1 = __reduce_max_sync(0xffffffffu, my1);
  if ((threadIdx.x & 31) == 0 && mx1 >= 0 && p.bbox_ren) {
    atomicMin(&p.bbox_ren[4 * b + 0], mx0);
    atomicMax(&p.bbox_ren[4 * b + 1], mx1);
    atomicMin(&p.bbox_ren[4 * b + 2], my0);
    atomicMax(&p.bbox_ren[4 * b + 3], my1);
  }
}

// empty masks are reported as -1,-1,-1,-1 (oracle convention)
__global__ void raster_finish_kernel(int *bbox_ren, int *out_bbox, int B) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int x0 = bbox_ren[4 * b], x1 = bbox_ren[4 * b + 1], y0 = bbox_ren[4 * b + 2], y1 = bbox_ren[4 * b + 3];
  if (x1 < 0) x0 = x1 = y0 = y1 = -1;
  bbox_ren[4 * b] = x0; bbox_ren[4 * b + 1] = x1; bbox_ren[4 * b + 2] = y0; bbox_ren[4 * b + 3] = y1;
  if (out_bbox) {
    out_bbox[4 * b] = x0; out_bbox[4 * b + 1] = x1; out_bbox[4 * b + 2] = y0; out_bbox[4 * b + 3] = y1;
  }
}

// The data-preparation render (toolkit/LM6d_ds_1, ds_2, ds_4, LM6d_0): from one visibility pass, the Render_Py_Light colour
// (SHADE_PY_LIGHT, ratio per instance), the unlit colour rgb_gl.astype('uint8') (Render_Py), the depth file's
// (depth * depth_factor).astype(uint16) and the label depth != 0, as u8 / u16 planes ready for the PNG encoder.
template <bool LIT>
__global__ void __launch_bounds__(256) raster_dataset_kernel(RasterParams p, DatasetOut o) {
  const int b = blockIdx.y;
  const int W4 = p.W >> 2;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= W4 * p.H) return;
  const int i = q / W4, j4 = (q % W4) << 2;
  const size_t P = (size_t)p.H * p.W;
  const int vx0 = p.vbox[4 * b + 0], vx1 = p.vbox[4 * b + 1], vy0 = p.vbox[4 * b + 2], vy1 = p.vbox[4 * b + 3];
  unsigned long long *vis = p.vis + (size_t)b * P + (size_t)i * p.W + j4;

  unsigned lit[3] = {0u, 0u, 0u}, un[3] = {0u, 0u, 0u};  // 4 BGR pixels = 12 bytes, little-endian
  unsigned dep[2] = {0u, 0u}, lab = 0u;
  if (i >= vy0 && i <= vy1 && j4 + 3 >= vx0 && j4 <= vx1) {
    ulonglong2 k01 = *reinterpret_cast<const ulonglong2 *>(vis);
    ulonglong2 k23 = *reinterpret_cast<const ulonglong2 *>(vis + 2);
    unsigned long long keys[4] = {k01.x, k01.y, k23.x, k23.y};
    bool any = false;
    const MeshDev m = mesh_for(p, b);
    const PVert *pv = p.pverts + (size_t)b * p.max_verts;
    const float a1 = LIT ? o.ratio[b] : 0.f, a0 = 1.f - a1;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (keys[k] == VIS_EMPTY) continue;
      any = true;
      const int f = (int)(unsigned)(keys[k] & 0xffffffffull);
      PVert A = pv[m.faces[3 * f]], Bv = pv[m.faces[3 * f + 1]], Cv = pv[m.faces[3 * f + 2]];
      TriSetup t;
      tri_setup(A, Bv, Cv, t);
      float b0 = 0.f, b1 = 0.f, b2 = 0.f, iz = 1.f, z = 0.f;
      tri_fragment(t, i, j4 + k, p.zn, p.zf, b0, b1, b2, iz, z);
      float un_ = (b0 * A.uz + b1 * Bv.uz) + b2 * Cv.uz;
      float vn_ = (b0 * A.vz + b1 * Bv.vz) + b2 * Cv.vz;
      float u = un_ / iz, v = vn_ / iz;
      int tx = (int)floorf(u * (float)m.Tw), ty = (int)floorf(v * (float)m.Th);
      tx = min(max(tx, 0), m.Tw - 1);
      ty = min(max(ty, 0), m.Th - 1);
      const unsigned char *tp = m.tex + ((size_t)ty * m.Tw + tx) * 3;
#pragma unroll
      for (int e = 0; e < 3; ++e) {  // BGR byte 3k + e of the 12 holds channel 2 - e
        const int byte = 3 * k + e;
        un[byte >> 2] |= (unsigned)(unsigned char)colour_of(tp[2 - e], 0) << ((byte & 3) * 8);
      }
      if (LIT) {
        float c[3];
        shade_lit<SHADE_PY_LIGHT>(p, m, pv, b, f, b0, b1, b2, iz, A, Bv, Cv, tp, a0, a1, c);
#pragma unroll
        for (int e = 0; e < 3; ++e) {
          const int byte = 3 * k + e;
          lit[byte >> 2] |= (unsigned)c[2 - e] << ((byte & 3) * 8);
        }
      }
      dep[k >> 1] |= (unsigned)(unsigned short)(z * o.depth_factor) << ((k & 1) * 16);
      if (z != 0.f) lab |= 1u << (k * 8);
    }
    if (any) {  // hand the visibility buffer back empty for the next render
      *reinterpret_cast<ulonglong2 *>(vis) = make_ulonglong2(VIS_EMPTY, VIS_EMPTY);
      *reinterpret_cast<ulonglong2 *>(vis + 2) = make_ulonglong2(VIS_EMPTY, VIS_EMPTY);
    }
  }
  const size_t px = (size_t)b * P + (size_t)i * p.W + j4;
  if (LIT && o.lit_bgr) *reinterpret_cast<uint3 *>(o.lit_bgr + 3 * px) = make_uint3(lit[0], lit[1], lit[2]);
  if (o.bgr) *reinterpret_cast<uint3 *>(o.bgr + 3 * px) = make_uint3(un[0], un[1], un[2]);
  if (o.depth) *reinterpret_cast<uint2 *>(o.depth + px) = make_uint2(dep[0], dep[1]);
  if (o.label) *reinterpret_cast<unsigned *>(o.label + px) = lab;
}

// raster_init + raster_vertex + raster_coverage: the visibility buffer of every instance, for one resolve kernel
static int raster_front(dim_ctx *ctx, const RasterParams &p, int B, cudaStream_t st) {
  int maxV = 0, maxF = 0;
  for (auto &m : ctx->meshes_host) { maxV = maxV > m.V ? maxV : m.V; maxF = maxF > m.F ? maxF : m.F; }
  DIM_REQUIRE(maxV > 0 && maxF > 0, "dim_render: no mesh uploaded");
  raster_init_kernel<<<cdiv(B, 128), 128, 0, st>>>(ctx->vbox, ctx->bbox_ren, B, ctx->H, ctx->W);
  DIM_LAUNCH_CHECK();
  raster_vertex_kernel<<<dim3(cdiv(maxV, 256), B), 256, 0, st>>>(p);
  DIM_LAUNCH_CHECK();
  raster_coverage_kernel<<<dim3(cdiv(maxF, 128), B), 128, 0, st>>>(p);
  DIM_LAUNCH_CHECK();
  return 0;
}

int render_launch(dim_ctx *ctx, const int *cls, const float *pose, int B, const float *K9, float zn, float zf,
                  const double *means, int trunc_u8, float *out_image, float *out_depth, float *out_mask,
                  float *out_bgr, int *out_bbox, float4 *out_ren4, cudaStream_t st, const LitParams *lit, bool ren4_depth,
                  bool colour_box, const float *K_frames, const int32_t *frame_idx, int n_frames) {
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch, "dim_render: batch exceeds max_batch");
  DIM_REQUIRE((ctx->W & 3) == 0, "dim_render: width must be a multiple of 4");
  RasterParams p;
  p.meshes = ctx->meshes; p.cls = cls; p.pose = pose; p.pverts = ctx->pverts; p.vis = ctx->vis;
  p.vbox = ctx->vbox; p.bbox_ren = ctx->bbox_ren;
  p.max_verts = ctx->max_verts; p.max_faces = ctx->max_faces; p.H = ctx->H; p.W = ctx->W;
  p.num_classes = ctx->max_classes; p.cls_flag = ctx->cls_flag;
  p.fx = K9[0]; p.fy = K9[4]; p.cx = K9[2]; p.cy = K9[5]; p.zn = zn; p.zf = zf;
  p.K_frames = K_frames; p.frame_idx = frame_idx; p.n_frames = n_frames;
  for (int c = 0; c < 3; ++c) {
    p.mean[c] = means ? means[c] : 0.0;
    p.bg[c] = trunc_u8 ? (float)(0.0 - p.mean[c]) : 0.0f - (float)p.mean[c];
  }
  p.trunc_u8 = trunc_u8;
  p.out_image = out_image; p.out_depth = out_depth; p.out_mask = out_mask; p.out_bgr = out_bgr;
  p.out_ren4 = out_ren4;
  p.ren4_box_only = (out_ren4 && !out_image && !out_depth && !out_mask && !out_bgr) ? 1 : 0;
  p.lit = lit ? 1 : 0;
  p.light_pos = lit ? lit->light_pos : nullptr; p.light_int = lit ? lit->light_int : nullptr;
  p.a0 = lit ? lit->a0 : 0.f; p.a1 = lit ? lit->a1 : 0.f;
  if (int rc = raster_front(ctx, p, B, st)) return rc;
  const dim3 rgrid(cdiv((ctx->W / 4) * ctx->H, 256), B);
  DIM_REQUIRE(!(ren4_depth && colour_box), "dim_render: the colour bbox has no RGB-D variant");
  if (colour_box) {
    if (p.lit) raster_resolve_kernel<true, false, true><<<rgrid, 256, 0, st>>>(p);
    else raster_resolve_kernel<false, false, true><<<rgrid, 256, 0, st>>>(p);
  } else if (ren4_depth) {
    if (p.lit) raster_resolve_kernel<true, true><<<rgrid, 256, 0, st>>>(p);
    else raster_resolve_kernel<false, true><<<rgrid, 256, 0, st>>>(p);
  } else if (p.lit) {
    raster_resolve_kernel<true><<<rgrid, 256, 0, st>>>(p);
  } else {
    raster_resolve_kernel<false><<<rgrid, 256, 0, st>>>(p);
  }
  DIM_LAUNCH_CHECK();
  raster_finish_kernel<<<cdiv(B, 128), 128, 0, st>>>(ctx->bbox_ren, out_bbox, B);
  DIM_LAUNCH_CHECK();
  return 0;
}

int render_dataset_launch(dim_ctx *ctx, const int *cls, const float *pose, int B, const float *K9, float zn, float zf,
                          const float *light_pos, const float *light_int, const DatasetOut &o, cudaStream_t st) {
  DIM_REQUIRE(B >= 1 && B <= ctx->max_batch, "dim_render_dataset: batch exceeds max_batch");
  DIM_REQUIRE((ctx->W & 3) == 0, "dim_render_dataset: width must be a multiple of 4");
  RasterParams p = {};
  p.meshes = ctx->meshes; p.cls = cls; p.pose = pose; p.pverts = ctx->pverts; p.vis = ctx->vis;
  p.vbox = ctx->vbox; p.bbox_ren = ctx->bbox_ren;
  p.max_verts = ctx->max_verts; p.max_faces = ctx->max_faces; p.H = ctx->H; p.W = ctx->W;
  p.num_classes = ctx->max_classes; p.cls_flag = ctx->cls_flag;
  p.fx = K9[0]; p.fy = K9[4]; p.cx = K9[2]; p.cy = K9[5]; p.zn = zn; p.zf = zf;
  p.lit = o.lit_bgr ? 1 : 0;
  p.light_pos = light_pos; p.light_int = light_int;
  if (int rc = raster_front(ctx, p, B, st)) return rc;
  const dim3 rgrid(cdiv((ctx->W / 4) * ctx->H, 256), B);
  if (o.lit_bgr) raster_dataset_kernel<true><<<rgrid, 256, 0, st>>>(p, o);
  else raster_dataset_kernel<false><<<rgrid, 256, 0, st>>>(p, o);
  DIM_LAUNCH_CHECK();
  return 0;
}

}  // namespace dim
