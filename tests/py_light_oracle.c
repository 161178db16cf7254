/*
 * CPU checker of dim_render_dataset (TEST INFRASTRUCTURE): the data-preparation render of toolkit/LM6d_ds_1, ds_2, ds_4 and
 * LM6d_0_gen_gt_observed.py on the oracle's own rasteriser.  The oracle is compiled into this unit unchanged; what is
 * added is the Render_Py_Light shading (lib/render_glumpy/render_py_light.py get_fragment) and the conversions of the
 * dataset files, both in float32, one operation per line (built with -ffp-contract=off like the oracle).
 */
#include "../oracle/deepim_oracle.c"

/* orc_shade_lit's Lambert term, with the light colour on the diffuse part only:
 * colour = texel * (a0 + (a1 * brightness) * light_intensity), a0 = 1 - ratio, a1 = ratio. */
static void pyl_shade(float b0, float b1, float b2, float iz, float izA, float izB, float izC, const float *vA,
                      const float *vB, const float *vC, const float *nA, const float *nB, const float *nC, const float *pose,
                      const float *light_pos, const float *light_int, float a0, float a1, const uint8_t *tp, float *rgb) {
  float w0 = b0 * izA, w1 = b1 * izB, w2 = b2 * izC;
  float pm[3], nm[3], pc[3], nc[3];
  for (int k = 0; k < 3; ++k) {
    pm[k] = ((w0 * vA[k] + w1 * vB[k]) + w2 * vC[k]) / iz;
    nm[k] = ((w0 * nA[k] + w1 * nB[k]) + w2 * nC[k]) / iz;
  }
  for (int r = 0; r < 3; ++r) {
    pc[r] = ((pose[4 * r] * pm[0] + pose[4 * r + 1] * pm[1]) + pose[4 * r + 2] * pm[2]) + pose[4 * r + 3];
    nc[r] = (pose[4 * r] * nm[0] + pose[4 * r + 1] * nm[1]) + pose[4 * r + 2] * nm[2];
  }
  float s0 = light_pos[0] - pc[0], s1 = light_pos[1] - (0.f - pc[1]), s2 = light_pos[2] - (0.f - pc[2]);
  float g0 = nc[0], g1 = 0.f - nc[1], g2 = 0.f - nc[2];
  float dot = (g0 * s0 + g1 * s1) + g2 * s2;
  float ls = sqrtf((s0 * s0 + s1 * s1) + s2 * s2), ln = sqrtf((g0 * g0 + g1 * g1) + g2 * g2);
  float den = ls * ln, br = 0.f;
  if (den > 0.f) br = dot / den;
  br = br < 1.f ? br : 1.f;
  br = br > 0.f ? br : 0.f;
  float diffuse = a1 * br;
  for (int c = 0; c < 3; ++c) {
    float col = ((float)tp[c] / 255.0f) * (a0 + diffuse * light_int[c]);
    col = col < 1.f ? col : 1.f;
    col = col > 0.f ? col : 0.f;
    rgb[c] = rintf(col * 255.0f);
  }
}

/* One instance, as the dataset files hold it:
 *  out_lit_bgr : [H,W,3] u8  Render_Py_Light colour (needs normals, light_pos, light_int; may be NULL)
 *  out_bgr     : [H,W,3] u8  Render_Py colour .astype('uint8')
 *  out_depth   : [H,W]   u16 (depth * depth_factor).astype(np.uint16) on the float32 depth
 *  out_label   : [H,W]   u8  depth != 0
 * Visibility, fragment and texel lookup are the oracle's (orc_render_impl). */
ORC_API void pyl_render_dataset(const float *verts, const float *uvs, const float *normals, int32_t V, const int32_t *faces,
                                int32_t F, const uint8_t *tex, int32_t Th, int32_t Tw, const float *pose, const float *K4,
                                float zn, float zf, int32_t H, int32_t W, const float *light_pos, const float *light_int,
                                float ratio, float depth_factor, uint8_t *out_lit_bgr, uint8_t *out_bgr, uint16_t *out_depth,
                                uint8_t *out_label) {
  orc_pvert *pv = (orc_pvert *)malloc(sizeof(orc_pvert) * (size_t)V);
  uint64_t *zb = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)H * W);
  for (size_t k = 0; k < (size_t)H * W; ++k) zb[k] = ~(uint64_t)0;
  for (int32_t v = 0; v < V; ++v) orc_project_vertex(pose, K4[0], K4[1], K4[2], K4[3], verts + 3 * v, uvs + 2 * v, pv + v);
  for (int32_t f = 0; f < F; ++f) {
    orc_tri t;
    orc_setup_tri(pv, faces + 3 * f, &t);
    if (!t.valid) continue;
    int32_t minX = t.a.X < t.b.X ? t.a.X : t.b.X;
    if (t.c.X < minX) minX = t.c.X;
    int32_t maxX = t.a.X > t.b.X ? t.a.X : t.b.X;
    if (t.c.X > maxX) maxX = t.c.X;
    int32_t minY = t.a.Y < t.b.Y ? t.a.Y : t.b.Y;
    if (t.c.Y < minY) minY = t.c.Y;
    int32_t maxY = t.a.Y > t.b.Y ? t.a.Y : t.b.Y;
    if (t.c.Y > maxY) maxY = t.c.Y;
    int32_t j0 = (minX + 255) >> 8, j1 = maxX >> 8, i0 = (minY + 255) >> 8, i1 = maxY >> 8;
    if (j0 < 0) j0 = 0;
    if (i0 < 0) i0 = 0;
    if (j1 > W - 1) j1 = W - 1;
    if (i1 > H - 1) i1 = H - 1;
    for (int32_t i = i0; i <= i1; ++i)
      for (int32_t j = j0; j <= j1; ++j) {
        float b0, b1, b2, iz, z;
        if (!orc_fragment(&t, i, j, zn, zf, &b0, &b1, &b2, &iz, &z)) continue;
        uint64_t key = ((uint64_t)orc_fbits(z) << 32) | (uint32_t)f;
        if (key < zb[(size_t)i * W + j]) zb[(size_t)i * W + j] = key;
      }
  }
  const float a1 = ratio, a0 = 1.f - ratio;
  for (int32_t i = 0; i < H; ++i)
    for (int32_t j = 0; j < W; ++j) {
      size_t p = (size_t)i * W + j;
      uint64_t key = zb[p];
      float lit[3] = {0.f, 0.f, 0.f}, un[3] = {0.f, 0.f, 0.f}, depth = 0.f;
      if (key != ~(uint64_t)0) {
        int32_t f = (int32_t)(uint32_t)(key & 0xffffffffu);
        orc_tri t;
        orc_setup_tri(pv, faces + 3 * f, &t);
        float b0 = 0.f, b1 = 0.f, b2 = 0.f, iz = 1.f, z = 0.f;
        orc_fragment(&t, i, j, zn, zf, &b0, &b1, &b2, &iz, &z);
        float un_ = (b0 * t.a.uz + b1 * t.b.uz) + b2 * t.c.uz;
        float vn_ = (b0 * t.a.vz + b1 * t.b.vz) + b2 * t.c.vz;
        float u = un_ / iz, v = vn_ / iz;
        int32_t tx = (int32_t)floorf(u * (float)Tw), ty = (int32_t)floorf(v * (float)Th);
        if (tx < 0) tx = 0;
        if (tx > Tw - 1) tx = Tw - 1;
        if (ty < 0) ty = 0;
        if (ty > Th - 1) ty = Th - 1;
        const uint8_t *tp = tex + ((size_t)ty * Tw + tx) * 3;
        for (int c = 0; c < 3; ++c) un[c] = orc_colour(tp[c], 0);
        if (out_lit_bgr) {
          const int32_t *fi = faces + 3 * f;
          const int32_t iA = fi[0], iB = t.swapped ? fi[2] : fi[1], iC = t.swapped ? fi[1] : fi[2];
          pyl_shade(b0, b1, b2, iz, t.a.iz, t.b.iz, t.c.iz, verts + 3 * iA, verts + 3 * iB, verts + 3 * iC, normals + 3 * iA,
                    normals + 3 * iB, normals + 3 * iC, pose, light_pos, light_int, a0, a1, tp, lit);
        }
        depth = z;
      }
      for (int c = 0; c < 3; ++c) {
        if (out_bgr) out_bgr[3 * p + c] = (uint8_t)un[2 - c];
        if (out_lit_bgr) out_lit_bgr[3 * p + c] = (uint8_t)lit[2 - c];
      }
      if (out_depth) out_depth[p] = (uint16_t)(depth * depth_factor);
      if (out_label) out_label[p] = depth != 0.f;
    }
  free(pv);
  free(zb);
}
