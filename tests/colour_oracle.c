/*
 * CPU checker of vertex-coloured meshes (TEST INFRASTRUCTURE): the renders of dim_render, dim_render_lit and
 * dim_render_dataset for a mesh uploaded with dim_mesh_upload_colours, on the oracle's own rasteriser.  The oracle is
 * compiled into this unit unchanged (it stays the textured path's checker); what is added is the colour source: the
 * perspective-correct interpolation of the winner triangle's vertex colours,
 *     c = ((w0 * cA + w1 * cB) + w2 * cC) / iz,  w_k = b_k * iz_k,
 * with A, B, C in the order orc_setup_tri uses them (B and C exchanged on a negatively oriented triangle), in float32, one
 * operation per line (built with -ffp-contract=off like the oracle).  c replaces the texel's texel / 255 everywhere:
 * unlit c * 255 (truncated to u8 on the test path), ModelNet and Py_Light shading, the dataset's (uint8)(c * 255).
 */
#include "../oracle/deepim_oracle.c"

enum { COL_UNLIT = 0, COL_MODELNET = 1, COL_PY_LIGHT = 2 };

/* the Lambert shading of orc_shade_lit (ModelNet) and pyl_shade (Py_Light) on the GL float colour tc */
static void col_shade(int shader, float b0, float b1, float b2, float iz, float izA, float izB, float izC, const float *vA,
                      const float *vB, const float *vC, const float *nA, const float *nB, const float *nC, const float *pose,
                      const float *light_pos, const float *light_int, float a0, float a1, const float *tc, float *rgb) {
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
  for (int c = 0; c < 3; ++c) {
    float col;
    if (shader == COL_MODELNET) {
      float scale = a0 + a1 * br;
      col = tc[c] * (scale * light_int[c]);
    } else {
      float diffuse = a1 * br;
      col = tc[c] * (a0 + diffuse * light_int[c]);
    }
    col = col < 1.f ? col : 1.f;
    col = col > 0.f ? col : 0.f;
    rgb[c] = rintf(col * 255.0f);
  }
}

/*
 * One instance of a coloured mesh (colours f32[V,3] RGB in [0,1]).  shader COL_UNLIT / COL_MODELNET fill the float
 * outputs of orc_render / orc_render_lit (out_bgr, out_depth, out_image, out_mask, bbox_ren); COL_PY_LIGHT is used only
 * with the u8 outputs.  The dataset outputs of pyl_render_dataset: u8_bgr = (uint8)(c * 255), u8_lit_bgr = the Py_Light
 * colour (with shader COL_PY_LIGHT), u16_depth = (uint16)(depth * depth_factor), label = depth != 0.  Every output may
 * be NULL; normals, light_pos and light_int are read only by a lit shader.
 */
ORC_API void col_render(const float *verts, const float *colours, const float *normals, int32_t V, const int32_t *faces,
                        int32_t F, const float *pose, const float *K4, float zn, float zf, int32_t H, int32_t W,
                        const double *means_rgb, int32_t trunc_u8, int32_t shader, const float *light_pos,
                        const float *light_int, float a0, float a1, float *out_bgr, float *out_depth, float *out_image,
                        float *out_mask, int32_t *bbox_ren, float depth_factor, uint8_t *u8_bgr, uint8_t *u8_lit_bgr,
                        uint16_t *u16_depth, uint8_t *label) {
  static const float no_uv[2] = {0.f, 0.f};
  orc_pvert *pv = (orc_pvert *)malloc(sizeof(orc_pvert) * (size_t)V);
  uint64_t *zb = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)H * W);
  for (size_t k = 0; k < (size_t)H * W; ++k) zb[k] = ~(uint64_t)0;
  for (int32_t v = 0; v < V; ++v) orc_project_vertex(pose, K4[0], K4[1], K4[2], K4[3], verts + 3 * v, no_uv, pv + v);
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
  int32_t bx0 = W, bx1 = -1, by0 = H, by1 = -1;
  const size_t P = (size_t)H * W;
  for (int32_t i = 0; i < H; ++i)
    for (int32_t j = 0; j < W; ++j) {
      size_t p = (size_t)i * W + j;
      uint64_t key = zb[p];
      float rgb[3] = {0.f, 0.f, 0.f}, lit[3] = {0.f, 0.f, 0.f}, tc[3] = {0.f, 0.f, 0.f}, depth = 0.f;
      if (key != ~(uint64_t)0) {
        int32_t f = (int32_t)(uint32_t)(key & 0xffffffffu);
        orc_tri t;
        orc_setup_tri(pv, faces + 3 * f, &t);
        float b0 = 0.f, b1 = 0.f, b2 = 0.f, iz = 1.f, z = 0.f;
        orc_fragment(&t, i, j, zn, zf, &b0, &b1, &b2, &iz, &z);
        const int32_t *fi = faces + 3 * f;
        const int32_t iA = fi[0], iB = t.swapped ? fi[2] : fi[1], iC = t.swapped ? fi[1] : fi[2];
        float w0 = b0 * t.a.iz, w1 = b1 * t.b.iz, w2 = b2 * t.c.iz;
        for (int c = 0; c < 3; ++c)
          tc[c] = ((w0 * colours[3 * iA + c] + w1 * colours[3 * iB + c]) + w2 * colours[3 * iC + c]) / iz;
        if (shader != COL_UNLIT)
          col_shade(shader, b0, b1, b2, iz, t.a.iz, t.b.iz, t.c.iz, verts + 3 * iA, verts + 3 * iB, verts + 3 * iC,
                    normals + 3 * iA, normals + 3 * iB, normals + 3 * iC, pose, light_pos, light_int, a0, a1, tc, lit);
        for (int c = 0; c < 3; ++c) {
          rgb[c] = tc[c] * 255.0f;
          if (trunc_u8) rgb[c] = (float)(uint8_t)rgb[c];
        }
        if (shader == COL_MODELNET)
          for (int c = 0; c < 3; ++c) rgb[c] = lit[c];
        depth = z;
      }
      float m = depth > 0.2f ? 1.f : 0.f;
      if (m > 0.f) {
        if (j < bx0) bx0 = j;
        if (j > bx1) bx1 = j;
        if (i < by0) by0 = i;
        if (i > by1) by1 = i;
      }
      for (int c = 0; c < 3; ++c) {
        if (out_bgr) out_bgr[3 * p + c] = rgb[2 - c];
        if (u8_bgr) u8_bgr[3 * p + c] = (uint8_t)(tc[2 - c] * 255.0f);
        if (u8_lit_bgr) u8_lit_bgr[3 * p + c] = (uint8_t)lit[2 - c];
      }
      if (out_depth) out_depth[p] = depth;
      if (out_image) {
        for (int c = 0; c < 3; ++c)
          out_image[c * P + p] = trunc_u8 ? (float)((double)rgb[c] - means_rgb[c]) : rgb[c] - (float)means_rgb[c];
      }
      if (out_mask) out_mask[p] = m;
      if (u16_depth) u16_depth[p] = (uint16_t)(depth * depth_factor);
      if (label) label[p] = depth != 0.f;
    }
  if (bbox_ren) {
    if (bx1 < 0) {
      bbox_ren[0] = bbox_ren[1] = bbox_ren[2] = bbox_ren[3] = -1;
    } else {
      bbox_ren[0] = bx0;
      bbox_ren[1] = bx1;
      bbox_ren[2] = by0;
      bbox_ren[3] = by1;
    }
  }
  free(pv);
  free(zb);
}
