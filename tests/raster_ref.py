"""Float64 reference of what the rasteriser is meant to draw (TEST INFRASTRUCTURE).

An independent definition of the renders of `dim_render`, `dim_render_lit` and `dim_render_dataset` (and of the oracle's
`orc_render`, `orc_render_lit` and `pyl_render_dataset`): a ray caster in float64 numpy.  It does not use the oracle and does
not restate its integer edge functions, snapping or float32 sequences.  Semantics, with the file each comes from:

- Projection (lib/render_glumpy/render_py_multi.py, `my_compute_calib_proj`: u0 = cx + 0.5, v0 = cy + 0.5, and the
  framebuffer's pixel centres at +0.5): pixel (i, j) samples image point (u, v) = (j, i).  The camera is fx, fy, cx, cy of
  a float32 K; the skew K[0, 1] is ignored, as the GL projection matrix ignores it.
- Vertices: the float32 pose and vertices, promoted to float64 (`_get_view_mtx`: view = yz-flip . [R | t]).
- Visibility: the nearest ray-triangle hit with zn <= z <= zf (GL_LESS depth test, the clip volume's near and far planes;
  GL_CULL_FACE is never enabled, so both windings draw).
- Depth: the hit's camera z (the GL depth linearisation of `render` inverts the projection).
- UV and texel: perspective-correct UV from the 3-D barycentrics of the hit; nearest texel floor(u Tw), floor(v Th) of
  `Mesh.tex` (row 0 = v 0), clamped to the texture.  Nearest, clamp-to-edge sampling is this project's documented
  convention (DESIGN.md, "Oracle pinning"); GL leaves the filter to the texture object.
- Unlit colour (render_py_multi.py `render`: the GL float texel c / 255, "* 255"): float32(c / 255) * 255, and
  with uint8 truncation on the test path (deepim/core/tester.py, `.astype(np.uint8)`).
- Lit colour, from the GLSL of render_py_light_modelnet_multi.py (ModelNet) and render_py_light.py (Py_Light):
  position in GL eye coordinates p = yz-flip . (R x + t); normal direction n = yz-flip . R n_model (see `_normal_gl`
  for the `u_normal * vec4(n, 1)` quirk); x and n_model are interpolated perspective-correctly (GL's default `smooth`
  varyings); brightness = clamp(dot(n, L - p) / (|L - p| |n|), 0, 1); ModelNet colour = t . ((a0 + a1 br) . I),
  Py_Light colour = t . (a0 + a1 br I), with t = texel / 255; the 8-bit framebuffer clamps to [0, 1] and stores
  round(255 c).
- Dropped triangles (this project's rule, a divergence from GL): a triangle with a vertex at camera z <= 1e-6 or a
  projected coordinate |u| or |v| > 1e6 px draws nothing.  GL would clip such a triangle at the near plane and draw its
  part between zn and zf.
- Exact ties: triangles with identical vertex positions have identical depths, and the lowest face index wins.

Tolerance rule, one for every output.  The device snaps each projected vertex to 1/256 px, which moves it by at most
1/512 px per axis, and the float32 projection adds a few ulp of the projected coordinate.  Every pixel is evaluated at
its centre and at the four centres shifted by +-eps in u and in v, with eps = 1/256 px + 2 ulp(float32 max |projected
coordinate|) of the triangle (the second term matters only for vertices far off screen).  A linear function over the
+-1/512 box takes its extremes at the corners, and |a| + |b| <= 2 max(|a|, |b|), so the five points bracket every value
the snapped triangle can produce at the pixel.
- Discrete outputs (covered or not, texel, u8 colour, u16 depth, label): where all five evaluations agree, the render
  must equal that value; elsewhere the pixel is ambiguous and excluded.
- Continuous outputs (float depth, the lit colour before rounding): the render must lie within [min, max] of the five
  evaluations, widened by 8 ulp of the depth, or by 0.5 + 1e-3 levels for the colour.
The u16 depth trunc(z . factor) is discrete, but the float32 depth it truncates carries its own rounding, so its five
evaluations are taken on the depth interval widened by the same 8 ulp.
"""
from __future__ import annotations

import warnings

import numpy as np

EPS_PX = 1.0 / 256.0
DEPTH_ULPS = 8
COLOUR_LEVELS = 0.5 + 1e-3
FLIP = np.array([1.0, -1.0, -1.0])  # OpenCV camera -> GL eye coordinates (y and z flipped), _get_view_mtx
# evaluation points: the pixel centre, then +-eps in u, then +-eps in v
SHIFTS = np.array([[0, 0], [1, 0], [-1, 0], [0, 1], [0, -1]], np.float64)
NE = len(SHIFTS)
_CHUNK = 1 << 21  # pixel samples per vectorised block


def camera(K):
    """fx, fy, cx, cy of the float32 K, as float64 (the skew is ignored)"""
    K = np.asarray(K, np.float32).astype(np.float64)
    return K[0, 0], K[1, 1], K[0, 2], K[1, 2]


def _normal_gl(R, n_model):
    """GL eye-space direction of a model normal.  The shader computes normalize(u_normal * vec4(n, 1)).xyz with
    u_normal = ((view . model)^-1)^T.  For view . model = [[R', t'], [0, 1]] (R' = flip . R), that inverse transpose is
    [[R', 0], [-(R'^T t')^T, 1]], so the product is (R' n, 1 - t'.R'n): its xyz is R' n, and normalising the 4-vector
    only scales it by a positive number, which the brightness divides out again with |n|."""
    return (n_model @ R.T) * FLIP


class Render:
    """The five evaluations of one instance, over the pixels `sel` (flat indices) that some evaluation hits: `face`
    [5, len(sel)] (-1 where nothing is hit), `z` (camera z, nan where nothing is hit), `lam` [5, len(sel), 3] (3-D
    barycentrics of the hit on the face's vertices, in the mesh's face order) and `z2` (the next strictly farther hit,
    inf where there is none).  `dropped` counts the triangles the drop rule removes."""

    def __init__(self, mesh, pose, K, H, W, zn=0.25, zf=6.0, normals=None):
        self.mesh, self.H, self.W, self.zn, self.zf = mesh, H, W, zn, zf
        pose = np.asarray(pose, np.float32).astype(np.float64)
        self.R, self.t = pose[:, :3], pose[:, 3]
        self.normals = normals
        self.fx, self.fy, self.cx, self.cy = camera(K)
        self._cast()

    # ---------------------------------------------------------------------------------------------------- visibility
    def _cast(self):
        m, H, W = self.mesh, self.H, self.W
        Pc = m.verts.astype(np.float64) @ self.R.T + self.t  # camera coordinates
        zc = Pc[:, 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            su = self.fx * Pc[:, 0] / zc + self.cx
            sv = self.fy * Pc[:, 1] / zc + self.cy
        ok = (zc > 1e-6) & (np.abs(su) <= 1e6) & (np.abs(sv) <= 1e6)
        f = m.faces
        keep = np.nonzero(ok[f].all(1))[0]
        self.dropped = len(f) - len(keep)
        fu, fv = su[f[keep]], sv[f[keep]]
        big = np.maximum(np.abs(fu).max(1), np.abs(fv).max(1)).astype(np.float32)
        eps = EPS_PX + 2.0 * np.spacing(big).astype(np.float64)
        j0 = np.maximum(np.ceil(fu.min(1) - eps), 0).astype(np.int64)
        j1 = np.minimum(np.floor(fu.max(1) + eps), W - 1).astype(np.int64)
        i0 = np.maximum(np.ceil(fv.min(1) - eps), 0).astype(np.int64)
        i1 = np.minimum(np.floor(fv.max(1) + eps), H - 1).astype(np.int64)
        on = (j1 >= j0) & (i1 >= i0)
        keep, eps, j0, j1, i0, i1 = keep[on], eps[on], j0[on], j1[on], i0[on], i1[on]
        A, B, C = Pc[f[keep, 0]], Pc[f[keep, 1]], Pc[f[keep, 2]]
        # the ray through image point (u, v) is s . d, d = ((u - cx) / fx, (v - cy) / fy, 1); the hit's barycentrics are
        # proportional to the triple products d.(B x C), d.(C x A), d.(A x B), and its z is det(A, B, C) / (d . normal)
        cr = np.stack([np.cross(B, C), np.cross(C, A), np.cross(A, B)], 1)  # [n,3 (vertex),3 (xyz)]
        self._Pc = Pc
        self._eps = np.zeros(len(f))
        self._eps[keep] = eps
        det = np.einsum("nk,nk->n", A, cr[:, 0])
        # group by padded box size so that each block is a dense [n, bh, bw] array
        bh, bw = _pad(i1 - i0 + 1), _pad(j1 - j0 + 1)
        frags = []
        for key in np.unique(bh * (1 << 20) + bw):
            g = np.nonzero(bh * (1 << 20) + bw == key)[0]
            gh, gw = int(key >> 20), int(key & ((1 << 20) - 1))
            step = max(1, _CHUNK // (gh * gw * NE))
            for s in range(0, len(g), step):
                frags.append(self._block(g[s:s + step], gh, gw, keep, eps, j0, j1, i0, i1, cr, det))
        pix = np.concatenate([a[0] for a in frags]) if frags else np.zeros(0, np.int64)
        fid = np.concatenate([a[1] for a in frags]) if frags else np.zeros(0, np.int64)
        z = np.concatenate([a[2] for a in frags]) if frags else np.zeros(0)
        lam = np.concatenate([a[3] for a in frags]) if frags else np.zeros((0, 3))
        # nearest hit per (evaluation, pixel); equal depths go to the lowest face index
        order = np.lexsort((fid, z, pix))
        ps, zs = pix[order], z[order]
        start = np.r_[True, ps[1:] != ps[:-1]] if len(order) else np.zeros(0, bool)
        first = order[start]
        # the next strictly farther hit: the winner is a comparison of two depths, each known only to its bracket
        zfirst = zs[np.flatnonzero(start)[np.cumsum(start) - 1]]
        far = zs > zfirst
        p2, i2 = np.unique(ps[far], return_index=True)
        z2 = zs[far][i2]
        # the outputs are kept for the pixels some evaluation hits: `sel` (flat pixel indices), then [5, len(sel)] arrays
        e, p = np.divmod(pix[first], H * W)
        self.sel = np.unique(p)
        k = np.searchsorted(self.sel, p)
        n = len(self.sel)
        self.face = np.full((NE, n), -1, np.int64)
        self.z = np.full((NE, n), np.nan)
        self.lam = np.zeros((NE, n, 3))
        self.face[e, k] = fid[first]
        self.z[e, k] = z[first]
        self.lam[e, k] = lam[first]
        self.z2 = np.full((NE, n), np.inf)
        e2, q2 = np.divmod(p2, H * W)
        self.z2[e2, np.searchsorted(self.sel, q2)] = z2

    def _block(self, g, gh, gw, keep, eps, j0, j1, i0, i1, cr, det):
        ii = i0[g, None, None] + np.arange(gh)[None, :, None]
        jj = j0[g, None, None] + np.arange(gw)[None, None, :]
        inbox = (ii <= i1[g, None, None]) & (jj <= j1[g, None, None])
        n = len(g)
        ii = np.broadcast_to(ii, (n, gh, gw))[inbox]
        jj = np.broadcast_to(jj, (n, gh, gw))[inbox]
        tri = np.broadcast_to(np.arange(n)[:, None, None], (n, gh, gw))[inbox]
        crt, dett, epst = cr[g][tri], det[g][tri], eps[g][tri]
        out = []
        for e in range(NE):
            u = jj + SHIFTS[e, 0] * epst
            v = ii + SHIFTS[e, 1] * epst
            d = np.stack([(u - self.cx) / self.fx, (v - self.cy) / self.fy, np.ones_like(u)], -1)
            t3 = np.einsum("pk,pvk->pv", d, crt)
            inside = (t3 > 0).all(1) | (t3 < 0).all(1)
            ssum = t3.sum(1)
            with np.errstate(divide="ignore", invalid="ignore"):
                z = dett / ssum
            hit = inside & (z >= self.zn) & (z <= self.zf)
            pix = (e * self.H + ii[hit]) * self.W + jj[hit]
            out.append((pix, keep[g][tri[hit]], z[hit], t3[hit] / ssum[hit, None]))
        return tuple(np.concatenate([o[k] for o in out]) for k in range(4))

    def plane_z(self, face):
        """[5, len(sel)] camera z of the plane of triangle face[k] through pixel sel[k]'s five evaluation points (nan where
        face < 0): a hidden part of a winning triangle still bounds the depth it can show at the pixel"""
        f = self.mesh.faces[np.maximum(face, 0)]
        A, B, C = self._Pc[f[:, 0]], self._Pc[f[:, 1]], self._Pc[f[:, 2]]
        n = np.cross(B - A, C - A)
        eps = self._eps[np.maximum(face, 0)]
        i, j = np.divmod(self.sel, self.W)
        out = np.empty((NE, len(face)))
        for e in range(NE):
            u, v = j + SHIFTS[e, 0] * eps, i + SHIFTS[e, 1] * eps
            den = n[:, 0] * (u - self.cx) / self.fx + n[:, 1] * (v - self.cy) / self.fy + n[:, 2]
            with np.errstate(divide="ignore", invalid="ignore"):
                out[e] = np.where(face >= 0, np.einsum("nk,nk->n", n, A) / den, np.nan)
        return out

    # ------------------------------------------------------------------------------------------------------- outputs
    # Every output below is [5, len(sel), ...] over the pixels `sel`.
    @property
    def covered(self):
        return self.face >= 0

    def _interp(self, attr):
        """perspective-correct interpolation of a per-vertex attribute [V,k] at every hit (0 where nothing is hit)"""
        a = attr.astype(np.float64)[self.mesh.faces[np.maximum(self.face, 0)]]  # [5,n,3,k]
        return np.einsum("env,envk->enk", self.lam, a) * self.covered[..., None]

    def uv(self):
        return self._interp(self.mesh.uvs)

    def texel_xy(self):
        """texel column and row of every hit, floor(u Tw) and floor(v Th) clamped to the texture"""
        Th, Tw = self.mesh.tex.shape[:2]
        uv = self.uv()
        tx = np.clip(np.floor(uv[..., 0] * Tw), 0, Tw - 1).astype(np.int64)
        ty = np.clip(np.floor(uv[..., 1] * Th), 0, Th - 1).astype(np.int64)
        return tx, ty

    def texel(self):
        """flat texel index ty * Tw + tx (-1 where nothing is hit)"""
        tx, ty = self.texel_xy()
        return np.where(self.covered, ty * self.mesh.tex.shape[1] + tx, -1)

    def unlit_bgr(self, trunc_u8=True):
        """BGR of the unlit render: float32(c / 255) * 255, truncated to uint8 on the test path (0 where nothing is hit)"""
        lut = (np.arange(256, dtype=np.float32) / np.float32(255.0)) * np.float32(255.0)
        if trunc_u8:
            lut = lut.astype(np.uint8).astype(np.float32)
        tex = lut[self.mesh.tex.reshape(-1, 3)][:, ::-1].astype(np.float64)
        t = self.texel()
        return tex[np.maximum(t, 0)] * (t >= 0)[..., None]

    def brightness(self, light_pos):
        """the Lambert term clamp(cos(n, L - p), 0, 1) in GL eye coordinates (light_pos in that frame)"""
        assert self.normals is not None, "the lit render needs per-vertex normals"
        p = (self._interp(self.mesh.verts) @ self.R.T + self.t) * FLIP
        n = _normal_gl(self.R, self._interp(self.normals))
        s = np.asarray(light_pos, np.float32).astype(np.float64) - p
        den = np.linalg.norm(s, axis=-1) * np.linalg.norm(n, axis=-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            br = np.where(den > 0, np.einsum("...k,...k->...", n, s) / den, 0.0)
        return np.clip(br, 0.0, 1.0)

    def lit_bounds(self, light_pos, light_int, ratio, shader, span=4):
        """lowest and highest BGR framebuffer level 255 c the lit render can take before rounding, [len(sel), 3] each,
        and the pixels where they hold.  shader "modelnet": c = t . ((a0 + a1 br) I); "py_light": c = t . (a0 + a1 br I);
        a1 = float32 ratio, a0 = float32(1 - a1), as the renderers take them.  c grows with the texel value t and with the
        brightness br, so its bounds are those of t over every texel between the evaluations' (a rectangle of at most
        span x span texels; wider ones are left unchecked) times those of the light factor over the five brightnesses."""
        a1 = float(np.float32(ratio))
        a0 = float(np.float32(1.0 - np.float32(ratio)))
        I = np.asarray(light_int, np.float32).astype(np.float64)
        br = self.brightness(light_pos)
        cov = self.covered
        brlo = np.where(cov, br, np.inf).min(0)[:, None]
        brhi = np.where(cov, br, -np.inf).max(0)[:, None]
        glo, ghi = ((a0 + a1 * brlo) * I, (a0 + a1 * brhi) * I) if shader == "modelnet" else \
            (a0 + a1 * brlo * I, a0 + a1 * brhi * I)
        tx, ty = self.texel_xy()
        big = np.iinfo(np.int64).max
        x0, x1 = np.where(cov, tx, big).min(0), np.where(cov, tx, -1).max(0)
        y0, y1 = np.where(cov, ty, big).min(0), np.where(cov, ty, -1).max(0)
        ok = cov.any(0) & (x1 - x0 < span) & (y1 - y0 < span)
        Tw = self.mesh.tex.shape[1]
        tex = self.mesh.tex.reshape(-1, 3).astype(np.float64) / 255.0
        tlo, thi = np.full((len(ok), 3), np.inf), np.full((len(ok), 3), -np.inf)
        for a in range(span):
            for b in range(span):
                m = ok & (y0 + a <= y1) & (x0 + b <= x1)
                v = tex[np.where(m, (y0 + a) * Tw + x0 + b, 0)]
                tlo = np.where(m[:, None], np.minimum(tlo, v), tlo)
                thi = np.where(m[:, None], np.maximum(thi, v), thi)
        lo = np.clip(tlo * glo, 0.0, 1.0) * 255.0
        hi = np.clip(thi * ghi, 0.0, 1.0) * 255.0
        return lo[:, ::-1], hi[:, ::-1], ok

    def lit_levels(self, light_pos, light_int, ratio, shader):
        """[5, len(sel), 3] BGR level 255 c of each evaluation, with its own texel and brightness"""
        a1 = float(np.float32(ratio))
        a0 = float(np.float32(1.0 - np.float32(ratio)))
        br = self.brightness(light_pos)[..., None]
        I = np.asarray(light_int, np.float32).astype(np.float64)
        tex = self.mesh.tex.reshape(-1, 3).astype(np.float64) / 255.0
        t = self.texel()
        t = tex[np.maximum(t, 0)] * (t >= 0)[..., None]
        c = t * ((a0 + a1 * br) * I) if shader == "modelnet" else t * (a0 + a1 * br * I)
        return (np.clip(c, 0.0, 1.0) * 255.0)[..., ::-1]


def _pad(n):
    """box extents rounded up to 1, 2, 3, 4, 6, 8, 12, 16, ...: a few dense block shapes with little waste"""
    p = np.maximum(2 ** np.ceil(np.log2(np.maximum(n, 1))), 1).astype(np.int64)
    three = (p // 4) * 3
    return np.where((p >= 4) & (n <= three), three, p)


# ------------------------------------------------------------------------------------------------------------ checks
def unanimous(vals):
    """vals [5,...]: mask where all five evaluations agree (trailing channel axes must agree as a whole)"""
    same = np.ones(vals.shape[1:], bool)
    for e in range(1, NE):
        same &= vals[e] == vals[0]
    return same


class Report:
    """Per-render tally: ambiguous pixels, mismatches and the largest ratios of error to bound."""

    def __init__(self, name):
        self.name = name
        self.ambiguous = 0
        self.mismatch = {}
        self.ratio = {}

    def bad(self, what, n):
        self.mismatch[what] = self.mismatch.get(what, 0) + int(n)

    def worst(self, what, r):
        if np.size(r):
            self.ratio[what] = max(self.ratio.get(what, 0.0), float(np.max(r)))

    @property
    def ok(self):
        return not any(self.mismatch.values()) and all(r <= 1.0 for r in self.ratio.values())

    def __str__(self):
        rs = " ".join("%s %.3f" % kv for kv in sorted(self.ratio.items()))
        ms = " ".join("%s %d" % kv for kv in sorted(self.mismatch.items()) if kv[1])
        return "%-28s ambiguous: coverage %6d crossing %5d lit texel %4d  ratio %s%s" % (
            self.name, self.ambiguous, getattr(self, "crossing", 0), getattr(self, "ambiguous_lit", 0), rs,
            ("  MISMATCH " + ms) if ms else "")


def _ratio(got, lo, hi, centre):
    """position of got in the bound: 0 at the centre evaluation, 1 at the widened end of the interval on its side"""
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(got >= centre, (got - centre) / (hi - centre), (centre - got) / (centre - lo))
    return np.where(got == centre, 0.0, np.nan_to_num(r, nan=np.inf))


def _depth_interval(ref):
    """the depth bracket of every pixel: every triangle that wins one of the five evaluations, at all five points"""
    zs = np.concatenate([ref.plane_z(ref.face[e]) for e in range(NE)])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)  # all-nan columns: pixels no evaluation covers
        lo, hi = np.nanmin(zs, 0), np.nanmax(zs, 0)
    ulp = np.spacing(np.abs(hi).astype(np.float32)).astype(np.float64)
    return lo - DEPTH_ULPS * ulp, hi + DEPTH_ULPS * ulp


def clear_winner(ref):
    """pixels whose winning surface is decided: the next strictly farther hit of every evaluation lies beyond the
    nearest one's widened depth bracket.  Where two surfaces cross, the device's float32 depths decide between them, and
    the crossing line moves with both triangles' snapping; such pixels are ambiguous like those on an edge.  Exact ties
    (identical vertex positions) are not ambiguous: both depths are the same bits and the lowest face index wins."""
    lo, hi = _depth_interval(ref)
    z2 = ref.z2.min(0)
    ulp = np.spacing(np.abs(np.minimum(z2, 1e30)).astype(np.float32)).astype(np.float64)
    return ~(z2 - DEPTH_ULPS * ulp <= hi)


def check_render(rep, ref, depth, mask=None, bgr=None, trunc_u8=True, label=False):
    """one render's float32 depth [H,W] (0 off the object; with label=True a 0 / 1 label instead, checked for coverage
    only), and optionally its mask and unlit BGR, against the reference.  Pixels no evaluation hits must be background."""
    flat = depth.reshape(-1)
    rest = np.ones(flat.shape, bool)
    rest[ref.sel] = False
    rep.bad("coverage", (flat[rest] != 0).sum())
    d = flat[ref.sel].astype(np.float64)
    cov = ref.covered
    agree = unanimous(cov)
    rep.ambiguous += int((~agree).sum())
    rep.crossing = getattr(rep, "crossing", 0) + int((agree & cov[0] & ~clear_winner(ref)).sum())
    on, off = agree & cov[0] & clear_winner(ref), agree & ~cov[0]
    rep.bad("coverage", ((d != 0) != cov[0])[agree].sum())
    if not label:
        lo, hi = _depth_interval(ref)
        ok = on & (d != 0)
        rep.worst("depth", _ratio(d[ok], lo[ok], hi[ok], ref.z[0][ok]))
    if mask is not None:
        mk = mask.reshape(-1)
        rep.bad("mask", (mk[rest] != 0).sum() + (mk[ref.sel] != (cov[0] & (ref.z[0] > 0.2)))[agree].sum())
    if bgr is not None:
        c = bgr.reshape(-1, 3)
        rep.bad("background", (c[rest] != 0).any(-1).sum())
        c = c[ref.sel]
        want = ref.unlit_bgr(trunc_u8)[0]
        sure = on & unanimous(ref.texel())
        rep.bad("texel", (c != want).any(-1)[sure].sum())
        rep.bad("background", (c != 0).any(-1)[off].sum())


def check_u16(rep, ref, depth_u16, label, factor):
    """the dataset's u16 depth trunc(z . factor) and label depth != 0"""
    rest = np.ones(depth_u16.size, bool)
    rest[ref.sel] = False
    du, lb = depth_u16.reshape(-1), label.reshape(-1)
    rep.bad("u16 depth", (du[rest] != 0).sum())
    rep.bad("label", (lb[rest] != 0).sum())
    du, lb = du[ref.sel].astype(np.float64), lb[ref.sel]
    cov = ref.covered
    agree = unanimous(cov)
    lo, hi = _depth_interval(ref)
    qlo, qhi = np.trunc(np.nan_to_num(lo) * factor), np.trunc(np.nan_to_num(hi) * factor)
    sure = agree & (qlo == qhi) & (clear_winner(ref) | ~cov[0])
    rep.bad("u16 depth", (du != np.where(cov[0], qlo, 0))[sure].sum())
    rep.bad("label", (lb != cov[0])[agree].sum())


def check_lit(rep, ref, bgr, light_pos, light_int, ratio, shader):
    """a lit render's u8-valued BGR [H,W,3] against the bounds of its level before rounding, widened by 0.5 + 1e-3"""
    c = bgr.reshape(-1, 3)
    rest = np.ones(len(c), bool)
    rest[ref.sel] = False
    rep.bad("lit background", (c[rest] != 0).any(-1).sum())
    c = c[ref.sel].astype(np.float64)
    cov = ref.covered
    agree = unanimous(cov)
    lo, hi, ok = ref.lit_bounds(light_pos, light_int, ratio, shader)
    centre = ref.lit_levels(light_pos, light_int, ratio, shader)[0]
    on = agree & cov[0] & ok & clear_winner(ref)
    rep.ambiguous_lit = getattr(rep, "ambiguous_lit", 0) + int((agree & cov[0] & ~ok).sum())
    r = _ratio(c, lo - COLOUR_LEVELS, hi + COLOUR_LEVELS, np.clip(centre, lo, hi))
    rep.worst("lit", r[on])
    rep.bad("lit background", (c != 0).any(-1)[agree & ~cov[0]].sum())
