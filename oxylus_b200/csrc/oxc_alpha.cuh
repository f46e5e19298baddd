// oxc_alpha.cuh — the alpha test of the vis-buffer encode (visbuffer_encode.slang:54-66) as pure per-thread functions:
// perspective-correct uv at a covered sample from the raster's own integer edge functions, one filtered alpha fetch, the
// comparison against the clamped cutoff; the uv-carrying clipper for triangles that take the clip path.
// No warp intrinsics, no shared memory: tests compile this source for the host.
// Specification: include/oxcull.h (comment above OxcMaterial) == oracle/oxc_oracle.c (comment above raster_triangle),
// operation for operation.
#pragma once
#include "oxc_shader_math.cuh"

namespace oxc {

// Device copy of one material, reduced to what the encode pass reads (scene.slang:51-66).
struct __align__(16) AlphaMaterial {
  const uint8_t* texels; // level 0 (the other levels follow, tightly packed); null: no albedo image (opaque for this pass)
  uint32_t width, height;
  uint32_t format;       // OxcImageFormat
  uint32_t levels;       // >= 1
  uint32_t mag_filter, min_filter, mipmap_mode;
  uint32_t address_u, address_v;
  float albedo_a;        // dequantize_half(albedo_color.w)
  float cutoff;          // the clamped cutoff: min(max(dequantize_half(alpha_cutoff), 0.001), 1.0); NaN stays NaN
  uint32_t pad[3];
};
static_assert(sizeof(AlphaMaterial) == 64, "AlphaMaterial");

// Per drawn triangle, in the raster's (a, b, c) order (TriSetup: a = vertex 0, b = vertex 2, c = vertex 1): 1 / w and uv.
struct AlphaTri {
  float rw[3];
  float u[3], v[3];
};

// clip-space vertices + uv of the triangle as submitted (vertex order 0, 1, 2) -> the raster's order
OXC_DI void alpha_tri_setup(const float4 c0, const float4 c1, const float4 c2, float u0, float v0, float u1, float v1, float u2, float v2,
                            AlphaTri& t) {
  t.rw[0] = fd(1.0f, c0.w); t.rw[1] = fd(1.0f, c2.w); t.rw[2] = fd(1.0f, c1.w); // the rw of to_screen (raster spec step 3)
  t.u[0] = u0; t.u[1] = u2; t.u[2] = u1;
  t.v[0] = v0; t.v[1] = v2; t.v[2] = v1;
}

OXC_DI uint32_t alpha_wrap(long long i, uint32_t n, uint32_t mode) {
  const long long N = (long long)n;
  if (mode == OXC_ADDRESS_CLAMP_TO_EDGE) return (uint32_t)(i < 0 ? 0 : (i > N - 1 ? N - 1 : i));
  if (mode == OXC_ADDRESS_MIRRORED_REPEAT) {
    long long r = i % (2 * N);
    if (r < 0) r += 2 * N;
    return (uint32_t)(r < N ? r : 2 * N - 1 - r);
  }
  long long r = i % N;
  if (r < 0) r += N;
  return (uint32_t)r;
}

OXC_DI float alpha_texel(const AlphaMaterial& m, const uint8_t* base, uint32_t w, uint32_t x, uint32_t y) {
  const size_t i = (size_t)y * w + x;
  const uint32_t t = m.format == OXC_IMAGE_R8_UNORM ? base[i] : base[i * 4 + 3];
  return fd((float)t, 255.0f);
}

// one level of the albedo image's alpha channel at (u, v) with one filter
OXC_DI float alpha_sample_level(const AlphaMaterial& m, uint32_t level, uint32_t filter, float u, float v) {
  const uint8_t* base = m.texels;
  uint32_t w = m.width, h = m.height;
  for (uint32_t l = 0; l < level; l++) { // levels are tightly packed one after the other
    base += (size_t)w * h * (m.format == OXC_IMAGE_R8_UNORM ? 1u : 4u);
    w = w > 1u ? w >> 1 : 1u;
    h = h > 1u ? h >> 1 : 1u;
  }
  const float fw = (float)w, fh = (float)h;
  if (filter == OXC_FILTER_NEAREST) {
    const int ix = sat_i32(floorf(fm(u, fw))), iy = sat_i32(floorf(fm(v, fh)));
    return alpha_texel(m, base, w, alpha_wrap(ix, w, m.address_u), alpha_wrap(iy, h, m.address_v));
  }
  const float x = fs(fm(u, fw), 0.5f), y = fs(fm(v, fh), 0.5f);
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = fs(x, x0), wy = fs(y, y0);
  const int ix = sat_i32(x0), iy = sat_i32(y0);
  const uint32_t xa = alpha_wrap(ix, w, m.address_u), xb = alpha_wrap((long long)ix + 1, w, m.address_u);
  const uint32_t ya = alpha_wrap(iy, h, m.address_v), yb = alpha_wrap((long long)iy + 1, h, m.address_v);
  const float a00 = alpha_texel(m, base, w, xa, ya), a10 = alpha_texel(m, base, w, xb, ya), a01 = alpha_texel(m, base, w, xa, yb),
              a11 = alpha_texel(m, base, w, xb, yb);
  const float top = fa(a00, fm(wx, fs(a10, a00))), bot = fa(a01, fm(wx, fs(a11, a01)));
  return fa(top, fm(wy, fs(bot, top)));
}

// uv from three edge-function values (weights of a, b, c; exact integers, >= 0 inside, sum = 2 * area > 0): perspective
// correction of non-negative terms only, so tiny and thin triangles interpolate without cancellation
OXC_DI void alpha_interpolate(const AlphaTri& t, long long e0, long long e1, long long e2, float& u, float& v) {
  const float p0 = fm((float)e0, t.rw[0]), p1 = fm((float)e1, t.rw[1]), p2 = fm((float)e2, t.rw[2]);
  const float inv = fd(1.0f, fa(fa(p0, p1), p2));
  const float l0 = fm(p0, inv), l1 = fm(p1, inv), l2 = fm(p2, inv);
  u = fa(fa(fm(l0, t.u[0]), fm(l1, t.u[1])), fm(l2, t.u[2]));
  v = fa(fa(fm(l0, t.v[0]), fm(l1, t.v[1])), fm(l2, t.v[2]));
}

// SampleGrad's level rule (oracle spec 4) from the texel-space derivatives mx = ddx(u) * width0, my = ddx(v) * height0, nx / ny
// likewise for ddy: the isotropic lambda with the canonical log2, lambda > 0 -> min filter, then the nearest level or the trilinear
// blend.  sample(level, filter) fetches one level.  alpha_keep below keeps its own written-out copy of this rule: calling the template
// changed the SASS of k_raster_alpha and of the shadow raster's kernels (DESIGN §4.6).
template <typename Sample>
OXC_DI auto sample_grad_levels(float mx, float my, float nx, float ny, uint32_t levels, uint32_t mag_filter, uint32_t min_filter,
                               uint32_t mipmap_mode, Sample sample) -> decltype(sample(0u, 0u)) {
  const float rx2 = fa(fm(mx, mx), fm(my, my)), ry2 = fa(fm(nx, nx), fm(ny, ny));
  const float r2 = rx2 > ry2 ? rx2 : ry2;
  const float lambda = fm(0.5f, canonical_log2(r2));
  const uint32_t filter = lambda > 0.0f ? min_filter : mag_filter;
  const uint32_t qi = levels > 1u ? levels - 1u : 0u;
  const float q = (float)qi;
  const float lc = !(lambda > 0.0f) ? 0.0f : (lambda > q ? q : lambda);
  if (mipmap_mode == OXC_MIPMAP_NEAREST) {
    uint32_t d = lc <= 0.5f ? 0u : (uint32_t)ceilf(fa(lc, 0.5f)) - 1u;
    d = d > qi ? qi : d;
    return sample(d, filter);
  }
  const uint32_t d = (uint32_t)floorf(lc), dn = d + 1u > qi ? qi : d + 1u;
  const float f = fs(lc, (float)d);
  const auto lo = sample(d, filter), hi = sample(dn, filter);
  return lerp_levels(f, lo, hi);
}

// alpha_keep is called from five places of k_raster_alpha (small / whole-warp / clipped paths); inlined everywhere the kernel was
// 27 k instructions.  One out-of-line copy keeps it at a size the instruction cache can hold; the call costs nothing next to the
// fetches.  (Host builds of this header — emulated library, tests — just inline it.)
#ifdef __CUDACC__
#define OXC_DNI __device__ __noinline__
#else
#define OXC_DNI inline
#endif

// true = the fragment at pixel (px, py) survives the alpha test (visbuffer_encode.slang:62-64 with the comparison negated).
// e0..e2 = the raster's edge-function values at the sample, ex / ey = their increments per pixel in x / y (from the TriSetup).
// Images with a mip chain (or different mag / min filters) select the level from the fine quad differences of uv (oracle spec 4).
OXC_DNI bool alpha_keep(const AlphaMaterial& m, const AlphaTri& t, int px, int py, long long e0, long long e1, long long e2, const long long ex[3],
                        const long long ey[3]) {
  float u, v, a;
  alpha_interpolate(t, e0, e1, e2, u, v);
  if (m.levels <= 1u && m.mag_filter == m.min_filter) {
    a = alpha_sample_level(m, 0u, m.min_filter, u, v); // nothing to select
  } else {
    const long long ox = -(long long)(px & 1), oy = -(long long)(py & 1); // to the quad's first column / row
    const long long a0 = e0 + ox * ex[0], a1 = e1 + ox * ex[1], a2 = e2 + ox * ex[2];
    const long long c0 = e0 + oy * ey[0], c1 = e1 + oy * ey[1], c2 = e2 + oy * ey[2];
    float uA, vA, uB, vB, uC, vC, uD, vD;
    alpha_interpolate(t, a0, a1, a2, uA, vA);
    alpha_interpolate(t, a0 + ex[0], a1 + ex[1], a2 + ex[2], uB, vB);
    alpha_interpolate(t, c0, c1, c2, uC, vC);
    alpha_interpolate(t, c0 + ey[0], c1 + ey[1], c2 + ey[2], uD, vD);
    const float w0 = (float)m.width, h0 = (float)m.height;
    const float mx = fm(fs(uB, uA), w0), my = fm(fs(vB, vA), h0), nx = fm(fs(uD, uC), w0), ny = fm(fs(vD, vC), h0);
    const float rx2 = fa(fm(mx, mx), fm(my, my)), ry2 = fa(fm(nx, nx), fm(ny, ny));
    const float r2 = rx2 > ry2 ? rx2 : ry2;
    const float lambda = fm(0.5f, canonical_log2(r2));
    const uint32_t filter = lambda > 0.0f ? m.min_filter : m.mag_filter;
    const uint32_t qi = m.levels > 1u ? m.levels - 1u : 0u;
    const float q = (float)qi;
    const float lc = !(lambda > 0.0f) ? 0.0f : (lambda > q ? q : lambda);
    if (m.mipmap_mode == OXC_MIPMAP_NEAREST) {
      uint32_t d = lc <= 0.5f ? 0u : (uint32_t)ceilf(fa(lc, 0.5f)) - 1u;
      d = d > qi ? qi : d;
      a = alpha_sample_level(m, d, filter, u, v);
    } else {
      const uint32_t d = (uint32_t)floorf(lc), dn = d + 1u > qi ? qi : d + 1u;
      const float f = fs(lc, (float)d);
      const float lo = alpha_sample_level(m, d, filter, u, v), hi = alpha_sample_level(m, dn, filter, u, v);
      a = fa(fm(fs(1.0f, f), lo), fm(f, hi));
    }
  }
  return !(fm(m.albedo_a, a) < m.cutoff);
}

// Sutherland-Hodgman of clip_polygon (oxc_raster_core.cuh) carrying uv: clip space is linear in the attributes, so a cut vertex
// gets uv_I + t * (uv_O - uv_I) with the position's t and operation order.  Same planes, same order, same inside rule.
struct ClipVertUV {
  float4 c;
  float u, v;
};
OXC_DI float clip_plane_distance_uv(const float4 v, int plane) {
  switch (plane) {
    case 0: return fs(v.w, v.z);
    case 1: return fa(v.w, v.x);
    case 2: return fs(v.w, v.x);
    case 3: return fa(v.w, v.y);
    default: return fs(v.w, v.y);
  }
}
OXC_DI int clip_polygon_uv(const ClipVertUV v0, const ClipVertUV v1, const ClipVertUV v2, ClipVertUV (*poly)[12], int& cur) {
  int n = 3;
  cur = 0;
  poly[0][0] = v0; poly[0][1] = v1; poly[0][2] = v2;
  for (int plane = 0; plane < 5 && n >= 3; plane++) {
    const ClipVertUV* in = poly[cur];
    ClipVertUV* out = poly[cur ^ 1];
    int m = 0;
    for (int i = 0; i < n; i++) {
      const ClipVertUV A = in[i], B = in[(i + 1) % n];
      const float dA = clip_plane_distance_uv(A.c, plane), dB = clip_plane_distance_uv(B.c, plane);
      const bool inA = dA >= 0.0f, inB = dB >= 0.0f;
      if (inA) out[m++] = A;
      if (inA != inB) {
        const ClipVertUV I = inA ? A : B, O = inA ? B : A;
        const float dI = inA ? dA : dB, dO = inA ? dB : dA;
        const float tt = fd(dI, fs(dI, dO));
        ClipVertUV r;
        r.c = make_float4(fa(I.c.x, fm(tt, fs(O.c.x, I.c.x))), fa(I.c.y, fm(tt, fs(O.c.y, I.c.y))), fa(I.c.z, fm(tt, fs(O.c.z, I.c.z))),
                          fa(I.c.w, fm(tt, fs(O.c.w, I.c.w))));
        r.u = fa(I.u, fm(tt, fs(O.u, I.u)));
        r.v = fa(I.v, fm(tt, fs(O.v, I.v)));
        out[m++] = r;
      }
    }
    n = m;
    cur ^= 1;
  }
  return n;
}

} // namespace oxc
