// oxc_contact_shadows.cuh — the contact shadow of one pixel (passes/contact_shadows.slang:29-78 with the raymarch.slang DepthRayMarch,
// HybridRootFinder and DepthRaymarchDistanceFn code it calls, on the path that call site takes: linear steps, jitter 1, exponent 1, no
// bisection, no secant step, march_behind_surfaces false) as pure per-thread functions: unproject, ray set-up and frustum clip, the
// linear march over the depth plane's bilinear and nearest taps, the contact decision.
// No warp intrinsics, no shared memory: tests compile this source for the host.
// Specification: include/oxcull.h (comment above oxc_contact_shadows) == oracle/oxc_oracle_contact_shadows.c, operation for operation.
#pragma once
#include "oxc_gtao.cuh" // alpha_f2i, gtao_clamp

namespace oxc {

struct ContactShadowParams {
  const float* depth;
  float* out;
  int width, height;
  float4 inv_pv_row[4];     // rows of Camera::inv_projection_view
  float4 view_row[4];       // rows of Camera::view
  float4 proj_row[4];       // rows of Camera::projection
  float near_clip;
  float sun[3];             // as given; normalized by cs_constants
  float thickness, length;
  uint32_t steps;           // 1..OXC_CONTACT_SHADOW_MAX_STEPS
};

// the kernel's parameters from the C ABI's arguments (oxc_contact_shadows, and the host build of the tests)
__host__ inline ContactShadowParams cs_make_params(const OxcContactShadowCamera& cam, const OxcContactShadowSettings& st, const float* depth,
                                                   uint32_t w, uint32_t h, float* out) {
  ContactShadowParams p{};
  p.depth = depth; p.out = out; p.width = (int)w; p.height = (int)h;
  for (int i = 0; i < 4; i++) {
    p.inv_pv_row[i] = make_float4(cam.inv_projection_view[i], cam.inv_projection_view[4 + i], cam.inv_projection_view[8 + i],
                                  cam.inv_projection_view[12 + i]);
    p.view_row[i] = make_float4(cam.view[i], cam.view[4 + i], cam.view[8 + i], cam.view[12 + i]);
    p.proj_row[i] = make_float4(cam.projection[i], cam.projection[4 + i], cam.projection[8 + i], cam.projection[12 + i]);
  }
  p.near_clip = cam.near_clip;
  for (int i = 0; i < 3; i++) p.sun[i] = st.sun_direction[i];
  p.thickness = st.thickness; p.length = st.length; p.steps = st.steps;
  return p;
}

// the per-pass values every pixel derives from the settings: normalize(sun_dir) (contact_shadows.slang:60) and depth_thickness =
// thickness * (1 / near_clip) (:57, raymarch.slang:597-598).  One function, so the bits do not depend on where they are computed.
struct ContactShadowConstants {
  float dir[3];
  float depth_thickness;
};
OXC_DI ContactShadowConstants cs_constants(const ContactShadowParams& p) {
  ContactShadowConstants c;
  const float l = fsq(dot3(p.sun[0], p.sun[1], p.sun[2], p.sun[0], p.sun[1], p.sun[2]));
  c.dir[0] = fd(p.sun[0], l); c.dir[1] = fd(p.sun[1], l); c.dir[2] = fd(p.sun[2], l);
  c.depth_thickness = fm(p.thickness, fd(1.0f, p.near_clip));
  return c;
}

OXC_DI float cs_sign(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }
OXC_DI uint32_t cs_u32(float f) { return !(f > 0.0f) ? 0u : (f >= 4294967296.0f ? 0xFFFFFFFFu : (uint32_t)f); }
OXC_DI float cs_to_uv(float c) { return fa(fm(c, 0.5f), 0.5f); } // raymarch.slang:15-17

// SampleLevel(linear_clamp, uv, 0) of the depth plane, in two parts so that the nearest tap can pick among the four texels: the
// texel columns / rows and binary32 weights at uv * size - 0.5, then the blend.  The arithmetic is oxc_gtao.cuh gtao_bilinear's, written
// out again: making gtao_bilinear call these two functions changes k_gtao_main's SASS (2296 -> 2440 instructions for sm_90a).
struct BilinearTap {
  int xa, xb, ya, yb;
  float wx, wy;
};
OXC_DI BilinearTap cs_bilinear_tap(int w, int h, float u, float v) {
  const float x = fs(fm(u, (float)w), 0.5f), y = fs(fm(v, (float)h), 0.5f);
  const float x0 = floorf(x), y0 = floorf(y);
  BilinearTap t;
  t.wx = fs(x, x0); t.wy = fs(y, y0);
  const long long ix = alpha_f2i(x0), iy = alpha_f2i(y0);
  t.xa = gtao_clamp(ix, w); t.xb = gtao_clamp(ix + 1, w); t.ya = gtao_clamp(iy, h); t.yb = gtao_clamp(iy + 1, h);
  return t;
}
OXC_DI float cs_bilinear_blend(const BilinearTap& t, float a00, float a10, float a01, float a11) {
  const float top = fa(a00, fm(t.wx, fs(a10, a00))), bot = fa(a01, fm(t.wx, fs(a11, a01)));
  return fa(top, fm(t.wy, fs(bot, top)));
}

// SampleLevel(nearest_clamp, uv, 0): texel column floor(u * W) (row likewise), NaN-safe saturating, clamped to the edge
OXC_DI int cs_nearest_index(float u, int n) { return gtao_clamp(alpha_f2i(floorf(fm(u, (float)n))), n); }

// DepthRaymarchDistanceFn::call (raymarch.slang:254-322): the bilinear and the nearest tap at the point's uv.  The nearest texel is
// always one of the bilinear tap's four: with a = fl(u * W), x = fl(a - 0.5) is a - 0.5 exactly below 2^23 and a or a - 1 above, so
// floor(a) is floor(x) or floor(x) + 1, and the saturating index and the clamp keep that (NaN gives 0 in both, +-Inf the same edge).
// It is picked from the four loaded values instead of being loaded again.
OXC_DI void cs_distance(const ContactShadowParams& p, float px, float py, float pz, float& distance, float& penetration) {
  const float u = cs_to_uv(px), v = cs_to_uv(py);
  const float ray_depth = fd(1.0f, pz);
  const int w = p.width;
  const BilinearTap t = cs_bilinear_tap(w, p.height, u, v);
  const float a00 = __ldg(&p.depth[(size_t)t.ya * w + t.xa]), a10 = __ldg(&p.depth[(size_t)t.ya * w + t.xb]);
  const float a01 = __ldg(&p.depth[(size_t)t.yb * w + t.xa]), a11 = __ldg(&p.depth[(size_t)t.yb * w + t.xb]);
  const bool left = cs_nearest_index(u, w) == t.xa, top = cs_nearest_index(v, p.height) == t.ya;
  const float nearest = top ? (left ? a00 : a10) : (left ? a01 : a11);
  const float linear_depth = fd(1.0f, cs_bilinear_blend(t, a00, a10, a01, a11));
  const float unfiltered_depth = fd(1.0f, nearest);
  const float max_depth = vmax(linear_depth, unfiltered_depth), min_depth = vmin(linear_depth, unfiltered_depth);
  const float bias_factor = fa(1.0f, 0.000002f); // (1.0 + bias), :307-310
  distance = fs(fm(max_depth, bias_factor), ray_depth);
  penetration = fs(ray_depth, min_depth);
}

// contact_shadows.slang:45-77 for pixel (x, y): 1 - shadow
OXC_DI float cs_pixel(const ContactShadowParams& p, const ContactShadowConstants& c, int x, int y) {
  const float fw = (float)p.width, fh = (float)p.height;
  const float u = fd(fa((float)x, 0.5f), fw), v = fd(fa((float)y, 0.5f), fh);
  const float depth = __ldg(&p.depth[(size_t)cs_nearest_index(v, p.height) * p.width + cs_nearest_index(u, p.width)]);
  float cs[3] = {fs(fm(u, 2.0f), 1.0f), fs(fm(v, 2.0f), 1.0f), depth};
  const float hw = row_dot4(p.inv_pv_row[3], cs[0], cs[1], cs[2], 1.0f);
  const float ws[3] = {fd(row_dot4(p.inv_pv_row[0], cs[0], cs[1], cs[2], 1.0f), hw), fd(row_dot4(p.inv_pv_row[1], cs[0], cs[1], cs[2], 1.0f), hw),
                       fd(row_dot4(p.inv_pv_row[2], cs[0], cs[1], cs[2], 1.0f), hw)};
  const float end[3] = {fa(ws[0], fm(c.dir[0], p.length)), fa(ws[1], fm(c.dir[1], p.length)), fa(ws[2], fm(c.dir[2], p.length))};
  // raymarch.slang:559-563 position_world_to_sample: mul(projection, mul(view, (end, 1))), then / w
  float pv[4], pp[4];
  for (int i = 0; i < 4; i++) pv[i] = row_dot4(p.view_row[i], end[0], end[1], end[2], 1.0f);
  for (int i = 0; i < 4; i++) pp[i] = row_dot4(p.proj_row[i], pv[0], pv[1], pv[2], pv[3]);
  const float end_cs[3] = {fd(pp[0], pp[3]), fd(pp[1], pp[3]), fd(pp[2], pp[3])};
  // :542-546 to_cs, :502-537 to_cs_dir_impl(dir, false)
  const float s = cs_sign(end_cs[2]);
  float e[4] = {fa(cs[0], fm(fs(end_cs[0], cs[0]), s)), fa(cs[1], fm(fs(end_cs[1], cs[1]), s)), fa(cs[2], fm(fs(end_cs[2], cs[2]), s)),
                fa(1.0f, fm(0.0f, s))};
  const float den = fm(e[3] >= 0.0f ? 1.0f : -1.0f, vmax(1e-10f, fabsf(e[3])));
  for (int i = 0; i < 3; i++) e[i] = fd(e[i], den);
  float delta[3], dist[3];
  for (int i = 0; i < 3; i++) {
    delta[i] = fs(e[i], cs[i]);
    dist[i] = fd(fs(delta[i] < 0.0f ? 1.0f : (i < 2 ? -1.0f : 0.0f), cs[i]), delta[i]);
  }
  const float k = vmax(0.0f, vmax(dist[0], dist[1]));
  for (int i = 0; i < 3; i++) cs[i] = fa(cs[i], fm(delta[i], k)); // the clipped start
  for (int i = 0; i < 3; i++) {
    delta[i] = fs(e[i], cs[i]);
    dist[i] = fd(fs(delta[i] >= 0.0f ? 1.0f : (i < 2 ? -1.0f : 0.0f), cs[i]), delta[i]);
  }
  const float m = vmin(1.0f, vmin(vmin(dist[0], dist[1]), dist[2]));
  float rd[3];
  for (int i = 0; i < 3; i++) {
    const float d = fm(delta[i], m);
    rd[i] = fs(fa(cs[i], d), cs[i]); // find_root's dir = end - start
  }
  // :588-595 the step count
  const float su = cs_to_uv(cs[0]), sv = cs_to_uv(cs[1]);
  const float lx = fm(fs(cs_to_uv(fa(cs[0], fm(delta[0], m))), su), fw), ly = fm(fs(cs_to_uv(fa(cs[1], fm(delta[1], m))), sv), fh);
  const uint32_t len = cs_u32(floorf(fd(fsq(fa(fm(lx, lx), fm(ly, ly))), 1.0f)));
  const uint32_t m_steps = p.steps < len ? p.steps : len;
  const uint32_t n = m_steps > 2u ? m_steps : 2u;
  // :104-175 the linear search, t = lerp(0, 1, pow((step + 1) / n, 1)) = (step + 1) / n
  const float fn = (float)n;
  float distance = 0.0f, penetration = 0.0f;
  bool hit = false;
  for (uint32_t step = 0; step < n; step++) {
    const float t = fd(fa((float)step, 1.0f), fn);
    cs_distance(p, fa(cs[0], fm(rd[0], t)), fa(cs[1], fm(rd[1], t)), fa(cs[2], fm(rd[2], t)), distance, penetration);
    if (distance < 0.0f) { hit = true; break; }
  }
  float shadow = 0.0f;
  if (hit && penetration < c.depth_thickness && distance < c.depth_thickness) {
    // smoothstep(1.0, 0.3, penetration / depth_thickness)
    const float ts = vmin(vmax(fd(fs(fd(penetration, c.depth_thickness), 1.0f), fs(0.3f, 1.0f)), 0.0f), 1.0f);
    shadow = fm(fm(ts, ts), fs(3.0f, fm(2.0f, ts)));
  }
  return fs(1.0f, shadow);
}

} // namespace oxc
