/*
 * oxc_oracle_contact_shadows.c — CPU ORACLE (test infrastructure) of the contact-shadow pass: RendererInstance's contact_shadows pass
 * (RendererInstance.cpp:990-1020), passes/contact_shadows.slang:29-78 and the raymarch.slang functions it calls, one C function per
 * shader function, in the shader's structure.  Only the path this call site takes is restated: linear steps with jitter 1 and exponent
 * 1, no bisection, no secant step, no sloppy march, march_behind_surfaces = false (so every sample is valid).  Same rules as
 * oxc_oracle.c: plain C11, IEEE binary32 with round to nearest, no contraction, IEEE divide / sqrt, sums and products in written order,
 * dot(a, b) = (a.x*b.x + a.y*b.y) + a.z*b.z, mul(M, v) row by row in the same order.  It is one translation unit with
 * oxc_oracle_pbr.c (and so the GTAO and resolve oracles and oxc_oracle.c), included below, so that it runs the library's own alpha_f2i
 * and smoothstep.  Built into liboxc_oracle_contact_shadows.so by oracle/pyoracle_contact_shadows.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_contact_shadows.c -lm
 *
 * SPECIFICATION of orc_contact_shadows (include/oxcull.h oxc_contact_shadows repeats it).  Where the shader does not define an outcome,
 * this commits to one:
 *   1. the nearest tap at uv reads texel (floor(u * W), floor(v * H)), indices NaN-safe and saturating (alpha_f2i), clamped to the edge.
 *   2. the bilinear tap at uv: x = u * W - 0.5, x0 = floor(x), wx = x - x0 (y likewise), texels x0, x0 + 1 and y0, y0 + 1 by the same
 *      index rule, top = a00 + wx * (a10 - a00), bottom = a01 + wx * (a11 - a01), top + wy * (bottom - top): the GTAO's level tap
 *      (oxc_oracle_gtao.c item 4).  Deviation: binary32 weights, no 8-bit weight quantisation.
 *   3. pow(x, 1.0) = x; lerp(0, 1, t) = 0 + (1 - 0) * t; sign(NaN) = 0; max / min return the other operand for a NaN; saturate(NaN) = 0;
 *      u32(x) truncates and saturates, NaN -> 0; smoothstep as orc_pbr_smoothstep (also with reversed edges).
 *   4. (1.0 + bias) = fl(1 + fl(2e-6)) = 0x3F800011.  Slang types an unsuffixed literal as float, so the shader adds two binary32
 *      values; a compiler that folds the sum in binary64 and rounds once gets the same bits (2e-6 is 16.78 ulps of 1 either way).
 *   5. the w guard of to_cs_dir_impl is evaluated as written, for all four components (w is always 1 there).
 *   6. output: 1 - shadow, binary32; in [0, 1] and never NaN.
 */
#include "oxc_oracle_pbr.c"

#include "oxc_oracle_contact_shadows.h"

static float cs_max(float a, float b) { return (b != b || a > b) ? a : b; }
static float cs_min(float a, float b) { return (b != b || a < b) ? a : b; }
static float cs_sign(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }
static uint32_t cs_u32(float f) { return !(f > 0.0f) ? 0u : (f >= 4294967296.0f ? 0xFFFFFFFFu : (uint32_t)f); }
static int64_t cs_clampi(int64_t i, int64_t n) { return i < 0 ? 0 : (i > n - 1 ? n - 1 : i); }

/* mul(M, v) of a column-major matrix: M[i][j] = m[j * 4 + i] */
static void cs_mul(const float m[16], const float v[4], float out[4]) {
  for (int i = 0; i < 4; i++) out[i] = ((m[i] * v[0] + m[4 + i] * v[1]) + m[8 + i] * v[2]) + m[12 + i] * v[3];
}

/* raymarch.slang:307, (1.0 + bias) */
float orc_cs_bias_factor(void) {
  const float bias = 0.000002f;
  return 1.0f + bias;
}

/* SampleLevel(sampler_nearest_clamp, uv, 0) */
float orc_cs_nearest(const float* depth, uint32_t W, uint32_t H, float u, float v) {
  const int64_t ix = cs_clampi(alpha_f2i(floorf(u * (float)W)), W), iy = cs_clampi(alpha_f2i(floorf(v * (float)H)), H);
  return depth[(size_t)iy * W + (size_t)ix];
}

/* SampleLevel(sampler_linear_clamp, uv, 0) */
float orc_cs_bilinear(const float* depth, uint32_t W, uint32_t H, float u, float v) {
  const float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = x - x0, wy = y - y0;
  const int64_t ix = alpha_f2i(x0), iy = alpha_f2i(y0);
  const int64_t xa = cs_clampi(ix, W), xb = cs_clampi(ix + 1, W), ya = cs_clampi(iy, H), yb = cs_clampi(iy + 1, H);
  const float a00 = depth[ya * W + xa], a10 = depth[ya * W + xb], a01 = depth[yb * W + xa], a11 = depth[yb * W + xb];
  const float top = a00 + wx * (a10 - a00), bot = a01 + wx * (a11 - a01);
  return top + wy * (bot - top);
}

/* raymarch.slang:15-17 */
static float cs_to_uv(float c) { return c * 0.5f + 0.5f; }

/* raymarch.slang:542-546 to_cs, then :502-537 to_cs_dir_impl(dir, false) */
void orc_cs_clip_ray(const float start_cs[3], const float end_cs_in[3], float out[6]) {
  const float s = cs_sign(end_cs_in[2]);
  const float dir[4] = {(end_cs_in[0] - start_cs[0]) * s, (end_cs_in[1] - start_cs[1]) * s, (end_cs_in[2] - start_cs[2]) * s, 0.0f * s};
  float e[4] = {start_cs[0] + dir[0], start_cs[1] + dir[1], start_cs[2] + dir[2], 1.0f + dir[3]};
  const float den = (e[3] >= 0.0f ? 1.0f : -1.0f) * cs_max(1e-10f, fabsf(e[3]));
  for (int i = 0; i < 4; i++) e[i] = e[i] / den;
  /* clip the start to the frustum's near edges (x and y only) */
  float start[3] = {start_cs[0], start_cs[1], start_cs[2]};
  {
    float delta[3], dist[3];
    const float near_pos[3] = {1.0f, 1.0f, 1.0f}, near_neg[3] = {-1.0f, -1.0f, 0.0f};
    for (int i = 0; i < 3; i++) {
      delta[i] = e[i] - start[i];
      dist[i] = ((delta[i] < 0.0f ? near_pos[i] : near_neg[i]) - start[i]) / delta[i];
    }
    const float k = cs_max(0.0f, cs_max(dist[0], dist[1]));
    for (int i = 0; i < 3; i++) start[i] = start[i] + delta[i] * k;
  }
  /* clip the end to the far edges */
  float delta[3], dist[3];
  const float far_pos[3] = {1.0f, 1.0f, 1.0f}, far_neg[3] = {-1.0f, -1.0f, 0.0f};
  for (int i = 0; i < 3; i++) {
    delta[i] = e[i] - start[i];
    dist[i] = ((delta[i] >= 0.0f ? far_pos[i] : far_neg[i]) - start[i]) / delta[i];
  }
  const float m = cs_min(1.0f, cs_min(cs_min(dist[0], dist[1]), dist[2]));
  for (int i = 0; i < 3; i++) {
    delta[i] = delta[i] * m;
    out[i] = start[i];
    out[3 + i] = start[i] + delta[i];
  }
}

/* raymarch.slang:588-595 */
uint32_t orc_cs_step_count(const float ray[6], uint32_t W, uint32_t H, uint32_t steps) {
  const float su = cs_to_uv(ray[0]), sv = cs_to_uv(ray[1]), eu = cs_to_uv(ray[3]), ev = cs_to_uv(ray[4]);
  const float lx = (eu - su) * (float)W, ly = (ev - sv) * (float)H;
  const uint32_t n = cs_u32(floorf(sqrtf(lx * lx + ly * ly) / 1.0f));
  const uint32_t m = steps < n ? steps : n;
  return m > 2u ? m : 2u;
}

/* raymarch.slang:254-322 DepthRaymarchDistanceFn::call (march_behind_surfaces and use_sloppy_march false) */
static void cs_distance(const float* depth, uint32_t W, uint32_t H, const float p[3], float* distance, float* penetration) {
  const float u = cs_to_uv(p[0]), v = cs_to_uv(p[1]);
  const float ray_depth = 1.0f / p[2];
  const float linear_depth = 1.0f / orc_cs_bilinear(depth, W, H, u, v);
  const float unfiltered_depth = 1.0f / orc_cs_nearest(depth, W, H, u, v);
  const float max_depth = cs_max(linear_depth, unfiltered_depth), min_depth = cs_min(linear_depth, unfiltered_depth);
  *distance = max_depth * orc_cs_bias_factor() - ray_depth;
  *penetration = ray_depth - min_depth;
}

float orc_cs_pixel(const OxcContactShadowCamera* cam, const OxcContactShadowSettings* st, const float* depth, uint32_t W, uint32_t H,
                   uint32_t x, uint32_t y, int32_t march_out[3]) {
  /* contact_shadows.slang:45-61 */
  const float u = ((float)x + 0.5f) / (float)W, v = ((float)y + 0.5f) / (float)H;
  const float d = orc_cs_nearest(depth, W, H, u, v);
  const float cs[3] = {u * 2.0f - 1.0f, v * 2.0f - 1.0f, d};
  const float c4[4] = {cs[0], cs[1], cs[2], 1.0f};
  float wh[4];
  cs_mul(cam->inv_projection_view, c4, wh);
  const float ws[3] = {wh[0] / wh[3], wh[1] / wh[3], wh[2] / wh[3]};
  const float rcp_near = 1.0f / cam->near_clip;
  const float* sd = st->sun_direction;
  const float l = sqrtf((sd[0] * sd[0] + sd[1] * sd[1]) + sd[2] * sd[2]);
  const float dir[3] = {sd[0] / l, sd[1] / l, sd[2] / l};
  const float end[4] = {ws[0] + dir[0] * st->length, ws[1] + dir[1] * st->length, ws[2] + dir[2] * st->length, 1.0f};
  /* raymarch.slang:559-568 position_world_to_sample */
  float pv[4], pp[4];
  cs_mul(cam->view, end, pv);
  cs_mul(cam->projection, pv, pp);
  const float end_cs[3] = {pp[0] / pp[3], pp[1] / pp[3], pp[2] / pp[3]};
  float ray[6];
  orc_cs_clip_ray(cs, end_cs, ray);
  /* raymarch.slang:584-629 march, :104-242 find_root with linear steps only */
  const uint32_t n = orc_cs_step_count(ray, W, H, st->steps);
  const float depth_thickness = st->thickness * rcp_near;
  const float rd[3] = {ray[3] - ray[0], ray[4] - ray[1], ray[5] - ray[2]};
  int32_t hit_step = -1;
  float distance = 0.0f, penetration = 0.0f;
  for (uint32_t step = 0; step < n; step++) {
    const float t = 0.0f + (1.0f - 0.0f) * (((float)step + 1.0f) / (float)n);
    const float p[3] = {ray[0] + rd[0] * t, ray[1] + rd[1] * t, ray[2] + rd[2] * t};
    cs_distance(depth, W, H, p, &distance, &penetration);
    if (distance < 0.0f) { hit_step = (int32_t)step; break; }
  }
  const int contact = hit_step >= 0 && penetration < depth_thickness && distance < depth_thickness;
  float shadow = 0.0f;
  if (contact) shadow = orc_pbr_smoothstep(1.0f, 0.3f, penetration / depth_thickness);
  if (march_out) { march_out[0] = (int32_t)n; march_out[1] = hit_step; march_out[2] = contact; }
  return 1.0f - shadow;
}

void orc_contact_shadows(const OxcContactShadowCamera* cam, const OxcContactShadowSettings* st, const float* depth, uint32_t W, uint32_t H,
                         float* out) {
  for (uint32_t y = 0; y < H; y++)
    for (uint32_t x = 0; x < W; x++) out[(size_t)y * W + x] = orc_cs_pixel(cam, st, depth, W, H, x, y, NULL);
}
