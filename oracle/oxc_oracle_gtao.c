/*
 * oxc_oracle_gtao.c — CPU ORACLE (test infrastructure) of the visibility-bitmask GTAO: RendererInstance::generate_ambient_occlusion
 * (Passes/PBR.cpp:143-311, called at RendererInstance.cpp:1040-1055) with its three compute passes, passes/gtao/vbgtao_prefilter.slang
 * :17-116, vbgtao_main.slang:31-254 and vbgtao_denoise.slang:12-82.  Same rules as oxc_oracle.c: plain C11, IEEE binary32 with round
 * to nearest, no contraction, IEEE divide / sqrt, dot(a, b) = (a.x*b.x + a.y*b.y) + a.z*b.z, mul(M, v) row by row in the same order.
 * It is one translation unit with oxc_oracle_vsm_resolve.c (and so oxc_oracle.c), included below, so that it runs the library's own
 * log2, sin / cos and binary16 rounding.  Built into liboxc_oracle_gtao.so by oracle/pyoracle_gtao.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_gtao.c -lm
 *
 * SPECIFICATION of orc_generate_ambient_occlusion (include/oxcull.h oxc_generate_ambient_occlusion repeats it).  Where the reference
 * does not define an outcome, this commits to one:
 *   1. linearize(d) = m23 / (d + m22), (m23, m22) = (projection[3][2], projection[2][2]) in glm's [column][row] (PBR.cpp:183-186).
 *   2. virtual pyramid: level 0 at any (x, y) >= 0 is linearize(depth[min(y, H-1)][min(x, W-1)]) (the prefilter's clamped gather at
 *      the texel corner 2t with offset (1, 1): .w = 2t, .z = 2t + (1, 0), .x = 2t + (0, 1), .y = 2t + (1, 1)); level k at t is
 *      weighted_average of level k-1 at 2t, 2t + (1, 0), 2t + (0, 1), 2t + (1, 1).  The reference's 16 x 16-pixel groups compute
 *      exactly these values, also beyond the extent, and store those inside max(1, W >> k) x max(1, H >> k).
 *   3. gathers and point samples: integer texel reads with clamp to edge.  GatherRed at the texel corner uv = p / size reads the quad
 *      {p - 1, p} + offset, components x = (0, 1), y = (1, 1), z = (1, 0), w = (0, 0) of it: calculate_edges reads mip 0 at p (centre),
 *      p - (1, 0) (left), p + (1, 0) (right), p - (0, 1) (top), p + (0, 1) (bottom); the denoise reads the noisy plane at p + (i, j),
 *      i, j in -1..1, and the edges at p and its four direct neighbours.  The normal's SampleLevel at the pixel centre reads p.
 *   4. SampleLevel(linear_clamp, uv, lambda): levels floor(lambda) and min(floor(lambda) + 1, 4), both always read, weight f = lambda -
 *      floor(lambda), result (1 - f) * lo + f * hi.  A level of size (w, h): x = u * w - 0.5, x0 = floor(x), wx = x - x0, texel index
 *      saturating with NaN -> 0 (oxc_alpha.cuh alpha_f2i) clamped to 0..w-1 for x0 and x0 + 1 (y likewise); top = a00 + wx * (a10 -
 *      a00), bottom = a01 + wx * (a11 - a01), top + wy * (bottom - top).  Deviation: no 8-bit quantisation of the weights.
 *   5. normals: .zw rounded to binary16 (R16G16B16A16Sfloat), oct_to_vec3 (which normalizes), mul(view, (n, 0)).xyz, normalize.
 *   6. transcendentals: cos / sin orc_sincos_canonical; log2 orc_log2_canonical; pow orc_pow_canonical (below); fast_acos as written.
 *   7. operations: normalize(v) = v / sqrt(dot(v, v)); length = sqrt(dot); sign(NaN) = 0; saturate(NaN) = 0; max / min return the
 *      other operand for a NaN (clamp(x, a, b) = min(max(x, a), b)); u32(x) truncates and saturates, NaN -> 0; frac(x) = x - floor(x);
 *      countbits = popcount; a scalar times a vector is applied per component; constants are the binary32 roundings of the literals.
 *   8. edge packing: packUnorm4x8 = round to nearest even of saturate(c) * 255, .x in the low byte; unpack = byte / 255.
 *   9. noise: Hilbert index (RendererInstance.cpp:151-170) at (x % 64, y % 64) + 288 * (noise_index % 64), converted to binary32,
 *      frac(0.5 + index * (0.75487766624669276005, 0.5698402909980532659114)).
 *  10. sky: centre linear depth >= far_clip * 0.999 writes 1.0 to the noisy plane (the edges are written first, for every pixel).
 *  11. stored formats: mips binary32 (a NaN texel is stored as 0x7FFFFFFF, the NaN the GPU's arithmetic produces), edges u32, noisy
 *      occlusion binary16 round to nearest even (read back as such by the denoise), the final AO binary32 (the value before the
 *      reference's R16F store).
 * orc_pow_canonical: binary64 throughout, one rounding to binary32.  x = m * 2^e with m in [sqrt(1/2), sqrt(2)], log(m) = 2 atanh(t),
 * t = (m - 1) / (m + 1), by its series to t^23; L = e * LN2_HI + (e * LN2_LO + log m); z = y * L; exp(z) = 2^k exp(r), k = rint(z /
 * ln 2), r = (z - k * LN2_HI) - k * LN2_LO, exp(r) by Taylor to r^13.  Special cases: pow(1, y) = 1, pow(x, 0) = 1, NaN -> NaN,
 * x < 0 -> NaN, pow(+-0, y > 0) = 0 and +inf for y < 0, pow(inf, y) = inf / 0, y = +-inf by |x| against 1.  The binary64 result
 * is within a few units of 2^-50 relative of the exact power for |z| <= 1100, so the binary32 result is within 1 ulp of the correctly
 * rounded one (it differs from it only next to a rounding tie).
 */
#include "oxc_oracle_vsm_resolve.c"

#include "oxc_oracle_gtao.h"

#define G_HALF_PI 1.57079632679f /* common/math.slang:3-4 */
#define G_PI 3.1415926535897932384626433832795f
#define G_SECTORS 32u
#define G_LEVELS 5u

static float g_max(float a, float b) { return (b != b || a > b) ? a : b; }
static float g_min(float a, float b) { return (b != b || a < b) ? a : b; }
static float g_sat(float x) { return g_min(g_max(x, 0.0f), 1.0f); }
static float g_frac(float x) { return x - floorf(x); }
static float g_sign(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }
static uint32_t g_u32(float f) { return !(f > 0.0f) ? 0u : (f >= 4294967296.0f ? 0xFFFFFFFFu : (uint32_t)f); }
static int32_t g_i32(float f) { return !(f == f) ? 0 : (f >= 2147483648.0f ? INT32_MAX : (f <= -2147483648.0f ? INT32_MIN : (int32_t)f)); }
static float g_dot3(const float a[3], const float b[3]) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
static void g_normalize(const float v[3], float out[3]) {
  const float l = sqrtf(g_dot3(v, v));
  out[0] = v[0] / l; out[1] = v[1] / l; out[2] = v[2] / l;
}
static int64_t g_clampi(int64_t i, int64_t n) { return i < 0 ? 0 : (i > n - 1 ? n - 1 : i); }

/* binary32 -> binary16 bits, round to nearest even (values this pass stores are in [0, 1]) */
static uint16_t g_half_bits(float f) {
  const float r = orc_round_to_half(f);
  const uint32_t u = f2bits(r), s = (u >> 16) & 0x8000u, a = u & 0x7FFFFFFFu;
  if (a > 0x7F800000u) return (uint16_t)(s | 0x7FFFu);
  if (a == 0x7F800000u) return (uint16_t)(s | 0x7C00u);
  if (a >= 0x38800000u) return (uint16_t)(s | (((a >> 23) - 112u) << 10) | ((a >> 13) & 0x3FFu));
  return (uint16_t)(s | (uint32_t)(bits2f(a) * 16777216.0f));
}
static float g_half_float(uint16_t h) {
  const uint32_t s = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 31u, m = h & 1023u;
  if (e == 0) return bits2f(s | f2bits((float)m * 5.9604644775390625e-08f));
  if (e == 31) return bits2f(s | 0x7F800000u | (m ? (0x00400000u | (m << 13)) : 0u));
  return bits2f(s | ((e + 112u) << 23) | (m << 13));
}

float orc_pow_canonical(float xf, float yf) {
  if (xf == 1.0f || yf == 0.0f) return 1.0f;
  if (xf != xf || yf != yf || xf < 0.0f) return NAN;
  if (xf == 0.0f) return yf > 0.0f ? 0.0f : INFINITY;
  if (xf == INFINITY) return yf > 0.0f ? INFINITY : 0.0f;
  if (fabsf(yf) == INFINITY) return (xf < 1.0f) == (yf > 0.0f) ? 0.0f : INFINITY;
  int e = 0;
  float xm = xf;
  if (xm < 1.17549435e-38f) { xm = xm * 16777216.0f; e = -24; }
  const uint32_t bits = f2bits(xm);
  e += (int)(bits >> 23) - 127;
  float m = bits2f((bits & 0x007FFFFFu) | 0x3F800000u);
  if (m > 1.41421354f) { m = m * 0.5f; e += 1; }
  const double md = (double)m;
  const double t = (md - 1.0) / (md + 1.0);
  const double s = t * t;
  double p = 1.0 / 23.0;
  p = 1.0 / 21.0 + s * p;
  p = 1.0 / 19.0 + s * p;
  p = 1.0 / 17.0 + s * p;
  p = 1.0 / 15.0 + s * p;
  p = 1.0 / 13.0 + s * p;
  p = 1.0 / 11.0 + s * p;
  p = 1.0 / 9.0 + s * p;
  p = 1.0 / 7.0 + s * p;
  p = 1.0 / 5.0 + s * p;
  p = 1.0 / 3.0 + s * p;
  const double u = t * 2.0;
  const double lm = u + (u * s) * p;
  const double ed = (double)e;
  const double L = ed * 6.93147180369123816490e-01 + (ed * 1.90821492927058770002e-10 + lm);
  double z = (double)yf * L;
  z = z > 1100.0 ? 1100.0 : (z < -1100.0 ? -1100.0 : z);
  const double k = rint(z * 1.44269504088896338700e+00);
  const double r = (z + -(k * 6.93147180369123816490e-01)) + -(k * 1.90821492927058770002e-10);
  double q = 1.0 / 6227020800.0;           /* 1/13! */
  q = 1.0 / 479001600.0 + r * q;           /* 1/12! */
  q = 1.0 / 39916800.0 + r * q;
  q = 1.0 / 3628800.0 + r * q;
  q = 1.0 / 362880.0 + r * q;
  q = 1.0 / 40320.0 + r * q;
  q = 1.0 / 5040.0 + r * q;
  q = 1.0 / 720.0 + r * q;
  q = 1.0 / 120.0 + r * q;
  q = 1.0 / 24.0 + r * q;
  q = 1.0 / 6.0 + r * q;
  q = 0.5 + r * q;
  q = 1.0 + r * q;
  const double er = 1.0 + r * q;
  return (float)ldexp(er, (int)k);
}

/* RendererInstance.cpp:151-170 */
uint32_t orc_gtao_hilbert_index(uint32_t px, uint32_t py) {
  uint32_t index = 0;
  for (uint32_t level = 32u; level > 0u; level /= 2u) {
    const uint32_t rx = (px & level) > 0u, ry = (py & level) > 0u;
    index += level * level * ((3u * rx) ^ ry);
    if (ry == 0u) {
      if (rx == 1u) { px = 63u - px; py = 63u - py; }
      const uint32_t t = px; px = py; py = t;
    }
  }
  return index & 0xFFFFu;
}

/* vbgtao_main.slang:39-45 */
void orc_gtao_noise(uint32_t x, uint32_t y, uint32_t noise_index, float out[2]) {
  const uint32_t index = orc_gtao_hilbert_index(x % 64u, y % 64u) + 288u * (noise_index % 64u);
  const float fi = (float)index;
  out[0] = g_frac(0.5f + fi * 0.75487766624669276005f);
  out[1] = g_frac(0.5f + fi * 0.5698402909980532659114f);
}

/* :32-37 */
float orc_gtao_fast_acos(float in_x) {
  const float x = fabsf(in_x);
  float res = -0.156583f * x + G_HALF_PI;
  res = res * sqrtf(g_sat(1.0f - x));
  return in_x >= 0.0f ? res : G_PI - res;
}

/* :102-119 */
uint32_t orc_gtao_update_sectors(float min_h, float max_h, uint32_t bitmask) {
  const uint32_t angle = g_u32(ceilf(g_sat(max_h - min_h) * (float)G_SECTORS));
  if (angle == 0u) return bitmask;
  uint32_t start = g_u32(g_sat(min_h) * (float)G_SECTORS);
  start = start < G_SECTORS - 1u ? start : G_SECTORS - 1u;
  const uint32_t bits = 0xFFFFFFFFu >> (G_SECTORS - angle);
  return bitmask | (bits << start);
}

/* :124-146 */
uint32_t orc_gtao_calc_sector_mask(float thickness, const float dp[3], const float vd[3], float sd, float n) {
  const float back[3] = {dp[0] - vd[0] * thickness, dp[1] - vd[1] * thickness, dp[2] - vd[2] * thickness};
  float a[3], b[3];
  g_normalize(dp, a);
  g_normalize(back, b);
  float h0 = orc_gtao_fast_acos(g_dot3(a, vd)), h1 = orc_gtao_fast_acos(g_dot3(b, vd));
  h0 = g_sat(((sd * -h0 + n) + G_HALF_PI) / G_PI);
  h1 = g_sat(((sd * -h1 + n) + G_HALF_PI) / G_PI);
  return sd >= 0.0f ? orc_gtao_update_sectors(h1, h0, 0u) : orc_gtao_update_sectors(h0, h1, 0u);
}

float orc_gtao_linearize(const float P[16], float d) { return P[14] / (d + P[10]); }

/* vbgtao_prefilter.slang:23-39 */
float orc_gtao_weighted_average(float d0, float d1, float d2, float d3) {
  const float effect_radius = 0.75f * 0.5f * 1.457f;
  const float falloff_range = 0.615f * effect_radius;
  const float falloff_from = effect_radius * (1.0f - 0.615f);
  const float falloff_mul = -1.0f / falloff_range;
  const float falloff_add = falloff_from / falloff_range + 1.0f;
  const float mn = g_min(g_min(d0, d1), g_min(d2, d3));
  const float w0 = g_sat((d0 - mn) * falloff_mul + falloff_add), w1 = g_sat((d1 - mn) * falloff_mul + falloff_add);
  const float w2 = g_sat((d2 - mn) * falloff_mul + falloff_add), w3 = g_sat((d3 - mn) * falloff_mul + falloff_add);
  const float total = w0 + w1 + w2 + w3;
  return (w0 * d0 + w1 * d1 + w2 * d2 + w3 * d3) / total;
}

static uint32_t g_dim(uint32_t n, uint32_t k) { return (n >> k) > 1u ? (n >> k) : 1u; }

uint64_t orc_gtao_mip_offset(uint32_t W, uint32_t H, uint32_t level) {
  uint64_t off = 0;
  for (uint32_t k = 0; k < level; k++) off += (uint64_t)g_dim(W, k) * g_dim(H, k);
  return off;
}

typedef struct GCtx {
  const float* depth;
  uint32_t W, H;
  float m23, m22;
} GCtx;

/* the virtual pyramid (spec 2) at any (x, y) >= 0 */
static float g_virtual(const GCtx* g, uint32_t k, uint64_t x, uint64_t y) {
  if (k == 0) {
    const uint64_t cx = x < g->W - 1u ? x : g->W - 1u, cy = y < g->H - 1u ? y : g->H - 1u;
    return g->m23 / (g->depth[cy * g->W + cx] + g->m22);
  }
  return orc_gtao_weighted_average(g_virtual(g, k - 1, 2 * x, 2 * y), g_virtual(g, k - 1, 2 * x + 1, 2 * y), g_virtual(g, k - 1, 2 * x, 2 * y + 1),
                                   g_virtual(g, k - 1, 2 * x + 1, 2 * y + 1));
}

static float g_level_bilinear(const float* lvl, uint32_t w, uint32_t h, float u, float v) {
  const float x = u * (float)w - 0.5f, y = v * (float)h - 0.5f;
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = x - x0, wy = y - y0;
  const int64_t ix = g_i32(x0), iy = g_i32(y0);
  const int64_t xa = g_clampi(ix, w), xb = g_clampi(ix + 1, w), ya = g_clampi(iy, h), yb = g_clampi(iy + 1, h);
  const float a00 = lvl[ya * w + xa], a10 = lvl[ya * w + xb], a01 = lvl[yb * w + xa], a11 = lvl[yb * w + xb];
  const float top = a00 + wx * (a10 - a00), bot = a01 + wx * (a11 - a01);
  return top + wy * (bot - top);
}

float orc_gtao_sample_level(const float* mips, uint32_t W, uint32_t H, float u, float v, float lambda) {
  const float fl = floorf(lambda);
  const uint32_t lo = (uint32_t)fl, hi = lo + 1u < G_LEVELS - 1u ? lo + 1u : G_LEVELS - 1u;
  const float f = lambda - fl;
  const float a = g_level_bilinear(mips + orc_gtao_mip_offset(W, H, lo), g_dim(W, lo), g_dim(H, lo), u, v);
  const float b = g_level_bilinear(mips + orc_gtao_mip_offset(W, H, hi), g_dim(W, hi), g_dim(H, hi), u, v);
  return (1.0f - f) * a + f * b;
}

/* :59-67 */
static void g_view_position(const float P[16], float u, float v, float ld, float out[3]) {
  const float nx = u * 2.0f - 1.0f, ny = v * 2.0f - 1.0f;
  out[0] = (nx / P[0]) * ld;
  out[1] = (ny / P[5]) * ld;
  out[2] = -1.0f * ld;
}

static float g_unorm8(uint32_t p, int i) { return (float)((p >> (8 * i)) & 0xFFu) / 255.0f; }

/* :148-254 for pixel (x, y); writes the edges and returns the noisy occlusion before its binary16 store */
static float g_main_pixel(const OxcGtaoCamera* cam, const OxcGtaoSettings* st, const float* mips, const float* normals, uint32_t W, uint32_t H,
                          uint32_t x, uint32_t y, uint32_t* edge_out) {
  const float* P = cam->projection;
  const float rx = (float)W, ry = (float)H;
  /* calculate_edges :69-100 */
  const float c = mips[(size_t)y * W + x];
  const float l = mips[(size_t)y * W + g_clampi((int64_t)x - 1, W)], r = mips[(size_t)y * W + g_clampi((int64_t)x + 1, W)];
  const float t = mips[(size_t)g_clampi((int64_t)y - 1, H) * W + x], b = mips[(size_t)g_clampi((int64_t)y + 1, H) * W + x];
  float e[4] = {l - c, r - c, t - c, b - c};
  const float slr = (e[1] - e[0]) * 0.5f, stb = (e[3] - e[2]) * 0.5f;
  const float adj[4] = {e[0] + slr, e[1] + -slr, e[2] + stb, e[3] + -stb};
  const float scale = c * 0.011f;
  uint32_t packed = 0;
  for (int i = 0; i < 4; i++) {
    e[i] = g_min(fabsf(e[i]), fabsf(adj[i]));
    e[i] = g_sat((1.0f + 0.25f) - e[i] / scale);
    packed |= (uint32_t)rintf(g_sat(e[i]) * 255.0f) << (8 * i);
  }
  *edge_out = packed;
  float ld = c;
  if (ld >= cam->far_clip * 0.999f) return 1.0f;
  const float thickness = st->thickness, slice_count = (float)st->slice_count, sps = (float)st->samples_per_slice_side;
  const float effect_radius = st->effect_radius * 1.457f;
  const float falloff_range = 0.615f * effect_radius;
  const float falloff_from = effect_radius * (1.0f - 0.615f);
  const float falloff_mul = -1.0f / falloff_range;
  const float falloff_add = falloff_from / falloff_range + 1.0f;
  const float u = ((float)x + 0.5f) / rx, v = ((float)y + 0.5f) / ry;
  ld = ld * 0.99999f;
  float origin[3], vd[3];
  g_view_position(P, u, v, ld, origin);
  const float neg[3] = {-origin[0], -origin[1], -origin[2]};
  g_normalize(neg, vd);
  /* load_normal_view_space :47-57 */
  const float* np = normals + ((size_t)y * W + x) * 4;
  const float ex = orc_round_to_half(np[2]), ey = orc_round_to_half(np[3]);
  float o[3] = {ex, ey, (1.0f - fabsf(ex)) - fabsf(ey)};
  const float sx = o[0] >= 0.0f ? 1.0f : -1.0f, sy = o[1] >= 0.0f ? 1.0f : -1.0f;
  if (o[2] < 0.0f) { o[0] = (1.0f - fabsf(ey)) * sx; o[1] = (1.0f - fabsf(ex)) * sy; }
  float wn[3];
  g_normalize(o, wn);
  const float* V = cam->view;
  float vn[3], normal[3];
  for (int i = 0; i < 3; i++) vn[i] = ((V[i] * wn[0] + V[4 + i] * wn[1]) + V[8 + i] * wn[2]) + V[12 + i] * 0.0f;
  g_normalize(vn, normal);
  float noise[2];
  orc_gtao_noise(x, y, st->noise_index, noise);
  const float half_r = 0.5f * effect_radius;
  const float sr_u = (half_r * fabsf(P[0])) / ld, sr_v = (half_r * fabsf(P[5])) / ld;
  const float sr_px = sr_u * rx;
  const float min_s = 1.3f / g_max(sr_px, 1.3f);
  float visibility = 0.0f;
  for (float slice_t = 0.0f; slice_t < slice_count; slice_t += 1.0f) {
    const float slice = (slice_t + noise[0]) / slice_count;
    const float phi = slice * G_PI;
    float sn, cs;
    orc_sincos_canonical(phi, &sn, &cs);
    const float dir[3] = {cs, sn, 0.0f};
    const float dd = g_dot3(dir, vd);
    const float od_raw[3] = {dir[0] - dd * vd[0], dir[1] - dd * vd[1], dir[2] - dd * vd[2]};
    float od[3], axis[3];
    g_normalize(od_raw, od);
    const float cr[3] = {dir[1] * vd[2] - dir[2] * vd[1], dir[2] * vd[0] - dir[0] * vd[2], dir[0] * vd[1] - dir[1] * vd[0]};
    g_normalize(cr, axis);
    const float na = g_dot3(normal, axis);
    const float pn[3] = {normal[0] - axis[0] * na, normal[1] - axis[1] * na, normal[2] - axis[2] * na};
    const float pnl = g_max(sqrtf(g_dot3(pn, pn)), 1e-6f);
    const float sign_norm = g_sign(g_dot3(od, pn));
    const float cos_norm = g_sat(g_dot3(pn, vd) / pnl);
    const float n = sign_norm * orc_gtao_fast_acos(cos_norm);
    const float mul_u = cs * sr_u, mul_v = -sn * sr_v;
    uint32_t bitmask = 0;
    float occlusion = 0.0f;
    for (float sample_t = 0.0f; sample_t < sps; sample_t += 1.0f) {
      const float sample_noise = g_frac(noise[1] + (slice_t + sample_t * sps) * 0.6180339887498948482f);
      float s = (sample_t + sample_noise) / sps;
      s = s * s;
      s = s + min_s;
      const float off_u = s * mul_u, off_v = s * mul_v;
      const float p1u = u + off_u, p1v = v + off_v, p2u = u - off_u, p2v = v - off_v;
      const float lu = off_u * rx, lv = off_v * ry;
      const float lam = g_min(g_max(orc_log2_canonical(sqrtf(lu * lu + lv * lv)) - 3.30f, 0.0f), (float)(G_LEVELS - 1u));
      const float d1 = orc_gtao_sample_level(mips, W, H, p1u, p1v, lam), d2 = orc_gtao_sample_level(mips, W, H, p2u, p2v, lam);
      float sp1[3], sp2[3];
      g_view_position(P, p1u, p1v, d1, sp1);
      g_view_position(P, p2u, p2v, d2, sp2);
      const float del1[3] = {sp1[0] - origin[0], sp1[1] - origin[1], sp1[2] - origin[2]};
      const float del2[3] = {sp2[0] - origin[0], sp2[1] - origin[1], sp2[2] - origin[2]};
      const uint32_t m1 = orc_gtao_calc_sector_mask(thickness, del1, vd, 1.0f, n);
      const uint32_t m2 = orc_gtao_calc_sector_mask(thickness, del2, vd, -1.0f, n);
      const float f1 = g_sat(sqrtf(g_dot3(del1, del1)) * falloff_mul + falloff_add);
      const float f2 = g_sat(sqrtf(g_dot3(del2, del2)) * falloff_mul + falloff_add);
      occlusion = occlusion + (f1 * (float)__builtin_popcount(m1 & ~bitmask)) / (float)G_SECTORS;
      bitmask |= m1;
      occlusion = occlusion + (f2 * (float)__builtin_popcount(m2 & ~bitmask)) / (float)G_SECTORS;
      bitmask |= m2;
    }
    visibility = visibility + g_sat(1.0f - occlusion);
  }
  return g_sat(visibility / slice_count);
}

/* vbgtao_denoise.slang:14-82 */
float orc_gtao_denoise_pixel(const uint16_t* noisy, const uint32_t* edges, uint32_t W, uint32_t H, uint32_t x, uint32_t y, float final_power) {
#define G_AT(plane, i, j) plane[(size_t)g_clampi((int64_t)y + (j), H) * W + (size_t)g_clampi((int64_t)x + (i), W)]
  const uint32_t ec = G_AT(edges, 0, 0), el = G_AT(edges, -1, 0), er = G_AT(edges, 1, 0), et = G_AT(edges, 0, -1), eb = G_AT(edges, 0, 1);
  const float center_w = 1.2f;
  const float left_w = g_unorm8(ec, 0) * g_unorm8(el, 1);
  const float right_w = g_unorm8(ec, 1) * g_unorm8(er, 0);
  const float top_w = g_unorm8(ec, 2) * g_unorm8(et, 3);
  const float bottom_w = g_unorm8(ec, 3) * g_unorm8(eb, 2);
  const float tl_w = 0.425f * (top_w * g_unorm8(et, 0) + left_w * g_unorm8(el, 2));
  const float tr_w = 0.425f * (top_w * g_unorm8(et, 1) + right_w * g_unorm8(er, 2));
  const float bl_w = 0.425f * (bottom_w * g_unorm8(eb, 0) + left_w * g_unorm8(el, 3));
  const float br_w = 0.425f * (bottom_w * g_unorm8(eb, 1) + right_w * g_unorm8(er, 3));
  float sum = g_half_float(G_AT(noisy, 0, 0)) * center_w;
  sum = sum + g_half_float(G_AT(noisy, -1, 0)) * left_w;
  sum = sum + g_half_float(G_AT(noisy, 1, 0)) * right_w;
  sum = sum + g_half_float(G_AT(noisy, 0, -1)) * top_w;
  sum = sum + g_half_float(G_AT(noisy, 0, 1)) * bottom_w;
  sum = sum + g_half_float(G_AT(noisy, -1, -1)) * tl_w;
  sum = sum + g_half_float(G_AT(noisy, 1, -1)) * tr_w;
  sum = sum + g_half_float(G_AT(noisy, -1, 1)) * bl_w;
  sum = sum + g_half_float(G_AT(noisy, 1, 1)) * br_w;
#undef G_AT
  float sw = center_w;
  sw = sw + left_w;
  sw = sw + right_w;
  sw = sw + top_w;
  sw = sw + bottom_w;
  sw = sw + tl_w;
  sw = sw + tr_w;
  sw = sw + bl_w;
  sw = sw + br_w;
  return orc_pow_canonical(g_max(sum / sw, 0.0f), final_power);
}

void orc_generate_ambient_occlusion(const OxcGtaoCamera* cam, const OxcGtaoSettings* st, const float* depth, const float* normals, uint32_t W,
                                    uint32_t H, float* mips, uint32_t* edges, uint16_t* noisy, float* ao) {
  const GCtx g = {depth, W, H, cam->projection[14], cam->projection[10]};
  /* prefilter: the stored texels of the virtual pyramid; level k from level k-1's stored and virtual texels */
  for (uint32_t k = 0; k < G_LEVELS; k++) {
    const uint32_t w = g_dim(W, k), h = g_dim(H, k);
    float* lvl = mips + orc_gtao_mip_offset(W, H, k);
    for (uint32_t ty = 0; ty < h; ty++)
      for (uint32_t tx = 0; tx < w; tx++) {
        const float v = g_virtual(&g, k, tx, ty);
        lvl[(size_t)ty * w + tx] = v != v ? bits2f(0x7FFFFFFFu) : v; /* spec 11: the stored NaN */
      }
  }
  for (uint32_t y = 0; y < H; y++)
    for (uint32_t x = 0; x < W; x++) noisy[(size_t)y * W + x] = g_half_bits(g_main_pixel(cam, st, mips, normals, W, H, x, y, &edges[(size_t)y * W + x]));
  for (uint32_t y = 0; y < H; y++)
    for (uint32_t x = 0; x < W; x++) ao[(size_t)y * W + x] = orc_gtao_denoise_pixel(noisy, edges, W, H, x, y, st->final_power);
}
