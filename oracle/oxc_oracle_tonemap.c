/*
 * oxc_oracle_tonemap.c — CPU ORACLE (test infrastructure) of the tonemap pass (passes/tonemap.slang fs_main with ACES_Fitted, AgX_DS
 * and GT7ToneMapping, passes/lens.slang, common/color.slang, PostProcess.cpp:205-247), one C function per shader function.  One
 * translation unit with oxc_oracle_post.c, included below, so that it runs the library's own log2 (orc_log2_canonical), exp
 * (orc_exp_canonical), pow (orc_pow_canonical), cos (orc_sincos_canonical) and the saturating float -> int conversion (alpha_f2i).
 * Built into liboxc_oracle_tonemap.so by oracle/pyoracle_tonemap.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_tonemap.c -lm
 *
 * SPECIFICATION: include/oxcull.h above oxc_tonemap (items 1-10).  binary32, no contraction, each expression in the shader's written
 * order; max / min take the other operand for a NaN; every stored NaN is 0x7FFFFFFF.
 */
#include "oxc_oracle_post.c"

#include "oxc_oracle_tonemap.h"

static const float T_PI = 0x1.921fb6p+1f;

/* ---------------------------------------------------------------- shader math */

typedef struct { float v[3]; } TV3;
typedef struct { float m[9]; } TM3; /* row-major: m[3 * row + col] */

static TV3 t_v3(float x, float y, float z) { TV3 r = {{x, y, z}}; return r; }
static float t_dot(TV3 a, TV3 b) { return (a.v[0] * b.v[0] + a.v[1] * b.v[1]) + a.v[2] * b.v[2]; }
/* mul(M, v): row . v */
static TV3 t_mul_mv(const TM3* m, TV3 c) {
  TV3 r;
  for (int i = 0; i < 3; i++) r.v[i] = t_dot(t_v3(m->m[3 * i], m->m[3 * i + 1], m->m[3 * i + 2]), c);
  return r;
}
/* mul(A, B): row of A . column of B */
static TM3 t_mul_mm(const TM3* a, const TM3* b) {
  TM3 r;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) r.m[3 * i + j] = (a->m[3 * i] * b->m[j] + a->m[3 * i + 1] * b->m[3 + j]) + a->m[3 * i + 2] * b->m[6 + j];
  return r;
}
static float t_clamp01(float x) { return a_min(a_max(x, 0.0f), 1.0f); }
static float t_exp2(float x) { return orc_pow_canonical(2.0f, x); }

/* tonemap.slang inverse() */
static TM3 t_inverse(const TM3* mm) {
  const float* m = mm->m;
  const float a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
  const float A = (e * i - f * h), B = -(d * i - f * g), C = (d * h - e * g);
  const float D = -(b * i - c * h), E = (a * i - c * g), F = -(a * h - b * g);
  const float G = (b * f - c * e), H = -(a * f - c * d), I = (a * e - b * d);
  const float det = a * A + b * B + c * C;
  const float inv = 1.0f / det;
  TM3 r = {{A * inv, D * inv, G * inv, B * inv, E * inv, H * inv, C * inv, F * inv, I * inv}};
  return r;
}

static TV3 t_unproject(float x, float y) { /* color_XyYToXYZ((x, y, 1)) */
  const float Y = 1.0f;
  return t_v3((x * Y) / y, Y, ((1.0f - x - y) * Y) / y);
}

static TM3 t_primaries_to_matrix(const float r[2], const float g[2], const float b[2], const float w[2]) {
  const TV3 R = t_unproject(r[0], r[1]), G = t_unproject(g[0], g[1]), B = t_unproject(b[0], b[1]), W = t_unproject(w[0], w[1]);
  const TM3 temp = {{R.v[0], G.v[0], B.v[0], 1.0f, 1.0f, 1.0f, R.v[2], G.v[2], B.v[2]}};
  const TM3 inv = t_inverse(&temp);
  const TV3 s = t_mul_mv(&inv, W);
  TM3 out;
  for (int row = 0; row < 3; row++) {
    out.m[3 * row] = R.v[row] * s.v[0];
    out.m[3 * row + 1] = G.v[row] * s.v[1];
    out.m[3 * row + 2] = B.v[row] * s.v[2];
  }
  return out;
}

/* ---------------------------------------------------------------- item 9: constants */

static const float XY_R[2] = {0.64f, 0.33f}, XY_G[2] = {0.3f, 0.6f}, XY_B[2] = {0.15f, 0.06f}, XY_W[2] = {0.3127f, 0.3290f};
static const float PQ_M1 = 0.1593017578125f, PQ_M2 = 78.84375f, PQ_C1 = 0.8359375f, PQ_C2 = 18.8515625f, PQ_C3 = 18.6875f, PQ_C = 10000.0f;
static const float REF_LUM = 100.0f;

static float t_inverse_eotf(float v) { /* inverseEotfSt2084(v, 1) */
  const float m2 = PQ_M2 * 1.0f;
  const float physical = v * REF_LUM;
  const float y = physical / PQ_C;
  const float ym = orc_pow_canonical(y, PQ_M1);
  return t_exp2(m2 * (orc_log2_canonical(PQ_C1 + PQ_C2 * ym) - orc_log2_canonical(1.0f + PQ_C3 * ym)));
}

static TV3 t_rgb_to_ictcp(TV3 c) {
  const float* rgb = c.v;
  const float l = (rgb[0] * 1688.0f + rgb[1] * 2146.0f + rgb[2] * 262.0f) / 4096.0f;
  const float m = (rgb[0] * 683.0f + rgb[1] * 2951.0f + rgb[2] * 462.0f) / 4096.0f;
  const float s = (rgb[0] * 99.0f + rgb[1] * 309.0f + rgb[2] * 3688.0f) / 4096.0f;
  const float lPQ = t_inverse_eotf(l), mPQ = t_inverse_eotf(m), sPQ = t_inverse_eotf(s);
  return t_v3((2048.0f * lPQ + 2048.0f * mPQ) / 4096.0f, (6610.0f * lPQ - 13613.0f * mPQ + 7003.0f * sPQ) / 4096.0f,
              (17933.0f * lPQ - 17390.0f * mPQ - 543.0f * sPQ) / 4096.0f);
}

void orc_tonemap_constants(float out[ORC_TM_CONSTANTS]) {
  const float AGX_COMPRESSION = 0.15f, AGX_LINEAR = 0.10f, AGX_PEAK = 1.0f;
  const TM3 srgb_to_xyz = t_primaries_to_matrix(XY_R, XY_G, XY_B, XY_W);
  /* color_ComputeCompressionMatrix: lerp(xyW, xy, 1 / (1 - compression)) */
  const float sf = 1.0f / (1.0f - AGX_COMPRESSION);
  float R[2], G[2], B[2];
  for (int k = 0; k < 2; k++) {
    R[k] = XY_W[k] + (XY_R[k] - XY_W[k]) * sf;
    G[k] = XY_W[k] + (XY_G[k] - XY_W[k]) * sf;
    B[k] = XY_W[k] + (XY_B[k] - XY_W[k]) * sf;
  }
  const TM3 adjusted_to_xyz = t_primaries_to_matrix(R, G, B, XY_W);
  const TM3 xyz_to_adjusted = t_inverse(&adjusted_to_xyz);
  const TM3 srgb_to_adjusted = t_mul_mm(&srgb_to_xyz, &xyz_to_adjusted);
  const TM3 adjusted_inv = t_inverse(&srgb_to_adjusted);
  for (int k = 0; k < 9; k++) {
    out[ORC_TM_AGX + k] = srgb_to_adjusted.m[k];
    out[ORC_TM_AGX_INV + k] = adjusted_inv.m[k];
  }
  const float S = AGX_PEAK * AGX_LINEAR;
  out[ORC_TM_AGX_S] = S;
  out[ORC_TM_AGX_C] = AGX_PEAK / (AGX_PEAK - S);
  out[ORC_TM_AGX_PEAK_S] = AGX_PEAK - S;
  /* GT7ToneMapping::initializeAsSDR -> initializeParameters(250) -> initializeCurve(target, 0.25, 0.538, 0.444, 1.280) */
  const float sdr = 1.0f / (250.0f / REF_LUM);
  const float target = 250.0f / REF_LUM;
  const float peak = target, alpha = 0.25f, linear = 0.444f;
  const float k = (linear - 1.0f) / (alpha - 1.0f);
  out[ORC_TM_GT7_KA] = peak * linear + peak * k;
  out[ORC_TM_GT7_KB] = -peak * k * orc_exp_canonical(linear / k);
  out[ORC_TM_GT7_KC] = -1.0f / (k * peak);
  out[ORC_TM_GT7_LINEAR_PEAK] = linear * peak;
  out[ORC_TM_GT7_TARGET] = target;
  out[ORC_TM_GT7_TARGET_UCS] = t_rgb_to_ictcp(t_v3(target, target, target)).v[0];
  out[ORC_TM_GT7_SDR] = sdr;
  out[ORC_TM_GT7_ONE_MINUS_BLEND] = 1.0f - 0.6f;
  out[ORC_TM_PQ_INV_M1] = 1.0f / PQ_M1;
  out[ORC_TM_PQ_INV_M2] = 1.0f / (PQ_M2 * 1.0f);
  const float sq3 = sqrtf(3.0f);
  out[ORC_TM_SIMPLEX_F2] = (sq3 - 1.0f) / 2.0f;
  out[ORC_TM_SIMPLEX_G2] = (3.0f - sq3) / 6.0f;
}

static float TK[ORC_TM_CONSTANTS];
static int TK_READY = 0;
static const float* t_k(void) {
  if (!TK_READY) {
    orc_tonemap_constants(TK);
    TK_READY = 1;
  }
  return TK;
}

/* ---------------------------------------------------------------- item 3: curves */

static const TM3 ACES_IN = {{0.59719f, 0.35458f, 0.04823f, 0.07600f, 0.90834f, 0.01566f, 0.02840f, 0.13383f, 0.83777f}};
static const TM3 ACES_OUT = {{1.60475f, -0.53108f, -0.07367f, -0.10208f, 1.10813f, -0.00605f, -0.00327f, -0.07276f, 1.07602f}};
static const TM3 REC709_TO_XYZ = {{0.4124564f, 0.3575761f, 0.1804375f, 0.2126729f, 0.7151522f, 0.0721750f, 0.0193339f, 0.1191920f, 0.9503041f}};
static const TM3 XYZ_TO_REC709 = {{3.2404542f, -1.5371385f, -0.4985314f, -0.9692660f, 1.8760108f, 0.0415560f, 0.0556434f, -0.2040259f, 1.0572252f}};
static const TM3 REC2020_TO_XYZ = {{0.636958f, 0.1446169f, 0.168881f, 0.2627002f, 0.6779981f, 0.0593017f, 0.0f, 0.0280727f, 1.0609851f}};
static const TM3 XYZ_TO_REC2020 = {{1.7166512f, -0.3556708f, -0.2533663f, -0.6666844f, 1.6164812f, 0.0157685f, 0.0176399f, -0.0427706f, 0.9421031f}};

static TV3 t_aces(TV3 c) {
  c = t_mul_mv(&ACES_IN, c);
  for (int i = 0; i < 3; i++) { /* RRTAndODTFit */
    const float v = c.v[i];
    const float a = v * (v + 0.0245786f) - 0.000090537f;
    const float b = v * (0.983729f * v + 0.4329510f) + 0.238081f;
    c.v[i] = a / b;
  }
  c = t_mul_mv(&ACES_OUT, c);
  for (int i = 0; i < 3; i++) c.v[i] = t_clamp01(c.v[i]); /* saturate */
  return c;
}

static TV3 t_agx(TV3 c) {
  const float* K = t_k();
  TM3 m, inv;
  memcpy(m.m, K + ORC_TM_AGX, sizeof m.m);
  memcpy(inv.m, K + ORC_TM_AGX_INV, sizeof inv.m);
  for (int i = 0; i < 3; i++) c.v[i] = a_max(c.v[i], 0.0f);
  c = t_mul_mv(&m, c);
  for (int i = 0; i < 3; i++) { /* clamp(color_DualSection(x, 0.1, 1), 0, 1) */
    const float x = c.v[i], S = K[ORC_TM_AGX_S], peak = 1.0f;
    const float d = x < S ? x : peak - K[ORC_TM_AGX_PEAK_S] * orc_exp_canonical((-K[ORC_TM_AGX_C] * (x - S)) / peak);
    c.v[i] = t_clamp01(d);
  }
  const float desat = t_dot(c, t_v3(0.2126729f, 0.7151522f, 0.0721750f));
  for (int i = 0; i < 3; i++) c.v[i] = t_clamp01(desat + (c.v[i] - desat) * 1.3f); /* lerp(desaturation, color, 1.3) */
  return t_mul_mv(&inv, c);
}

static float t_smooth_step(float x, float e0, float e1) {
  const float t = (x - e0) / (e1 - e0);
  if (x < e0) return 0.0f;
  if (x > e1) return 1.0f;
  return t * t * (3.0f - 2.0f * t);
}

static float t_gt7_curve(float x) { /* GTToneMappingCurveV2::evaluateCurve */
  const float* K = t_k();
  const float mid = 0.538f, toe = 1.280f;
  if (x < 0.0f) return 0.0f;
  const float wl = t_smooth_step(x, 0.0f, mid);
  const float wt = 1.0f - wl;
  const float shoulder = K[ORC_TM_GT7_KA] + K[ORC_TM_GT7_KB] * orc_exp_canonical(x * K[ORC_TM_GT7_KC]);
  if (x < K[ORC_TM_GT7_LINEAR_PEAK]) {
    const float toe_mapped = mid * orc_pow_canonical(x / mid, toe);
    return wt * toe_mapped + wl * x;
  }
  return shoulder;
}

static float t_eotf(float n) { /* eotfSt2084(n, 1) */
  const float* K = t_k();
  if (n < 0.0f) n = 0.0f;
  if (n > 1.0f) n = 1.0f;
  const float np = orc_pow_canonical(n, K[ORC_TM_PQ_INV_M2]);
  float l = np - PQ_C1;
  if (l < 0.0f) l = 0.0f;
  l = l / (PQ_C2 - PQ_C3 * np);
  l = orc_pow_canonical(l, K[ORC_TM_PQ_INV_M1]);
  return (l * PQ_C) / REF_LUM;
}

static TV3 t_ictcp_to_rgb(TV3 u) {
  const float* ictcp = u.v;
  const float l = ictcp[0] + 0.00860904f * ictcp[1] + 0.11103f * ictcp[2];
  const float m = ictcp[0] - 0.00860904f * ictcp[1] - 0.11103f * ictcp[2];
  const float s = ictcp[0] + 0.560031f * ictcp[1] - 0.320627f * ictcp[2];
  const float L = t_eotf(l), M = t_eotf(m), S = t_eotf(s);
  return t_v3(a_max(3.43661f * L - 2.50645f * M + 0.0698454f * S, 0.0f), a_max(-0.79133f * L + 1.9836f * M - 0.192271f * S, 0.0f),
              a_max(-0.0259499f * L - 0.0989137f * M + 1.12486f * S, 0.0f));
}

void orc_tonemap_gt7_rec2020(const float in[3], float out[3]) {
  const float* K = t_k();
  const TV3 rgb = t_v3(in[0], in[1], in[2]);
  const TV3 ucs = t_rgb_to_ictcp(rgb);
  const TV3 skewed = t_v3(t_gt7_curve(rgb.v[0]), t_gt7_curve(rgb.v[1]), t_gt7_curve(rgb.v[2]));
  const TV3 skewed_ucs = t_rgb_to_ictcp(skewed);
  const float chroma_scale = 1.0f - t_smooth_step(ucs.v[0] / K[ORC_TM_GT7_TARGET_UCS], 0.98f, 1.16f);
  const TV3 scaled_ucs = t_v3(skewed_ucs.v[0], ucs.v[1] * chroma_scale, ucs.v[2] * chroma_scale);
  const TV3 scaled = t_ictcp_to_rgb(scaled_ucs);
  for (int i = 0; i < 3; i++) {
    const float blended = K[ORC_TM_GT7_ONE_MINUS_BLEND] * skewed.v[i] + 0.6f * scaled.v[i];
    out[i] = K[ORC_TM_GT7_SDR] * a_min(blended, K[ORC_TM_GT7_TARGET]);
  }
}

static TV3 t_gt7(TV3 c) {
  const TV3 in = t_mul_mv(&XYZ_TO_REC2020, t_mul_mv(&REC709_TO_XYZ, c));
  TV3 o;
  orc_tonemap_gt7_rec2020(in.v, o.v);
  return t_mul_mv(&XYZ_TO_REC709, t_mul_mv(&REC2020_TO_XYZ, o));
}

static TV3 t_curve(uint32_t type, TV3 c) {
  switch (type) {
  case OXC_TONEMAP_ACES: return t_aces(c);
  case OXC_TONEMAP_AGX: return t_agx(c);
  case OXC_TONEMAP_GT7: return t_gt7(c);
  default: return c;
  }
}

void orc_tonemap_curve(uint32_t type, const float in[3], float out[3]) {
  const TV3 r = t_curve(type, t_v3(in[0], in[1], in[2]));
  memcpy(out, r.v, sizeof r.v);
}

/* ---------------------------------------------------------------- items 1, 2: taps */

static int64_t t_wrap(int64_t i, int64_t n) {
  const int64_t r = i % n;
  return r < 0 ? r + n : r;
}

void orc_tonemap_tap(const float* src, uint32_t W, uint32_t H, float u, float v, float out[4]) {
  const float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = x - x0, wy = y - y0;
  const int64_t ix = alpha_f2i(x0), iy = alpha_f2i(y0);
  const float* q[4];
  for (int k = 0; k < 4; k++) q[k] = src + ((size_t)t_wrap(iy + (k >> 1), H) * W + (size_t)t_wrap(ix + (k & 1), W)) * 4;
  for (int c = 0; c < 4; c++) {
    const float top = q[0][c] + wx * (q[1][c] - q[0][c]), bot = q[2][c] + wx * (q[3][c] - q[2][c]);
    out[c] = top + wy * (bot - top);
  }
}

/* ---------------------------------------------------------------- items 6-8: lens.slang */

void orc_tonemap_rg_mag(float amount, float out[2]) { /* FfxLensGetRGMag */
  const float A = 1.5220f, B = 0.00459f * amount;
  const float red = 0.612f, green = 0.549f, blue = 0.464f;
  const float ri = A + B / (red * red), gi = A + B / (green * green), bi = A + B / (blue * blue);
  out[0] = (ri - 1.0f) / (bi - 1.0f);
  out[1] = (gi - 1.0f) / (bi - 1.0f);
}

static void t_pcg3d16(uint32_t v[3]) {
  for (int i = 0; i < 3; i++) v[i] = v[i] * 12829u + 47989u;
  for (int r = 0; r < 2; r++) {
    v[0] += v[1] * v[2];
    v[1] += v[2] * v[0];
    v[2] += v[0] * v[1];
  }
  for (int i = 0; i < 3; i++) v[i] >>= 16u;
}

static void t_film_grain(int32_t x, int32_t y, float color[3], const OxcTonemapSettings* s) {
  const float* K = t_k();
  const int32_t d = alpha_f2i(s->film_grain_scale / 8.0f);
  /* item 8: a zero divisor gives the quotient -1 (all ones as u32) */
  uint32_t v[3] = {d == 0 ? 0xFFFFFFFFu : (uint32_t)(x / d), d == 0 ? 0xFFFFFFFFu : (uint32_t)(y / d), s->film_grain_seed};
  t_pcg3d16(v);
  const float rx = (float)v[0] * (1.0f / 65536.0f) - 0.5f, ry = (float)v[1] * (1.0f / 65536.0f) - 0.5f;
  const float P[2] = {(float)x / s->film_grain_scale + rx, (float)y / s->film_grain_scale + ry};
  /* simplex */
  const float u = (P[0] + P[1]) * K[ORC_TM_SIMPLEX_F2];
  const float Pi[2] = {rintf(P[0] + u), rintf(P[1] + u)};
  const float vv = (Pi[0] + Pi[1]) * K[ORC_TM_SIMPLEX_G2];
  const float p0 = P[0] - (Pi[0] - vv), p1 = P[1] - (Pi[1] - vv);
  const float len = sqrtf(p0 * p0 + p1 * p1);
  const float grain = 1.0f - 2.0f * t_exp2(-len * 3.0f);
  for (int c = 0; c < 3; c++) color[c] = color[c] + grain * a_min(color[c], 1.0f - color[c]) * s->film_grain_amount;
}

static void t_vignette(int32_t x, int32_t y, int32_t cx, int32_t cy, float color[3], float amount) {
  const float fx = (float)(x > cx ? x - cx : cx - x) / (float)cx, fy = (float)(y > cy ? y - cy : cy - y) / (float)cy;
  const float pi_over_4 = T_PI * 0.25f;
  float sx, mx, my;
  orc_sincos_canonical(fx * amount * pi_over_4, &sx, &mx);
  orc_sincos_canonical(fy * amount * pi_over_4, &sx, &my);
  mx = mx * mx;
  my = my * my;
  mx = mx * mx;
  my = my * my;
  const float f = t_clamp01(mx * my);
  for (int c = 0; c < 3; c++) color[c] *= f;
}

/* ---------------------------------------------------------------- the pass */

void orc_tonemap(const float* frame, uint32_t width, uint32_t height, const OxcTonemapSettings* s, const OxcExposure* record,
                 const float* bloom, float* out) {
  const uint32_t f = s->scene_flags;
  const int32_t W = (int32_t)width, H = (int32_t)height, cx = W / 2, cy = H / 2;
  float rg[2];
  orc_tonemap_rg_mag(s->chromatic_aberration_amount, rg);
  const float exposure = (f & OXC_SCENE_HAS_EYE_ADAPTATION) ? record->exposure : s->exposure;
  for (int32_t y = 0; y < H; y++)
    for (int32_t x = 0; x < W; x++) {
      const float u = ((float)x + 0.5f) / (float)W, v = ((float)y + 0.5f) / (float)H;
      float src[4];
      orc_tonemap_tap(frame, width, height, u, v, src);
      TV3 c = t_v3(src[0] * exposure, src[1] * exposure, src[2] * exposure);
      if (f & OXC_SCENE_HAS_BLOOM) {
        float b[4];
        orc_tonemap_tap(bloom, width / 2, height / 2, u, v, b);
        for (int k = 0; k < 3; k++) c.v[k] = c.v[k] + b[k] * s->bloom_intensity;
      }
      c = t_curve(s->tonemap_type, c);
      if (f & OXC_SCENE_HAS_CHROMATIC_ABERRATION) {
        const float rx = 1.0f / (float)(2 * cx), ry = 1.0f / (float)(2 * cy);
        float t[4];
        orc_tonemap_tap(frame, width, height, ((float)(x - cx) * rg[0] + (float)cx + 0.5f) * rx, ((float)(y - cy) * rg[0] + (float)cy + 0.5f) * ry, t);
        c.v[0] = t[0];
        orc_tonemap_tap(frame, width, height, ((float)(x - cx) * rg[1] + (float)cx + 0.5f) * rx, ((float)(y - cy) * rg[1] + (float)cy + 0.5f) * ry, t);
        c.v[1] = t[1];
        orc_tonemap_tap(frame, width, height, (float)x * rx, (float)y * ry, t);
        c.v[2] = t[2];
      }
      if (f & OXC_SCENE_HAS_VIGNETTE) t_vignette(x, y, cx, cy, c.v, s->vignette_amount);
      if (f & OXC_SCENE_HAS_FILM_GRAIN) t_film_grain(x, y, c.v, s);
      float* o = out + ((size_t)y * width + x) * 4;
      for (int k = 0; k < 3; k++) o[k] = p_nan(c.v[k]);
      o[3] = p_nan((f & OXC_SCENE_TRANSPARENT_BACKGROUND) ? src[3] : 1.0f);
    }
}
