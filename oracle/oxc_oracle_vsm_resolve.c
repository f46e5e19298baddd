/*
 * oxc_oracle_vsm_resolve.c — CPU ORACLE (test infrastructure) of the VSM shadow resolve: RendererInstance::resolve_shadowmap
 * (Passes/Shadowmaps.cpp:756-822, called at RendererInstance.cpp:974-988), a fullscreen pass of passes/resolve_shadowmaps.slang:27-209
 * with the rmvsm.slang helpers it calls.  Same rules as oxc_oracle.c: plain C11, IEEE binary32 with round to nearest, no
 * contraction, IEEE divide / sqrt, dot(a, b) = (a.x*b.x + a.y*b.y) + a.z*b.z, mul(M, v) row by row in the same order.  It is one
 * translation unit with oxc_oracle.c and oxc_oracle_vsm.c, included below, so that it runs the page marking's own unproject and
 * log2.  Built into liboxc_oracle_vsm_resolve.so by oracle/pyoracle_vsm_resolve.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_vsm_resolve.c -lm
 *
 * SPECIFICATION of orc_vsm_resolve_shadows (include/oxcull.h oxc_vsm_resolve_shadows repeats it).  Where the reference does not define
 * an outcome, this commits to one:
 *   1. pixel position: input.position.xy = (x + 0.5, y + 0.5), tex_coord = position / depth_extent, as k_vsm_mark_visible_pages
 *      (oxc_oracle.c orc_mark_visible_pages).  depth == 0 (sky) gives 1.0 (:193-196).
 *   2. normal: the decode's uv_normal plane, oct(world normal) in .zw, is what the reference stores in normal_attachment.ba
 *      (visbuffer_decode.slang:170), an R16G16B16A16Sfloat image (RendererInstance.cpp:709-716): both components are rounded to
 *      binary16 (round to nearest even) before oct_to_vec3 (common/encoding.slang:7-15, which normalizes); :199 normalizes again.
 *      Pixels the decode discards hold 0, as the cleared attachment does.
 *   3. world position: unproject of (tex_coord * 2 - 1, depth) (:201-203 == scene.slang:189-193).
 *   4. clipmap selection: exactly the page-marking rule (rmvsm.slang:156-188 with canonical_log2, bias, ceil, saturating u32, clamp).
 *   5. sin / cos: the reference calls the driver's sin / cos under fast-math, which are not bit-defined.  Here: orc_sincos_canonical
 *      (== oxc_exact.cuh canonical_sincos): binary64 reduction k = rint(x * 2/pi), r = (x - k*PIO2_HI) - k*PIO2_LO with a
 *      33-bit PIO2_HI (k*PIO2_HI exact for |k| < 2^20), Taylor polynomials of sin to r^15 and cos to r^16 in Horner form, quadrant
 *      k mod 4, one rounding to binary32.  Bound: <= 1 ulp of the binary32 result for x in [0, 2 pi] (the sample angles), <= 2^-24
 *      absolute for |x| <= 2^21 (hash2 reaches 1.43e6 at 3840 x 2160).  Non-finite x gives NaN.
 *   6. other helpers: hammersley2d(i, N) = (i / N, reversebits(i) * 2^-32); fract(x) = x - floor(x); lerp(a, b, t) = a + (b - a) * t;
 *      pow(2, k + 1) exact; normalize(v) = v / sqrt(dot(v, v)); cross in component order; base_bias = (quantize + b) + term;
 *      accum_depth_world summed in sample order; max / min (HLSL) return the other operand when one is NaN (IEEE maxNum / minNum)
 *      and b when equal.
 *   7. out-of-range reads: clipmap indices -1 and clipmap_count miss (:37-39); page coordinates outside the table miss; a page that
 *      is not Backed misses; a fetched depth equal to -1.0 is a miss (the shader compares the value).  Deviation: a physical address
 *      whose texel lies outside the atlas reads 0.0, what robustImageAccess returns (the draw does not write such a texel).
 */
#include "oxc_oracle.c"
#define to_i32_f32 vsm_to_i32_f32 /* oxc_oracle_vsm.c has its own copy of this helper */
#include "oxc_oracle_vsm.c"
#undef to_i32_f32

#include "oxc_oracle_vsm_resolve.h"

#define RS_BLOCKER_SAMPLES 16u /* :19-23 */
#define RS_PCF_SAMPLES 24u
#define RS_BLOCKER_SEARCH_RADIUS 0.1f
#define RS_LIGHT_WIDTH 0.002f
#define RS_MAX_PCF_RADIUS 0.1f
#define RS_DEPTH_MISS (-1.0f) /* :25 */
#define RS_TAU 6.28318548f    /* common/math.slang:5 as binary32 */

static float rs_max(float a, float b) { return (b != b || a > b) ? a : b; }
static float rs_min(float a, float b) { return (b != b || a < b) ? a : b; }
static float rs_fract(float x) { return x - floorf(x); }
static float rs_dot3(float ax, float ay, float az, float bx, float by, float bz) { return (ax * bx + ay * by) + az * bz; }

void orc_sincos_canonical(float xf, float* s_out, float* c_out) {
  const double x = (double)xf;
  if (!(x - x == 0.0)) { *s_out = *c_out = xf - xf; return; }
  const double k = rint(x * 0.63661977236758134308);
  const double r = (x + -(k * 1.57079632673412561417e+00)) + -(k * 6.07710050650619224932e-11);
  const double z = r * r;
  double ps = -7.6471637318198164759e-13;
  ps = 1.6059043836821614599e-10 + z * ps;
  ps = -2.5052108385441718775e-08 + z * ps;
  ps = 2.7557319223985890653e-06 + z * ps;
  ps = -1.9841269841269841270e-04 + z * ps;
  ps = 8.3333333333333333333e-03 + z * ps;
  ps = -1.6666666666666666667e-01 + z * ps;
  const double sn = r + (r * z) * ps;
  double pc = 4.7794773323873852974e-14;
  pc = -1.1470745597729724714e-11 + z * pc;
  pc = 2.0876756987868098979e-09 + z * pc;
  pc = -2.7557319223985890653e-07 + z * pc;
  pc = 2.4801587301587301587e-05 + z * pc;
  pc = -1.3888888888888888889e-03 + z * pc;
  pc = 4.1666666666666666667e-02 + z * pc;
  pc = -0.5 + z * pc;
  const double cs = 1.0 + z * pc;
  const int q = (int)(k + -(4.0 * floor(k * 0.25)));
  const double sv = q == 0 ? sn : (q == 1 ? cs : (q == 2 ? -sn : -cs));
  const double cv = q == 0 ? cs : (q == 1 ? -sn : (q == 2 ? -cs : sn));
  *s_out = (float)sv;
  *c_out = (float)cv;
}

static double rs_ulp(float f) { /* spacing of binary32 values at |f| */
  const float a = fabsf(f);
  if (a < 1.17549435e-38f) return 1.40129846e-45;
  return (double)nextafterf(a, INFINITY) - (double)a;
}

static void rs_error_of(float x, double out[4]) {
  float s, c;
  orc_sincos_canonical(x, &s, &c);
  const double es = fabs((double)s - sin((double)x)), ec = fabs((double)c - cos((double)x));
  if (es > out[0]) out[0] = es;
  if (ec > out[1]) out[1] = ec;
  const double us = es / rs_ulp((float)sin((double)x)), uc = ec / rs_ulp((float)cos((double)x));
  if (us > out[2]) out[2] = us;
  if (uc > out[3]) out[3] = uc;
}

void orc_sincos_error_scan(uint32_t lo, uint32_t hi, uint32_t stride, double out[4]) {
  out[0] = out[1] = out[2] = out[3] = 0.0;
  for (uint64_t b = lo; b <= hi; b += stride ? stride : 1u) rs_error_of(bits2f((uint32_t)b), out);
}

void orc_sincos_error_list(const float* x, uint64_t n, double out[4]) {
  out[0] = out[1] = out[2] = out[3] = 0.0;
  for (uint64_t i = 0; i < n; i++) rs_error_of(x[i], out);
}

/* common/math.slang:189-191 */
void orc_hammersley2d(uint32_t i, uint32_t n, float out[2]) {
  uint32_t v = 0;
  for (int k = 0; k < 32; k++) v |= ((i >> k) & 1u) << (31 - k); /* reversebits */
  out[0] = (float)i / (float)n;
  out[1] = (float)v * 2.3283064365386963e-10f;
}

/* :27-30 */
void orc_vsm_hash2(float px, float py, float out[2]) {
  const float d0 = px * 127.1f + py * 311.7f, d1 = px * 269.5f + py * 183.3f;
  float s, c;
  orc_sincos_canonical(d0, &s, &c);
  out[0] = rs_fract(s * 43758.5453f);
  orc_sincos_canonical(d1, &s, &c);
  out[1] = rs_fract(s * 43758.5453f);
}

/* :77-82 */
void orc_vsm_perpendicular_basis(const float L[3], float out[6]) {
  const int y_axis = fabsf(L[1]) < 0.999f;
  const float ax = y_axis ? 0.0f : 1.0f, ay = y_axis ? 1.0f : 0.0f, az = 0.0f;
  const float cx = ay * L[2] - az * L[1], cy = az * L[0] - ax * L[2], cz = ax * L[1] - ay * L[0]; /* cross(axis, L) */
  const float len = sqrtf(rs_dot3(cx, cy, cz, cx, cy, cz));
  const float tx = cx / len, ty = cy / len, tz = cz / len;
  out[0] = tx; out[1] = ty; out[2] = tz;
  out[3] = L[1] * tz - L[2] * ty; out[4] = L[2] * tx - L[0] * tz; out[5] = L[0] * ty - L[1] * tx; /* cross(L, t) */
}

/* common/encoding.slang:7-15 on binary16-rounded input (spec 2) */
float orc_round_to_half(float f) {
  const uint32_t u = f2bits(f), sign = u & 0x80000000u, a = u & 0x7FFFFFFFu;
  if (a >= 0x7F800000u) return f;
  if (a >= 0x38800000u) { /* normal binary16: round the 23-bit fraction to 10 bits, ties to even */
    const uint32_t r = (a + 0xFFFu + ((a >> 13) & 1u)) & ~0x1FFFu;
    return bits2f(sign | (r > 0x477FE000u ? 0x7F800000u : r));
  }
  const float m = rintf(bits2f(a) * 16777216.0f); /* subnormal binary16: a multiple of 2^-24 */
  return bits2f(sign | f2bits(m * 5.9604644775390625e-08f));
}

typedef struct RsCtx {
  const OxcVsmContext* vsm;
  const OxcVirtualClipmap* clipmaps;
  const uint32_t* page_tables;
  const float* atlas;
  float texel_length;
} RsCtx;

/* rmvsm.slang:214-221 get_clipmap_info */
static void rs_clipmap_info(const OxcVirtualClipmap* cm, float x, float y, float z, float* cu, float* cv, float* pd) {
  const Vec4_f32 p = {x, y, z, 1.0f};
  const Vec4_f32 h = mul_mv_f32(cm->projection_view_mat, p);
  *cu = (h.x / h.w + 1.0f) * 0.5f;
  *cv = (h.y / h.w + 1.0f) * 0.5f;
  *pd = h.z / h.w;
}

/* :32-61 sample_vsm_shadow_depth */
static float rs_sample(const RsCtx* g, int32_t ci, float x, float y, float z) {
  const OxcVsmContext* vsm = g->vsm;
  if (ci < 0 || ci >= vsm->clipmap_count) return RS_DEPTH_MISS;
  const OxcVirtualClipmap* cm = &g->clipmaps[ci];
  float cu, cv, pd;
  rs_clipmap_info(cm, x, y, z, &cu, &cv, &pd);
  if (cu < 0.0f || cv < 0.0f || cu > 1.0f || cv > 1.0f) return RS_DEPTH_MISS; /* rmvsm.slang:200-203 (NaN passes) */
  const int32_t size = vsm->page_table_size;
  const int32_t vx = vsm_to_i32_f32(floorf(cu * (float)size)), vy = vsm_to_i32_f32(floorf(cv * (float)size)); /* :205 */
  if (vx < 0 || vy < 0 || vx > size - 1 || vy > size - 1) return RS_DEPTH_MISS;                          /* :129-133 */
  int32_t wx, wy;
  if (!vsm_wrap(vx, cm->page_offset[0], size, &wx) || !vsm_wrap(vy, cm->page_offset[1], size, &wy)) return RS_DEPTH_MISS;
  const uint32_t e = g->page_tables[((size_t)ci * size + (size_t)wy) * size + (size_t)wx];
  if (!(e & VSM_BACKED)) return RS_DEPTH_MISS;                                                          /* :51-53 */
  const int32_t P = vsm->physical_page_table_size, ps = vsm->page_size;
  const uint32_t n = (uint32_t)(P / ps), addr = e >> 16;                                                 /* rmvsm.slang:99-106 */
  const float tx = (float)vsm_to_i32_f32(floorf(cu * (float)P)), ty = (float)vsm_to_i32_f32(floorf(cv * (float)P)); /* :56 */
  const float fps = (float)ps;
  const int32_t ix = (int32_t)(tx - fps * floorf(tx / fps)), iy = (int32_t)(ty - fps * floorf(ty / fps));  /* :57 com::mod */
  const int64_t ax = (int64_t)(addr % n) * ps + ix, ay = (int64_t)(addr / n) * ps + iy;                 /* :55, 58 */
  if (ax < 0 || ay < 0 || ax >= P || ay >= P) return 0.0f;                                               /* robustImageAccess */
  return g->atlas[(size_t)ay * P + (size_t)ax];
}

/* :63-75 */
static float rs_sample_fallback(const RsCtx* g, int32_t ci, float x, float y, float z) {
  const float d0 = rs_sample(g, ci, x, y, z);
  if (d0 != RS_DEPTH_MISS) return d0;
  const float d1 = rs_sample(g, ci - 1, x, y, z);
  if (d1 != RS_DEPTH_MISS) return d1;
  const float d2 = rs_sample(g, ci + 1, x, y, z);
  if (d2 != RS_DEPTH_MISS) return d2;
  return RS_DEPTH_MISS;
}

/* rmvsm.slang:147-154 */
static float rs_texel_length(const OxcVsmContext* vsm) {
  const float scale_ratio = (float)(vsm->page_table_size - 1) / (float)vsm->page_table_size;
  const float effective_width = vsm->first_clipmap_width * scale_ratio;
  return (effective_width * 2.0f) / vsm->virtual_extent;
}

/* :94-98 */
static float rs_base_bias(float cts, float nol, const float N[3], const float L[3]) {
  const float sqrt2 = 1.41421356f, quantize = 2.0f / (float)(1 << 23);
  const float b = sqrt2 * cts * 0.5f;
  float term = b;
  if (nol < 0.99f) {
    const float cx = N[1] * L[2] - N[2] * L[1], cy = N[2] * L[0] - N[0] * L[2], cz = N[0] * L[1] - N[1] * L[0];
    term = b * sqrtf(rs_dot3(cx, cy, cz, cx, cy, cz)) / rs_max(nol, 0.1f);
  }
  return (quantize + b) + term;
}

float orc_vsm_base_bias(const OxcVsmContext* vsm, int32_t ci, const float N[3]) {
  const float* L = vsm->directional_light_dir;
  const float nol = rs_max(rs_dot3(N[0], N[1], N[2], L[0], L[1], L[2]), 0.0f);
  const float cts = (float)(1 << (ci + 1)) * rs_texel_length(vsm);
  return rs_base_bias(cts, nol, N, L);
}

/* one tap of :118-127 / :160-169 */
static float rs_tap(const RsCtx* g, const float B[6], int32_t ci, const float o[3], const float h[2], float nx, float ny, float radius,
                    float nol, float base_bias, float inv_z, float* bias_norm) {
  const float xi_x = rs_fract(h[0] + nx), xi_y = rs_fract(h[1] + ny);
  const float r = sqrtf(xi_x) * radius;
  const float theta = xi_y * RS_TAU;
  float s, c;
  orc_sincos_canonical(theta, &s, &c);
  const float dx = r * (B[0] * c + B[3] * s), dy = r * (B[1] * c + B[4] * s), dz = r * (B[2] * c + B[5] * s);
  const float pcf_bias = 2.0f * r;
  *bias_norm = inv_z * (base_bias + (pcf_bias + (0.0f - pcf_bias) * nol)); /* lerp(pcf_bias, 0, NoL) */
  return rs_sample_fallback(g, ci, o[0] + dx, o[1] + dy, o[2] + dz);
}

/* :84-185 pcss_shadow */
static float rs_pcss(const RsCtx* g, int32_t ci, const float W[3], const float N[3], const float noise[2], int* ran_pcf) {
  const OxcVsmContext* vsm = g->vsm;
  const float* L = vsm->directional_light_dir;
  const float nol = rs_max(rs_dot3(N[0], N[1], N[2], L[0], L[1], L[2]), 0.0f);
  const float cts = (float)(1 << (ci + 1)) * g->texel_length; /* pow(2.0, f32(ci + 1)): exact */
  const float base_bias = rs_base_bias(cts, nol, N, L);
  const float inv_z = 1.0f / vsm->z_length;
  const float now = cts * (1.0f + 2.0f * (1.0f - nol));
  const float o[3] = {W[0] + N[0] * now, W[1] + N[1] * now, W[2] + N[2] * now};
  float B[6];
  orc_vsm_perpendicular_basis(L, B);
  float cu, cv, d_recv;
  rs_clipmap_info(&g->clipmaps[ci], o[0], o[1], o[2], &cu, &cv, &d_recv);
  const float d_recv_world = d_recv * vsm->z_length;
  const float center = rs_sample_fallback(g, ci, o[0], o[1], o[2]);
  float accum = 0.0f;
  uint32_t blockers = 0, valid = 0;
  for (uint32_t i = 0; i < RS_BLOCKER_SAMPLES; i++) {
    float h[2], bias_norm;
    orc_hammersley2d(i, RS_BLOCKER_SAMPLES, h);
    const float d = rs_tap(g, B, ci, o, h, noise[0], noise[1], RS_BLOCKER_SEARCH_RADIUS, nol, base_bias, inv_z, &bias_norm);
    if (d == RS_DEPTH_MISS) continue;
    valid++;
    if (d + bias_norm < d_recv) { accum = accum + d * vsm->z_length; blockers++; }
  }
  const float hard_bias_norm = inv_z * base_bias;
  const float hard = center == RS_DEPTH_MISS ? 1.0f : ((center + hard_bias_norm < d_recv) ? 0.0f : 1.0f);
  if (valid == 0u) return hard;
  if (blockers == 0u) return 1.0f;
  if (blockers == valid) return 0.0f;
  *ran_pcf = 1;
  const float d_blocker_world = accum / (float)blockers;
  const float radius = rs_min(RS_MAX_PCF_RADIUS, (d_recv_world - d_blocker_world) * RS_LIGHT_WIDTH);
  float lit = 0.0f;
  uint32_t valid_pcf = 0;
  for (uint32_t i = 0; i < RS_PCF_SAMPLES; i++) {
    float h[2], bias_norm;
    orc_hammersley2d(i, RS_PCF_SAMPLES, h);
    const float d = rs_tap(g, B, ci, o, h, noise[1], noise[0], radius, nol, base_bias, inv_z, &bias_norm); /* noise.yx */
    if (d == RS_DEPTH_MISS) continue;
    valid_pcf++;
    if (d + bias_norm >= d_recv) lit = lit + 1.0f;
  }
  if (valid_pcf == 0u) return hard;
  return lit / (float)valid_pcf;
}

uint64_t orc_vsm_resolve_shadows(const OxcVsmContext* vsm, const float inv_pv[16], const float resolution[2], const OxcVirtualClipmap* clipmaps,
                                 const float* depth, const float* normals, const uint32_t* page_tables, const float* atlas, float* shadow,
                                 uint8_t* pcf) {
  const int32_t Wd = vsm->depth_extent[0], Hd = vsm->depth_extent[1];
  RsCtx g = {vsm, clipmaps, page_tables, atlas, rs_texel_length(vsm)};
  uint64_t n_pcf = 0;
  for (int32_t y = 0; y < Hd; y++)
    for (int32_t x = 0; x < Wd; x++) {
      const size_t pix = (size_t)y * Wd + x;
      int ran = 0;
      float out = 1.0f;
      const float d = depth[pix];
      if (d != 0.0f) { /* :193-196 */
        /* :198-199 */
        const float ex = orc_round_to_half(normals[pix * 4 + 2]), ey = orc_round_to_half(normals[pix * 4 + 3]);
        float v[3] = {ex, ey, (1.0f - fabsf(ex)) - fabsf(ey)};
        const float sx = v[0] >= 0.0f ? 1.0f : -1.0f, sy = v[1] >= 0.0f ? 1.0f : -1.0f;
        if (v[2] < 0.0f) { v[0] = (1.0f - fabsf(ey)) * sx; v[1] = (1.0f - fabsf(ex)) * sy; }
        const float l0 = sqrtf(rs_dot3(v[0], v[1], v[2], v[0], v[1], v[2]));
        const float u0 = v[0] / l0, u1 = v[1] / l0, u2 = v[2] / l0;
        const float l1 = sqrtf(rs_dot3(u0, u1, u2, u0, u1, u2));
        const float N[3] = {u0 / l1, u1 / l1, u2 / l1};
        const float px = (float)x + 0.5f, py = (float)y + 0.5f;
        const float u = px / (float)Wd, vv = py / (float)Hd;
        const Vec4_f32 wp = unproject_uv_h(inv_pv, u, vv, d); /* :201-203 */
        const float W[3] = {wp.x, wp.y, wp.z};
        /* :205 get_clipmap_index: orc_mark_visible_pages' rule */
        const float ox = (1.0f / resolution[0]) * 0.5f, oy = (1.0f / resolution[1]) * 0.5f;
        const Vec4_f32 a = unproject_uv_h(inv_pv, u - ox, vv + oy, d), b = unproject_uv_h(inv_pv, u + ox, vv + oy, d);
        const float dx = a.x - b.x, dy = a.y - b.y, dz = a.z - b.z;
        const float dist = sqrtf((dx * dx + dy * dy) + dz * dz);
        float level_f = orc_log2_canonical(dist / g.texel_length);
        level_f = level_f > 0.0f ? level_f : 0.0f;
        const float lf = ceilf(vsm->clipmap_selection_bias + level_f);
        uint32_t ci = lf >= 4294967296.0f ? 0xFFFFFFFFu : (lf > 0.0f ? (uint32_t)lf : 0u);
        if (ci > (uint32_t)(vsm->clipmap_count - 1)) ci = (uint32_t)(vsm->clipmap_count - 1);
        float noise[2];
        orc_vsm_hash2(px, py, noise); /* :207 */
        out = rs_pcss(&g, (int32_t)ci, W, N, noise, &ran);
      }
      shadow[pix] = out;
      if (pcf) pcf[pix] = (uint8_t)ran;
      n_pcf += (uint64_t)ran;
    }
  return n_pcf;
}
