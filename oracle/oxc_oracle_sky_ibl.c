/*
 * oxc_oracle_sky_ibl.c — CPU ORACLE (test infrastructure) of the sky IBL cube (Passes/PBR.cpp:52-94, passes/sky_ibl.slang) with the
 * sky.slang functions it calls (get_atmosphere_illuminance_along_ray :296-322, sky_view_params_to_lut_uv :39-67), one C function per
 * shader function.  Same rules as oxc_oracle_atmosphere.c, which it includes (one translation unit, so it runs that oracle's acos, tap
 * rule, ray-sphere test and transmittance parametrisation and the library's sin / cos and binary16 rounding).  Built into
 * liboxc_oracle_sky_ibl.so by oracle/pyoracle_sky_ibl.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_sky_ibl.c -lm
 *
 * SPECIFICATION: include/oxcull.h above oxc_atmosphere_sky_ibl, items 1-5.  New here: atan2 = orc_atan2_canonical (binary64, one
 * rounding, C99 Annex F special cases); rsqrt(x) = fl(1 / fl(sqrt(x))); the per-call values (get_eye_pos, h = sqrt(fl(y * y)), beta,
 * PI - beta, up = eye / h, the normalized sun, dot(sun, (0, 1, 0))) are formed once per call, as sky_ibl_make_params does.
 */
#include "oxc_oracle_atmosphere.c"

#include "oxc_oracle_sky_ibl.h"

static const float S_UP_LIMIT = 0x1.ff7ceep-1f, S_IGN_X = 0x1.12e286p-4f, S_IGN_Y = 0x1.7e8b2p-8f, S_IGN_Z = 0x1.a7dd04p+5f,
                   S_GOLDEN = 0x1.3c6ef4p-1f, S_VDC = 0x1p-32f, S_ALPHA = 0x1.47ae14p-6f, S_SAFE_MIN = 0x1.79ca10p-67f,
                   S_SIDE_MIN = 0x1.4f8b58p-17f;

float orc_atan2_canonical(float yf, float xf) {
  const double y = (double)yf, x = (double)xf;
  const double PI_D = 3.141592653589793116, PIO2 = PI_D * 0.5, PIO4 = PI_D * 0.25;
  if (y != y || x != x) return bits2f(0x7FC00000u);
  const double ay = fabs(y), ax = fabs(x);
  const int x_neg = signbit(x) != 0;
  double r;
  if (ay == 0.0) r = x_neg ? PI_D : 0.0;
  else if (isinf(ay) && isinf(ax)) r = x_neg ? PI_D - PIO4 : PIO4;
  else if (isinf(ay) || ax == 0.0) r = PIO2;
  else if (isinf(ax)) r = x_neg ? PI_D : 0.0;
  else {
    const int swap = ay > ax;
    const double t = swap ? ax / ay : ay / ax;
    const int reduce = t > 0.41421356237309503;
    const double u = reduce ? (t - 1.0) / (t + 1.0) : t;
    const double z = u * u;
    double p = -1.0 / 45.0;
    for (int k = 21; k >= 1; k--) p = ((k & 1) ? 1.0 : -1.0) / (double)(2 * k + 1) + z * p;
    double a = u - (u * z) * p;
    if (reduce) a = PIO4 + a;
    r = swap ? PIO2 - a : a;
    if (x_neg) r = PI_D - r;
  }
  return (float)(signbit(y) ? -r : r);
}

void orc_atan2_canonical_array(const float* y, const float* x, float* out, uint64_t n) {
  for (uint64_t i = 0; i < n; i++) out[i] = orc_atan2_canonical(y[i], x[i]);
}

static void s_cross(const float a[3], const float b[3], float o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
static void s_normalize(const float v[3], float o[3]) {
  const float l = a_length(v);
  for (int i = 0; i < 3; i++) o[i] = v[i] / l;
}
static float s_frac(float x) { return x - floorf(x); }
static float s_sanitize(float x) { return isfinite(x) ? x : 0.0f; }
static float s_saturate(float x) { return a_min(a_max(x, 0.0f), 1.0f); }

/* orc_atm_tap's rule, all four channels */
void orc_sky_ibl_tap4(const uint16_t* lut, uint32_t W, uint32_t H, float u, float v, float out[4]) {
  const float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = x - x0, wy = y - y0;
  const int64_t ix = alpha_f2i(x0), iy = alpha_f2i(y0);
  const int64_t xa = a_clampi(ix, W), xb = a_clampi(ix + 1, W), ya = a_clampi(iy, H), yb = a_clampi(iy + 1, H);
  for (int c = 0; c < 4; c++) {
    const float a00 = g_half_float(lut[(ya * W + xa) * 4 + c]), a10 = g_half_float(lut[(ya * W + xb) * 4 + c]);
    const float a01 = g_half_float(lut[(yb * W + xa) * 4 + c]), a11 = g_half_float(lut[(yb * W + xb) * 4 + c]);
    const float top = a00 + wx * (a10 - a00), bot = a01 + wx * (a11 - a01);
    out[c] = top + wy * (bot - top);
  }
}

/* sky_ibl.slang:21-30, :67-68 */
static const float S_FACE[6][9] = {{+0, +0, -1, +0, -1, +0, -1, +0, +0}, {+0, +0, +1, +0, -1, +0, +1, +0, +0},
                                   {+1, +0, +0, +0, +0, -1, +0, +1, +0}, {+1, +0, +0, +0, +0, +1, +0, -1, +0},
                                   {+1, +0, +0, +0, -1, +0, +0, +0, -1}, {-1, +0, +0, +0, -1, +0, +0, +0, +1}};
void orc_sky_ibl_dir(uint32_t face, uint32_t x, uint32_t y, float out[3]) {
  const float uv[2] = {((float)x + 0.5f) / 32.0f, ((float)y + 0.5f) / 32.0f};
  const float v[3] = {uv[0] * 2.0f - 1.0f, uv[1] * 2.0f - 1.0f, -1.0f};
  const float* m = S_FACE[face < 5 ? face : 5];
  const float mv[3] = {a_dot(m, v), a_dot(m + 3, v), a_dot(m + 6, v)};
  s_normalize(mv, out);
}

/* sky_ibl.slang:32-44 */
float orc_sky_ibl_radical_inverse(uint32_t bits) {
  bits = (bits << 16u) | (bits >> 16u);
  bits = ((bits & 0x55555555u) << 1u) | ((bits & 0xAAAAAAAAu) >> 1u);
  bits = ((bits & 0x33333333u) << 2u) | ((bits & 0xCCCCCCCCu) >> 2u);
  bits = ((bits & 0x0F0F0F0Fu) << 4u) | ((bits & 0xF0F0F0F0u) >> 4u);
  bits = ((bits & 0x00FF00FFu) << 8u) | ((bits & 0xFF00FF00u) >> 8u);
  return (float)bits * S_VDC;
}
float orc_sky_ibl_ign(float px, float py) { return s_frac(S_IGN_Z * s_frac(px * S_IGN_X + py * S_IGN_Y)); }

/* the per-call values */
typedef struct SkyCall {
  const OxcAtmosphere* at;
  float eye[3], height, beta, zenith_horizon, up[3], sun[3];
} SkyCall;
static SkyCall s_call(const OxcAtmosphere* at, float camera_y, const float sun[3]) {
  SkyCall c;
  c.at = at;
  c.eye[0] = 0.0f; c.eye[1] = orc_atm_eye_y(at, camera_y); c.eye[2] = 0.0f;
  c.height = a_length(c.eye);
  const float horizon = a_safe_sqrt(c.height * c.height - at->planet_radius * at->planet_radius);
  c.beta = orc_acos_canonical(horizon / c.height);
  c.zenith_horizon = A_PI - c.beta;
  for (int i = 0; i < 3; i++) c.up[i] = c.eye[i] / c.height;
  s_normalize(sun, c.sun);
  return c;
}

/* sky.slang:39-67 */
static void s_sky_view_uv(const SkyCall* c, int intersect_planet, float view_zenith_cos_angle, const float light_on_plane[2], float uv[2]) {
  const float view_zenith_angle = orc_acos_canonical(view_zenith_cos_angle);
  if (!intersect_planet) {
    float coord = view_zenith_angle / c->zenith_horizon;
    coord = 1.0f - coord;
    coord = a_safe_sqrt(coord);
    coord = 1.0f - coord;
    uv[1] = coord * 0.5f;
  } else {
    float coord = (view_zenith_angle - c->zenith_horizon) / c->beta;
    coord = a_safe_sqrt(coord);
    uv[1] = coord * 0.5f + 0.5f;
  }
  const float theta = orc_atan2_canonical(-light_on_plane[1], -light_on_plane[0]);
  uv[0] = (theta + A_PI) / A_TAU;
  const float rw = (float)c->at->sky_view_lut_size[0], rh = (float)c->at->sky_view_lut_size[1];
  uv[0] = (uv[0] + 0.5f / rw) * (rw / (rw + 1.0f));
  uv[1] = (uv[1] + 0.5f / rh) * (rh / (rh + 1.0f));
}

/* sky.slang:296-322 */
static void s_illuminance(const SkyCall* c, const uint16_t* sky_view, const float eye_dir[3], float out[3]) {
  const float view_zenith_cos_angle = a_dot(eye_dir, c->up);
  float side_raw[3], side[3], fw_raw[3], forward[3];
  s_cross(c->up, eye_dir, side_raw);
  if (a_length(side_raw) > S_SIDE_MIN) s_normalize(side_raw, side);
  else { side[0] = 1.0f; side[1] = 0.0f; side[2] = 0.0f; }
  s_cross(side, c->up, fw_raw);
  s_normalize(fw_raw, forward);
  float lop[2] = {a_dot(c->sun, forward), a_dot(c->sun, side)};
  const float len_sq = lop[0] * lop[0] + lop[1] * lop[1];
  if (len_sq > S_SAFE_MIN) {
    const float rs = 1.0f / sqrtf(len_sq);
    lop[0] = lop[0] * rs; lop[1] = lop[1] * rs;
  } else {
    lop[0] = 1.0f; lop[1] = 0.0f;
  }
  float t;
  const int intersect_planet = orc_atm_ray_sphere_nearest(c->eye, eye_dir, c->at->planet_radius, &t);
  float uv[2], s[4];
  s_sky_view_uv(c, intersect_planet, view_zenith_cos_angle, lop, uv);
  orc_sky_ibl_tap4(sky_view, c->at->sky_view_lut_size[0], c->at->sky_view_lut_size[1], uv[0], uv[1], s);
  for (int i = 0; i < 3; i++) out[i] = s_sanitize(s[i] * s[3]);
}

void orc_sky_ibl_illuminance(const OxcAtmosphere* at, float camera_y, const float sun[3], const uint16_t* sky_view, const float eye_dir[3],
                             float out[3]) {
  const SkyCall c = s_call(at, camera_y, sun);
  s_illuminance(&c, sky_view, eye_dir, out);
}

/* sky_ibl.slang:46-52 */
void orc_sky_ibl_local_sample(uint32_t i, float rotation, float out[3]) {
  const float u1 = ((float)i + 0.5f) / 64.0f;
  const float u2 = s_frac(orc_sky_ibl_radical_inverse(i) + rotation);
  const float r = sqrtf(u1);
  const float phi = A_TAU * u2;
  float sn, cs;
  orc_sincos_canonical(phi, &sn, &cs);
  out[0] = r * cs;
  out[1] = r * sn;
  out[2] = sqrtf(a_max(0.0f, 1.0f - u1));
}

/* sky_ibl.slang:54-116 for texel (x, y) of `face` */
static void s_texel(const SkyCall* c, const float sun_raw[3], float sun_intensity, float sun_ambient_strength, uint32_t frame_index,
                    const uint16_t* tlut, const uint16_t* sky_view, uint32_t face, uint32_t x, uint32_t y, uint16_t* cube) {
  float dir[3], tangent[3], bitangent[3], tr[3];
  orc_sky_ibl_dir(face, x, y, dir);
  const float up_y[3] = {0.0f, 1.0f, 0.0f}, up_x[3] = {1.0f, 0.0f, 0.0f};
  s_cross(fabsf(dir[1]) < S_UP_LIMIT ? up_y : up_x, dir, tr);
  s_normalize(tr, tangent);
  s_cross(dir, tangent, bitangent);
  const size_t texel = ((size_t)face * 32 + y) * 32 + x;
  float history[4];
  for (int i = 0; i < 4; i++) history[i] = g_half_float(cube[texel * 4 + i]);
  const int has_history = history[3] > 0.0f && isfinite(history[0]) && isfinite(history[1]) && isfinite(history[2]);
  const float base_rotation = orc_sky_ibl_ign((float)x + (float)face * 37.0f, (float)y + (float)face * 17.0f);
  const float rotation = has_history ? s_frac(base_rotation + (float)frame_index * S_GOLDEN) : base_rotation;
  float frame_sum[3] = {0.0f, 0.0f, 0.0f};
  for (uint32_t i = 0; i < 64; i++) {
    float local[3], input_dir[3], in_raw[3], sample[3];
    orc_sky_ibl_local_sample(i, rotation, local);
    for (int k = 0; k < 3; k++) in_raw[k] = (local[0] * tangent[k] + local[1] * bitangent[k]) + local[2] * dir[k];
    s_normalize(in_raw, input_dir);
    s_illuminance(c, sky_view, input_dir, sample);
    for (int k = 0; k < 3; k++) frame_sum[k] += s_sanitize(sample[k]);
  }
  const float sun_cos_zenith = a_dot(sun_raw, up_y);
  float tuv[2], sun_color[4];
  orc_atm_transmittance_uv(c->at->atmos_radius, c->at->planet_radius, c->eye[1], sun_cos_zenith, tuv);
  orc_sky_ibl_tap4(tlut, c->at->transmittance_lut_size[0], c->at->transmittance_lut_size[1], tuv[0], tuv[1], sun_color);
  const float sun_facing = s_saturate(a_dot(dir, sun_raw));
  float out[3];
  for (int k = 0; k < 3; k++) {
    const float sun_term = sun_ambient_strength * sun_color[k] * sun_intensity * sun_facing / A_PI;
    const float frame_result = a_min(a_max(s_sanitize(frame_sum[k] / 64.0f + sun_term), 0.0f), A_HALF_MAX);
    out[k] = has_history ? history[k] + (frame_result - history[k]) * S_ALPHA : frame_result;
  }
  a_store(cube, texel, out[0], out[1], out[2], 1.0f);
}

void orc_atmosphere_sky_ibl(const OxcAtmosphere* at, const OxcPbrCamera* cam, const float sun[3], float sun_intensity,
                            float sun_ambient_strength, uint32_t frame_index, const uint16_t* transmittance, const uint16_t* sky_view,
                            uint16_t* cube) {
  const SkyCall c = s_call(at, cam->position[1], sun);
  for (uint32_t face = 0; face < 6; face++)
    for (uint32_t y = 0; y < 32; y++)
      for (uint32_t x = 0; x < 32; x++)
        s_texel(&c, sun, sun_intensity, sun_ambient_strength, frame_index, transmittance, sky_view, face, x, y, cube);
}
