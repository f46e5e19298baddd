/*
 * oxc_oracle_atmosphere.c — CPU ORACLE (test infrastructure) of the atmosphere's lookup tables: the transmittance bake
 * (RendererInstance.cpp:203-226, passes/sky_transmittance.slang) and the per-frame sky view and aerial perspective (Passes/PBR.cpp:11-50
 * and :96-140, passes/sky_view.slang, passes/sky_aerial_perspective.slang), with the sky.slang, common/math.slang and scene.slang
 * functions they call, one C function per shader function, in the shaders' structure.  Only the path these call sites take is restated:
 * eval_multiscattering and eval_planet_luminance are false (the multiple-scattering LUT is bound but never sampled), the aerial
 * perspective's dead start_depth / start_pos / ray_pos are left out (view_height is reassigned before they are read).  Same rules as
 * oxc_oracle.c: plain C11, IEEE binary32 with round to nearest, no contraction, IEEE divide / sqrt, sums and products in written order,
 * dot(a, b) = (a.x*b.x + a.y*b.y) + a.z*b.z, normalize(v) = v / length(v), lerp(a, b, t) = a + (b - a) * t, max / min return the
 * other operand for a NaN.  It is one translation unit with oxc_oracle_gtao.c (and so the resolve oracle and oxc_oracle.c), included
 * below, so that it runs the library's own pow, sin / cos, alpha_f2i and binary16 rounding.  Built into liboxc_oracle_atmosphere.so by
 * oracle/pyoracle_atmosphere.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_atmosphere.c -lm
 *
 * SPECIFICATION (include/oxcull.h oxc_atmosphere_transmittance repeats it).  Where the shaders do not define an outcome, this commits to:
 *   1. exp = orc_exp_canonical (binary32 Cody-Waite, below); cos = orc_sincos_canonical; pow(x, 3/2) = orc_pow_canonical(x, 1.5);
 *      acos = orc_acos_canonical (binary64, one rounding).  beta, get_eye_pos and the four exps of mie_asymmetry are constant per call
 *      and computed once (atmosphere_make_params on the library's side).
 *   2. Constants: PI 0x40490FDB, TAU 0x40C90FDB, 1 / (4 PI) = fl(1 / fl(4 * PI)) = 0x3DA2F983 and 3 / (16 PI) = fl(3 / fl(16 * PI)) =
 *      0x3D747645 (Slang folds 1.0 / (4.0 * PI) with PI a binary32 constant: 4 * PI and 16 * PI are exact, and one correctly rounded
 *      division gives the same bits whether it is folded in binary32 or in binary64 and rounded once), alpha * (1.0 / 3.0) with
 *      1.0 / 3.0 = 0x3EAAAAAB, 3.0 / 2.0 = 1.5, CAMERA_SCALE_UNIT 0x3C23D70A, PLANET_RADIUS_OFFSET 0x3A83126F, HALF_MIN_NORMAL 0x38800000,
 *      HALF_MAX 0x477FE000, the aerial perspective's f32x3(1.0 / 3.0) 0x3EAAAAAB.
 *   3. h = length((0, y, 0)) = sqrt(fl(y * y)), not |y|; the sky view's up_vec = moved eye_pos / h with h from before the move.
 *   4. Optional<f32>::value of `none` reads 0 (only the bake reads it unchecked; a record with atmos_radius below planet_radius, or NaN
 *      radii, reaches it).
 *   5. the MS * scattering_sum term is kept with MS = 0 (NaN for an infinite sum; +0 + -0 = +0).
 *   6. the transmittance tap: bilinear with binary32 weights over the binary16 texels (the GTAO's level tap, no 8-bit weights).
 *   7. every stored channel: binary16, round to nearest even, subnormals kept, every NaN 0x7FFF.
 *   8. max(NaN, 0) = 0 in the sky view's max(luminance, 0); sanitize replaces +-inf by 0.
 *   9. per_slice_depth = f32(size.x / size.z) in integers.
 */
#include "oxc_oracle_gtao.c"

#include "oxc_oracle_atmosphere.h"

static const float A_PI = 0x1.921fb6p+1f, A_TAU = 0x1.921fb6p+2f, A_INV_4PI = 0x1.45f306p-4f, A_RAYLEIGH_K = 0x1.e8ec8ap-5f,
                   A_THIRD = 0x1.555556p-2f, A_CSU = 0x1.47ae14p-7f, A_PRO = 0x1.0624dep-10f, A_HALF_MIN_NORMAL = 6.103515625e-5f,
                   A_HALF_MAX = 65504.0f;

static float a_max(float a, float b) { return (b != b || a > b) ? a : b; }
static float a_min(float a, float b) { return (b != b || a < b) ? a : b; }
static float a_safe_sqrt(float x) { return sqrtf(a_max(0.0f, x)); }
static float a_dot(const float a[3], const float b[3]) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
static float a_length(const float a[3]) { return sqrtf(a_dot(a, a)); }
static int64_t a_clampi(int64_t i, int64_t n) { return i < 0 ? 0 : (i > n - 1 ? n - 1 : i); }

static float a_pow2(int k) { return bits2f((uint32_t)(k + 127) << 23); }

float orc_exp_canonical(float x) {
  if (x != x) return x;
  if (x > 89.0f) return a_pow2(127) * a_pow2(127);
  if (x < -104.0f) return 0.0f;
  const float k = rintf(x * 1.44269502f);
  const float r = (x - k * 0.693359375f) - k * -2.12194440e-4f;
  float q = 2.48015873e-05f;
  q = 1.98412701e-04f + r * q;
  q = 1.38888892e-03f + r * q;
  q = 8.33333377e-03f + r * q;
  q = 4.16666679e-02f + r * q;
  q = 1.66666672e-01f + r * q;
  q = 0.5f + r * q;
  const float p = 1.0f + (r + (r * r) * q);
  const int ki = (int)k;
  if (ki > 127) return (p * a_pow2(127)) * a_pow2(ki - 127);
  if (ki < -126) return (p * a_pow2(ki + 100)) * a_pow2(-100);
  return p * a_pow2(ki);
}

void orc_exp_canonical_array(const float* x, float* out, uint64_t n) {
  for (uint64_t i = 0; i < n; i++) out[i] = orc_exp_canonical(x[i]);
}

float orc_acos_canonical(float xf) {
  const double x = (double)xf;
  if (!(x >= -1.0 && x <= 1.0)) return bits2f(0x7FC00000u);
  const double a = x < 0.0 ? -x : x;
  const double s = a <= 0.5 ? x : sqrt((1.0 - a) * 0.5);
  double c[29];
  double central = 1.0;
  for (int n = 0; n < 29; n++) {
    if (n > 0) central = central * (double)(2 * n - 1) / (double)(2 * n);
    c[n] = central / (double)(2 * n + 1);
  }
  const double z = s * s;
  double p = c[28];
  for (int n = 27; n >= 1; n--) p = c[n] + z * p;
  const double as = s + (s * z) * p;
  const double PI_D = 3.141592653589793116;
  if (a <= 0.5) return (float)(PI_D * 0.5 - as);
  return (float)(x > 0.0 ? 2.0 * as : PI_D - 2.0 * as);
}

void orc_acos_canonical_array(const float* x, float* out, uint64_t n) {
  for (uint64_t i = 0; i < n; i++) out[i] = orc_acos_canonical(x[i]);
}

/* binary16 bits of a stored channel (spec 7) */
uint16_t orc_atm_half(float f) { return f != f ? (uint16_t)0x7FFFu : g_half_bits(f); }

/* common/math.slang:104-138; returns 0 for `none` and leaves *t untouched */
int orc_atm_ray_sphere_nearest(const float o[3], const float d[3], float radius, float* t) {
  const float a = a_dot(d, d);
  const float b = 2.0f * a_dot(d, o);
  const float c = a_dot(o, o) - radius * radius;
  const float delta = b * b - 4.0f * a * c;
  if (delta < 0.0f) return 0;
  const float sq = sqrtf(delta);
  const float sol0 = (-b + -1.0f * sq) / (2.0f * a), sol1 = (-b + 1.0f * sq) / (2.0f * a);
  if (sol0 < 0.0f && sol1 < 0.0f) return 0;
  if (sol0 < 0.0f) *t = a_max(0.0f, sol1);
  else if (sol1 < 0.0f) *t = a_max(0.0f, sol0);
  else *t = a_max(0.0f, a_min(sol0, sol1));
  return 1;
}

/* sky.slang:15-29 */
void orc_atm_transmittance_uv(float atmos_radius, float planet_radius, float px, float py, float out[2]) {
  const float h = a_safe_sqrt(atmos_radius * atmos_radius - planet_radius * planet_radius);
  const float rho = a_safe_sqrt(px * px - planet_radius * planet_radius);
  const float discriminant = px * px * (py * py - 1.0f) + atmos_radius * atmos_radius;
  const float d = a_max(0.0f, -px * py + a_safe_sqrt(discriminant));
  const float d_min = atmos_radius - px;
  const float d_max = rho + h;
  out[0] = (d - d_min) / (d_max - d_min);
  out[1] = rho / h;
}

/* common/math.slang:28-31, :58-71 */
float orc_atm_rayleigh_phase(float c) { return A_RAYLEIGH_K * (1.0f + c * c); }
static float a_draine(float alpha, float g, float c) {
  return (A_INV_4PI * ((1.0f - (g * g)) / orc_pow_canonical((1.0f + (g * g) - (2.0f * g * c)), 1.5f))) *
         ((1.0f + (alpha * c * c)) / (1.0f + (alpha * A_THIRD * (1.0f + (2.0f * g * g)))));
}
void orc_atm_hg_draine_constants(float g, float out[4]) {
  out[0] = orc_exp_canonical(-(0.0990567f / (g - 1.67154f)));
  out[1] = orc_exp_canonical(-(2.20679f / (g + 3.91029f)) - 0.428934f);
  out[2] = orc_exp_canonical(3.62489f - (8.29288f / (g + 5.52825f)));
  out[3] = orc_exp_canonical(-(0.599085f / (g - 0.641583f)) - 0.665888f);
}
float orc_atm_mie_phase(float g, float c) {
  float k[4];
  orc_atm_hg_draine_constants(g, k);
  const float a = a_draine(0.0f, k[0], c), b = a_draine(k[2], k[1], c);
  return a + (b - a) * k[3];
}

/* sky.slang:119-150 */
typedef struct AtmMedium {
  float rayleigh_scattering[3], mie_scattering[3], scattering_sum[3], extinction_sum[3];
} AtmMedium;
static AtmMedium a_medium(const OxcAtmosphere* at, float altitude) {
  const float rayleigh_density = orc_exp_canonical(-altitude / at->rayleigh_density);
  const float mie_density = orc_exp_canonical(-altitude / at->mie_density);
  const float ozone_density = a_max(0.0f, 1.0f - fabsf(altitude - at->ozone_height) / at->ozone_thickness);
  AtmMedium m;
  const float mie_extinction = at->mie_extinction * mie_density;
  for (int i = 0; i < 3; i++) {
    m.rayleigh_scattering[i] = at->rayleigh_scatter[i] * rayleigh_density;
    m.mie_scattering[i] = at->mie_scatter[i] * mie_density;
    const float ozone = at->ozone_absorption[i] * ozone_density;
    m.scattering_sum[i] = m.rayleigh_scattering[i] + m.mie_scattering[i];
    m.extinction_sum[i] = m.rayleigh_scattering[i] + mie_extinction + ozone;
  }
  return m;
}
void orc_atm_medium_extinction(const OxcAtmosphere* at, float altitude, float out[3]) {
  const AtmMedium m = a_medium(at, altitude);
  for (int i = 0; i < 3; i++) out[i] = m.extinction_sum[i];
}

/* SampleLevel(linear_clamp, uv, 0).rgb of a binary16 RGBA LUT (spec 6) */
void orc_atm_tap(const uint16_t* lut, uint32_t W, uint32_t H, float u, float v, float out[3]) {
  const float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = x - x0, wy = y - y0;
  const int64_t ix = alpha_f2i(x0), iy = alpha_f2i(y0);
  const int64_t xa = a_clampi(ix, W), xb = a_clampi(ix + 1, W), ya = a_clampi(iy, H), yb = a_clampi(iy + 1, H);
  for (int c = 0; c < 3; c++) {
    const float a00 = g_half_float(lut[(ya * W + xa) * 4 + c]), a10 = g_half_float(lut[(ya * W + xb) * 4 + c]);
    const float a01 = g_half_float(lut[(yb * W + xa) * 4 + c]), a11 = g_half_float(lut[(yb * W + xb) * 4 + c]);
    const float top = a00 + wx * (a10 - a00), bot = a01 + wx * (a11 - a01);
    out[c] = top + wy * (bot - top);
  }
}

/* sky.slang:169-256 with eval_multiscattering = eval_planet_luminance = false: luminance and transmittance */
typedef struct AtmInfo {
  float eye_pos[3], eye_dir[3], sun_dir[3], sun_intensity, step_count, t_max;
} AtmInfo;
static void a_integrate(const AtmInfo* info, const OxcAtmosphere* at, const uint16_t* tlut, float lum[3], float trans[3]) {
  for (int i = 0; i < 3; i++) { lum[i] = 0.0f; trans[i] = 1.0f; }
  const float R = at->planet_radius;
  if (a_dot(info->eye_pos, info->eye_pos) <= R * R) return;
  float planet_t = 0.0f, atmos_t = 0.0f;
  const int planet_hit = orc_atm_ray_sphere_nearest(info->eye_pos, info->eye_dir, R, &planet_t);
  float integration_length;
  if (info->t_max == -1.0f) {
    if (!orc_atm_ray_sphere_nearest(info->eye_pos, info->eye_dir, at->atmos_radius, &atmos_t)) return;
    else if (!planet_hit) integration_length = atmos_t;
    else integration_length = a_max(0.0f, planet_t);
  } else {
    integration_length = info->t_max;
  }
  const float cos_theta = a_dot(info->sun_dir, info->eye_dir);
  const float rayleigh_phase = orc_atm_rayleigh_phase(cos_theta);
  const float mie_phase = orc_atm_mie_phase(at->mie_asymmetry, cos_theta);
  float old_ray_shift = 0.0f;
  for (float step = 0.0f; step < info->step_count; step += 1.0f) {
    const float new_ray_shift = integration_length * (step + 0.3f) / info->step_count;
    const float step_length = new_ray_shift - old_ray_shift;
    old_ray_shift = new_ray_shift;
    float step_pos[3];
    for (int i = 0; i < 3; i++) step_pos[i] = info->eye_pos[i] + new_ray_shift * info->eye_dir[i];
    const float h = a_length(step_pos);
    const float altitude = h - R;
    const AtmMedium m = a_medium(at, altitude);
    float up_vec[3], up_vec_scaled[3], shadow_origin[3];
    for (int i = 0; i < 3; i++) up_vec[i] = step_pos[i] / h;
    for (int i = 0; i < 3; i++) up_vec_scaled[i] = A_PRO * up_vec[i];
    const float sun_theta = a_dot(info->sun_dir, up_vec);
    float uv[2], sun_transmittance[3];
    orc_atm_transmittance_uv(at->atmos_radius, R, h, sun_theta, uv);
    orc_atm_tap(tlut, at->transmittance_lut_size[0], at->transmittance_lut_size[1], uv[0], uv[1], sun_transmittance);
    for (int i = 0; i < 3; i++) shadow_origin[i] = step_pos[i] - up_vec_scaled[i];
    float shadow_t;
    const float earth_shadow = orc_atm_ray_sphere_nearest(shadow_origin, info->sun_dir, R, &shadow_t) ? 0.0f : 1.0f;
    for (int i = 0; i < 3; i++) {
      const float scattering_phase = m.mie_scattering[i] * mie_phase + m.rayleigh_scattering[i] * rayleigh_phase;
      const float MS = 0.0f;
      const float sun_luminance = earth_shadow * sun_transmittance[i] * scattering_phase + (MS * m.scattering_sum[i]);
      const float step_transmittance = orc_exp_canonical(-step_length * m.extinction_sum[i]);
      const float integral = (sun_luminance - sun_luminance * step_transmittance) / m.extinction_sum[i];
      lum[i] += info->sun_intensity * (integral * trans[i]);
      trans[i] *= step_transmittance;
    }
  }
}

/* sky.slang:104-117 */
static int a_move_to_top(float pos[3], const float dir[3], float atmos_radius) {
  const float h = a_length(pos);
  if (h > atmos_radius) {
    float t;
    if (orc_atm_ray_sphere_nearest(pos, dir, atmos_radius, &t)) {
      for (int i = 0; i < 3; i++) {
        const float up_vec = pos[i] / h;
        const float up_offset = up_vec * -A_PRO;
        pos[i] = pos[i] + dir[i] * t + up_offset;
      }
    } else {
      return 0;
    }
  }
  return 1;
}

/* scene.slang:229-233 Atmosphere::get_eye_pos(position).y */
float orc_atm_eye_y(const OxcAtmosphere* at, float camera_y) {
  const float min_altitude = at->planet_radius + A_PRO;
  return a_max(camera_y * A_CSU + min_altitude, min_altitude);
}

/* sky.slang:7-9 */
static float a_from_sub_uv(float uv, float res) { return (uv - 0.5f / res) * (res / (res - 1.0f)); }

/* sky.slang:69-102 */
void orc_atm_sky_view_dir(const OxcAtmosphere* at, float u, float v, float altitude, float out[3]) {
  u = a_from_sub_uv(u, (float)at->sky_view_lut_size[0]);
  v = a_from_sub_uv(v, (float)at->sky_view_lut_size[1]);
  const float horizon = a_safe_sqrt(altitude * altitude - at->planet_radius * at->planet_radius);
  const float beta = orc_acos_canonical(horizon / altitude);
  const float zenith_horizon_angle = A_PI - beta;
  float view_zenith_angle = 0.0f;
  if (v < 0.5f) {
    float coord = v * 2.0f;
    coord = 1.0f - coord;
    coord *= coord;
    coord = 1.0f - coord;
    view_zenith_angle = zenith_horizon_angle * coord;
  } else {
    float coord = v * 2.0f - 1.0f;
    coord *= coord;
    view_zenith_angle = zenith_horizon_angle + beta * coord;
  }
  const float longitude_view_cos_angle = u * A_TAU;
  float s, view_zenith_cos_angle, cos_longitude;
  orc_sincos_canonical(view_zenith_angle, &s, &view_zenith_cos_angle);
  const float view_zenith_sin_angle =
      a_safe_sqrt(1.0f - view_zenith_cos_angle * view_zenith_cos_angle) * (view_zenith_angle > 0.0f ? 1.0f : -1.0f);
  orc_sincos_canonical(longitude_view_cos_angle, &s, &cos_longitude);
  const float sin_longitude = a_safe_sqrt(1.0f - cos_longitude * cos_longitude) * (longitude_view_cos_angle <= A_PI ? 1.0f : -1.0f);
  out[0] = view_zenith_sin_angle * cos_longitude;
  out[1] = view_zenith_cos_angle;
  out[2] = view_zenith_sin_angle * sin_longitude;
}

static void a_store(uint16_t* plane, size_t texel, float r, float g, float b, float a) {
  plane[texel * 4 + 0] = orc_atm_half(r);
  plane[texel * 4 + 1] = orc_atm_half(g);
  plane[texel * 4 + 2] = orc_atm_half(b);
  plane[texel * 4 + 3] = orc_atm_half(a);
}

/* passes/sky_transmittance.slang:31-45 for the texel's (lut_x, lut_y): exp(-optical_depth) before the binary16 store */
void orc_atm_transmittance_ray(const OxcAtmosphere* at, float lut_x, float lut_y, float out[3]) {
  const float sun_dir[3] = {0.0f, sqrtf(1.0f - lut_y * lut_y), lut_y};
  float ray_pos[3] = {0.0f, 0.0f, lut_x};
  const float STEP_COUNT = 1000.0f;
  float distance = 0.0f; /* spec 4: `none`.value reads 0 */
  orc_atm_ray_sphere_nearest(ray_pos, sun_dir, at->atmos_radius, &distance);
  const float distance_per_step = distance / STEP_COUNT;
  float optical_depth[3] = {0.0f, 0.0f, 0.0f};
  for (float i = 0.0f; i < STEP_COUNT; i += 1.0f) {
    for (int k = 0; k < 3; k++) ray_pos[k] += sun_dir[k] * distance_per_step;
    const float ray_altitude = a_length(ray_pos) - at->planet_radius;
    const AtmMedium m = a_medium(at, ray_altitude);
    for (int k = 0; k < 3; k++) optical_depth[k] += m.extinction_sum[k] * distance_per_step;
  }
  for (int k = 0; k < 3; k++) out[k] = orc_exp_canonical(-optical_depth[k]);
}

/* passes/sky_transmittance.slang:19-30: the (lut_x, lut_y) = (height, cos theta) of texel (x, y) */
void orc_atm_transmittance_params(const OxcAtmosphere* at, uint32_t x, uint32_t y, float out[2]) {
  const uint32_t W = at->transmittance_lut_size[0], H = at->transmittance_lut_size[1];
  const float u = ((float)x + 0.5f) / (float)W, v = ((float)y + 0.5f) / (float)H;
  const float h = a_safe_sqrt(at->atmos_radius * at->atmos_radius - at->planet_radius * at->planet_radius);
  const float rho = h * v;
  const float lut_x = sqrtf(rho * rho + at->planet_radius * at->planet_radius);
  const float d_min = at->atmos_radius - lut_x;
  const float d_max = rho + h;
  const float d = d_min + u * (d_max - d_min);
  float lut_y = d == 0.0f ? 1.0f : (h * h - rho * rho - d * d) / (2.0f * lut_x * d);
  out[0] = lut_x;
  out[1] = a_min(a_max(lut_y, -1.0f), 1.0f);
}

/* passes/sky_transmittance.slang:19-45 */
void orc_atmosphere_transmittance(const OxcAtmosphere* at, uint16_t* lut) {
  const uint32_t W = at->transmittance_lut_size[0], H = at->transmittance_lut_size[1];
  for (uint32_t y = 0; y < H; y++)
    for (uint32_t x = 0; x < W; x++) {
      float params[2], t[3];
      orc_atm_transmittance_params(at, x, y, params);
      orc_atm_transmittance_ray(at, params[0], params[1], t);
      a_store(lut, (size_t)y * W + x, t[0], t[1], t[2], 1.0f);
    }
}

/* passes/sky_view.slang:23-51 */
static void a_sky_view_texel(const OxcAtmosphere* at, const float camera_pos[3], const float sun[3], float sun_intensity,
                             const uint16_t* tlut, uint32_t x, uint32_t y, uint16_t* out) {
  const size_t texel = (size_t)y * at->sky_view_lut_size[0] + x;
  const float u = ((float)x + 0.5f) / (float)at->sky_view_lut_size[0], v = ((float)y + 0.5f) / (float)at->sky_view_lut_size[1];
  float eye_pos[3] = {0.0f, orc_atm_eye_y(at, camera_pos[1]), 0.0f};
  const float h = a_length(eye_pos);
  float eye_dir[3];
  orc_atm_sky_view_dir(at, u, v, h, eye_dir);
  if (!a_move_to_top(eye_pos, eye_dir, at->atmos_radius)) {
    a_store(out, texel, 0.0f, 0.0f, 0.0f, 0.0f);
    return;
  }
  const float up_vec[3] = {eye_pos[0] / h, eye_pos[1] / h, eye_pos[2] / h};
  const float sun_zenith_cos_angle = a_dot(sun, up_vec);
  const float sd[3] = {a_safe_sqrt(1.0f - sun_zenith_cos_angle * sun_zenith_cos_angle), sun_zenith_cos_angle, 0.0f};
  const float sl = a_length(sd);
  AtmInfo info;
  for (int i = 0; i < 3; i++) { info.eye_pos[i] = eye_pos[i]; info.eye_dir[i] = eye_dir[i]; info.sun_dir[i] = sd[i] / sl; }
  info.sun_intensity = sun_intensity;
  info.step_count = 48.0f;
  info.t_max = -1.0f;
  float lum[3], trans[3];
  a_integrate(&info, at, tlut, lum, trans);
  float l[3];
  for (int i = 0; i < 3; i++) {
    l[i] = a_max(lum[i], 0.0f);
    if (fabsf(l[i]) == INFINITY) l[i] = 0.0f; /* sanitize */
  }
  const float max_luminance = a_max(l[0], a_max(l[1], l[2]));
  const float mult = a_min(a_max(max_luminance, A_HALF_MIN_NORMAL), A_HALF_MAX);
  a_store(out, texel, l[0] / mult, l[1] / mult, l[2] / mult, mult);
}

/* passes/sky_aerial_perspective.slang:25-79 */
static void a_aerial_texel(const OxcAtmosphere* at, const OxcPbrCamera* cam, const float sun[3], float sun_intensity, const uint16_t* tlut,
                           uint32_t x, uint32_t y, uint32_t z, uint16_t* out) {
  const uint32_t X = at->aerial_perspective_lut_size[0], Y = at->aerial_perspective_lut_size[1], Z = at->aerial_perspective_lut_size[2];
  const size_t texel = ((size_t)z * Y + y) * X + x;
  const float u = ((float)x + 0.5f) / (float)X, v = ((float)y + 0.5f) / (float)Y;
  const float cs[4] = {2.0f * u - 1.0f, 2.0f * v - 1.0f, 1.0f, 1.0f};
  const float* m = cam->inv_projection_view;
  float ws[4];
  for (int i = 0; i < 4; i++) ws[i] = ((m[i] * cs[0] + m[4 + i] * cs[1]) + m[8 + i] * cs[2]) + m[12 + i] * cs[3];
  const float world_pos[3] = {ws[0] / ws[3], ws[1] / ws[3], ws[2] / ws[3]};
  const float wd[3] = {world_pos[0] - cam->position[0], world_pos[1] - cam->position[1], world_pos[2] - cam->position[2]};
  const float wl = a_length(wd);
  const float world_dir[3] = {wd[0] / wl, wd[1] / wl, wd[2] / wl};
  float eye_pos[3] = {0.0f, orc_atm_eye_y(at, cam->position[1]), 0.0f};
  float slice = (((float)z + 0.5f) * (1.0f / (float)Z));
  slice *= slice;
  slice *= (float)Z;
  const float per_slice_depth = (float)(X / Z); /* spec 9 */
  const float t_max = slice * per_slice_depth;
  float t_max_max = t_max;
  const float view_height = a_length(eye_pos);
  if (view_height >= at->atmos_radius) {
    const float prev_ray_pos[3] = {eye_pos[0], eye_pos[1], eye_pos[2]};
    if (!a_move_to_top(eye_pos, world_dir, at->atmos_radius)) {
      a_store(out, texel, 0.0f, 0.0f, 0.0f, 0.0f);
      return;
    }
    const float dd[3] = {prev_ray_pos[0] - eye_pos[0], prev_ray_pos[1] - eye_pos[1], prev_ray_pos[2] - eye_pos[2]};
    const float length_to_atmosphere = a_length(dd);
    if (t_max_max < length_to_atmosphere) {
      a_store(out, texel, 0.0f, 0.0f, 0.0f, 0.0f);
      return;
    }
    t_max_max = a_max(0.0f, t_max_max - length_to_atmosphere);
  }
  AtmInfo info;
  for (int i = 0; i < 3; i++) { info.eye_pos[i] = eye_pos[i]; info.eye_dir[i] = world_dir[i]; info.sun_dir[i] = sun[i]; }
  info.sun_intensity = sun_intensity;
  info.step_count = a_max(1.0f, ((float)z + 1.0f) * 2.0f);
  info.t_max = t_max_max;
  float lum[3], trans[3];
  a_integrate(&info, at, tlut, lum, trans);
  const float third[3] = {A_THIRD, A_THIRD, A_THIRD};
  a_store(out, texel, lum[0], lum[1], lum[2], a_dot(trans, third));
}

void orc_atmosphere_sky_view(const OxcAtmosphere* at, const OxcPbrCamera* cam, const float sun[3], float sun_intensity, const uint16_t* tlut,
                             uint16_t* out) {
  for (uint32_t y = 0; y < at->sky_view_lut_size[1]; y++)
    for (uint32_t x = 0; x < at->sky_view_lut_size[0]; x++) a_sky_view_texel(at, cam->position, sun, sun_intensity, tlut, x, y, out);
}

void orc_atmosphere_aerial_perspective(const OxcAtmosphere* at, const OxcPbrCamera* cam, const float sun[3], float sun_intensity,
                                       const uint16_t* tlut, uint16_t* out) {
  for (uint32_t z = 0; z < at->aerial_perspective_lut_size[2]; z++)
    for (uint32_t y = 0; y < at->aerial_perspective_lut_size[1]; y++)
      for (uint32_t x = 0; x < at->aerial_perspective_lut_size[0]; x++) a_aerial_texel(at, cam, sun, sun_intensity, tlut, x, y, z, out);
}
