// oxc_atmosphere.cuh — the atmosphere's lookup tables, one texel at a time: passes/sky_transmittance.slang (the init-time bake),
// passes/sky_view.slang and passes/sky_aerial_perspective.slang (the per-frame LUTs), with the sky.slang and common/math.slang functions
// they call, on the path those call sites take: eval_multiscattering and eval_planet_luminance false (the MS term is kept as 0 *
// scattering_sum, see atm_integrate), the aerial perspective's dead start_depth / start_pos / ray_pos left out.  Pure per-thread
// functions: no warp intrinsics, no shared memory, so tests compile this source for the host.
// Specification: include/oxcull.h (comment above oxc_atmosphere_transmittance) == oracle/oxc_oracle_atmosphere.c, operation for
// operation.
#pragma once
#include "oxc_shader_math.cuh"

namespace oxc {

// binary32 roundings of the shaders' constants (bits pinned by tests/test_oracle_atmosphere.py)
constexpr float ATM_TAU = 0x1.921fb6p+2f;   // 0x40C90FDB, :5
constexpr float ATM_INV_4PI = 0x1.45f306p-4f; // 0x3DA2F983 = fl(1 / fl(4 * PI)), :59 (4 * PI is exact)
constexpr float ATM_RAYLEIGH_K = 0x1.e8ec8ap-5f; // 0x3D747645 = fl(3 / fl(16 * PI)), :29 (16 * PI is exact)
constexpr float ATM_THIRD = 0x1.555556p-2f;   // 0x3EAAAAAB = fl(1 / 3), :61 and sky_aerial_perspective.slang:79
constexpr float ATM_CAMERA_SCALE_UNIT = 0x1.47ae14p-7f; // 0x3C23D70A, scene.slang:6
constexpr float ATM_PLANET_RADIUS_OFFSET = 0x1.0624dep-10f; // 0x3A83126F, scene.slang:8
constexpr float ATM_HALF_MIN_NORMAL = 6.103515625e-5f;       // 0x38800000, common/math.slang:77
constexpr float ATM_HALF_MAX = 65504.0f;                     // 0x477FE000, :76
constexpr uint16_t ATM_HALF_NAN = 0x7FFFu;                   // every NaN a LUT stores
constexpr uint16_t ATM_HALF_ONE = 0x3C00u;
constexpr int ATM_TRANSMITTANCE_STEPS = 1000;                // sky_transmittance.slang:34
constexpr int ATM_SKY_VIEW_STEPS = 48;                       // sky_view.slang:43

struct AtmosphereParams {
  // the record's fields the passes read
  float rayleigh_scatter[3], rayleigh_density;
  float mie_scatter[3], mie_density, mie_extinction;
  float ozone_absorption[3], ozone_height, ozone_thickness;
  float planet_radius, atmos_radius;
  int t_w, t_h;                // transmittance_lut_size.xy
  int sv_w, sv_h;              // sky_view_lut_size.xy
  int ap_w, ap_h, ap_d;        // aerial_perspective_lut_size
  // per-dispatch values, computed once by atmosphere_make_params
  float hg[4];                 // henyey_greenstein_draine_phase's g_hg, g_d, alpha, w_d (common/math.slang:65-68)
  float eye_y;                 // Atmosphere::get_eye_pos(camera position).y (scene.slang:229-233)
  float eye_h;                 // length(eye_pos) = sqrt(eye_y * eye_y)
  float beta, zenith_horizon;  // uv_to_sky_view_lut_params' beta = acos(horizon / eye_h) and PI - beta (sky.slang:75-77)
  float per_slice_depth;       // f32(lut_size.x / lut_size.z) in integers (sky_aerial_perspective.slang:38)
  float sun[3], sun_intensity; // the push constants, as given
  float4 inv_pv_row[4];        // rows of Camera::inv_projection_view
  float cam_pos[3];
  const uint16_t* transmittance; // the transmittance LUT the per-frame passes tap (binary16 RGBA)
  uint16_t* out_transmittance;
  uint16_t* out_sky_view;
  uint16_t* out_aerial;
  uint32_t sky_view_blocks;    // k_atmosphere_sky_luts: CTAs [0, sky_view_blocks) write the sky view, the rest the aerial perspective
};

// the kernels' parameters from the C ABI's arguments (oxc_atmosphere_transmittance / oxc_atmosphere_sky_luts, and the host build of the
// tests); camera and sun may be NULL for the bake, which reads neither
__host__ inline AtmosphereParams atmosphere_make_params(const OxcAtmosphere& a, const OxcPbrCamera* cam, const float* sun, float sun_intensity,
                                                        const uint16_t* transmittance, uint16_t* out_transmittance, uint16_t* out_sky_view,
                                                        uint16_t* out_aerial, uint32_t block) {
  AtmosphereParams p{};
  for (int i = 0; i < 3; i++) {
    p.rayleigh_scatter[i] = a.rayleigh_scatter[i]; p.mie_scatter[i] = a.mie_scatter[i]; p.ozone_absorption[i] = a.ozone_absorption[i];
  }
  p.rayleigh_density = a.rayleigh_density; p.mie_density = a.mie_density; p.mie_extinction = a.mie_extinction;
  p.ozone_height = a.ozone_height; p.ozone_thickness = a.ozone_thickness;
  p.planet_radius = a.planet_radius; p.atmos_radius = a.atmos_radius;
  p.t_w = (int)a.transmittance_lut_size[0]; p.t_h = (int)a.transmittance_lut_size[1];
  p.sv_w = (int)a.sky_view_lut_size[0]; p.sv_h = (int)a.sky_view_lut_size[1];
  p.ap_w = (int)a.aerial_perspective_lut_size[0]; p.ap_h = (int)a.aerial_perspective_lut_size[1]; p.ap_d = (int)a.aerial_perspective_lut_size[2];
  // common/math.slang:65-68, the four exps of mie_asymmetry
  const float g = a.mie_asymmetry;
  p.hg[0] = canonical_exp(-(0.0990567f / (g - 1.67154f)));
  p.hg[1] = canonical_exp(-(2.20679f / (g + 3.91029f)) - 0.428934f);
  p.hg[2] = canonical_exp(3.62489f - (8.29288f / (g + 5.52825f)));
  p.hg[3] = canonical_exp(-(0.599085f / (g - 0.641583f)) - 0.665888f);
  if (cam) {
    // scene.slang:229-233 get_eye_pos, then length((0, y, 0)) = sqrt((0 * 0 + y * y) + 0 * 0) = sqrt(y * y)
    const float min_altitude = a.planet_radius + ATM_PLANET_RADIUS_OFFSET;
    p.eye_y = vmax(cam->position[1] * ATM_CAMERA_SCALE_UNIT + min_altitude, min_altitude);
    p.eye_h = sqrtf(p.eye_y * p.eye_y);
    // sky.slang:75-77
    const float horizon = sqrtf(vmax(0.0f, p.eye_h * p.eye_h - a.planet_radius * a.planet_radius));
    p.beta = canonical_acos(horizon / p.eye_h);
    p.zenith_horizon = PI - p.beta;
    for (int i = 0; i < 4; i++)
      p.inv_pv_row[i] = make_float4(cam->inv_projection_view[i], cam->inv_projection_view[4 + i], cam->inv_projection_view[8 + i],
                                    cam->inv_projection_view[12 + i]);
    for (int i = 0; i < 3; i++) p.cam_pos[i] = cam->position[i];
  }
  if (sun)
    for (int i = 0; i < 3; i++) p.sun[i] = sun[i];
  p.sun_intensity = sun_intensity;
  p.per_slice_depth = p.ap_d > 0 ? (float)(p.ap_w / p.ap_d) : 0.0f;
  p.transmittance = transmittance; p.out_transmittance = out_transmittance; p.out_sky_view = out_sky_view; p.out_aerial = out_aerial;
  p.sky_view_blocks = block;
  return p;
}

OXC_DI float atm_safe_sqrt(float x) { return fsq(vmax(0.0f, x)); } // common/math.slang:79-81

// common/math.slang:104-138 ray_sphere_intersect_nearest; false for `none`
OXC_DI bool atm_ray_sphere_nearest(Vec3 o, Vec3 d, float radius, float& t) {
  const float a = vdot(d, d);
  const float b = fm(2.0f, vdot(d, o));
  const float c = fs(vdot(o, o), fm(radius, radius));
  const float delta = fs(fm(b, b), fm(fm(4.0f, a), c));
  if (delta < 0.0f) return false;
  const float sq = fsq(delta);
  const float two_a = fm(2.0f, a);
  const float sol0 = fd(fa(-b, -sq), two_a), sol1 = fd(fa(-b, sq), two_a);
  if (sol0 < 0.0f && sol1 < 0.0f) return false;
  if (sol0 < 0.0f) t = vmax(0.0f, sol1);
  else if (sol1 < 0.0f) t = vmax(0.0f, sol0);
  else t = vmax(0.0f, vmin(sol0, sol1));
  return true;
}

// sky.slang:15-29
OXC_DI void atm_transmittance_uv(float atmos_radius, float planet_radius, float px, float py, float& mu, float& r) {
  const float h = atm_safe_sqrt(fs(fm(atmos_radius, atmos_radius), fm(planet_radius, planet_radius)));
  const float rho = atm_safe_sqrt(fs(fm(px, px), fm(planet_radius, planet_radius)));
  const float discriminant = fa(fm(fm(px, px), fs(fm(py, py), 1.0f)), fm(atmos_radius, atmos_radius));
  const float d = vmax(0.0f, fa(fm(-px, py), atm_safe_sqrt(discriminant)));
  const float d_min = fs(atmos_radius, px);
  const float d_max = fa(rho, h);
  mu = fd(fs(d, d_min), fs(d_max, d_min));
  r = fd(rho, h);
}

// sky.slang:119-150 MediumScattering: the scattering and extinction sums
struct AtmMedium {
  Vec3 rayleigh_scattering, mie_scattering, scattering_sum, extinction_sum;
};
OXC_DI AtmMedium atm_medium(const AtmosphereParams& p, float altitude) {
  const float rayleigh_density = canonical_exp(fd(-altitude, p.rayleigh_density));
  const float mie_density = canonical_exp(fd(-altitude, p.mie_density));
  const float ozone_density = vmax(0.0f, fs(1.0f, fd(fabsf(fs(altitude, p.ozone_height)), p.ozone_thickness)));
  AtmMedium m;
  m.rayleigh_scattering = vscale(vec3(p.rayleigh_scatter[0], p.rayleigh_scatter[1], p.rayleigh_scatter[2]), rayleigh_density);
  m.mie_scattering = vscale(vec3(p.mie_scatter[0], p.mie_scatter[1], p.mie_scatter[2]), mie_density);
  const float mie_extinction = fm(p.mie_extinction, mie_density);
  const Vec3 ozone = vscale(vec3(p.ozone_absorption[0], p.ozone_absorption[1], p.ozone_absorption[2]), ozone_density);
  m.scattering_sum = vadd(m.rayleigh_scattering, m.mie_scattering);
  m.extinction_sum = vadd(vadd(m.rayleigh_scattering, vec3(mie_extinction, mie_extinction, mie_extinction)), ozone);
  return m;
}

// binary16 bits of a stored channel: round to nearest even, subnormals kept, every NaN 0x7FFF
OXC_DI uint16_t atm_half(float f) { return f != f ? ATM_HALF_NAN : half_bits(f); }
OXC_DI void atm_store(uint16_t* plane, size_t texel, float r, float g, float b, float a) {
  const uint2 v = make_uint2((uint32_t)atm_half(r) | ((uint32_t)atm_half(g) << 16), (uint32_t)atm_half(b) | ((uint32_t)atm_half(a) << 16));
  *reinterpret_cast<uint2*>(plane + texel * 4) = v;
}

// transmittance_image.SampleLevel(linear_clamp, (mu, r), 0).rgb of the binary16 LUT: x = u * W - 0.5, x0 = floor(x), wx = x - x0 (y
// likewise), texels x0, x0 + 1 / y0, y0 + 1 with NaN-safe saturating indices clamped to the edge, top = a00 + wx * (a10 - a00), bottom
// likewise, top + wy * (bottom - top): the GTAO's level tap without the 8-bit weight quantisation
OXC_DI Vec3 atm_tap_transmittance(const AtmosphereParams& p, float u, float v) {
  const int w = p.t_w, h = p.t_h;
  const float x = fs(fm(u, (float)w), 0.5f), y = fs(fm(v, (float)h), 0.5f);
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = fs(x, x0), wy = fs(y, y0);
  const long long ix = sat_i32(x0), iy = sat_i32(y0);
  const int xa = clamp_index(ix, w), xb = clamp_index(ix + 1, w), ya = clamp_index(iy, h), yb = clamp_index(iy + 1, h);
  const uint2* t = reinterpret_cast<const uint2*>(p.transmittance);
  const uint2 q00 = __ldg(t + (size_t)ya * w + xa), q10 = __ldg(t + (size_t)ya * w + xb);
  const uint2 q01 = __ldg(t + (size_t)yb * w + xa), q11 = __ldg(t + (size_t)yb * w + xb);
  float out[3];
  for (int c = 0; c < 3; c++) {
    const int sh = (c & 1) * 16;
    const float a00 = half_float((uint16_t)(((c < 2) ? q00.x : q00.y) >> sh)), a10 = half_float((uint16_t)(((c < 2) ? q10.x : q10.y) >> sh));
    const float a01 = half_float((uint16_t)(((c < 2) ? q01.x : q01.y) >> sh)), a11 = half_float((uint16_t)(((c < 2) ? q11.x : q11.y) >> sh));
    const float top = fa(a00, fm(wx, fs(a10, a00))), bot = fa(a01, fm(wx, fs(a11, a01)));
    out[c] = fa(top, fm(wy, fs(bot, top)));
  }
  return vec3(out[0], out[1], out[2]);
}

// common/math.slang:58-62 draine_phase, 3/2 folded to 1.5, alpha * (1.0 / 3.0) with 1.0 / 3.0 folded to fl(1/3)
OXC_DI float atm_draine(float alpha, float g, float c) {
  const float gg = fm(g, g), g2 = fm(2.0f, g);
  const float num = fd(fs(1.0f, gg), canonical_pow(fs(fa(1.0f, gg), fm(g2, c)), 1.5f));
  const float shape = fd(fa(1.0f, fm(fm(alpha, c), c)), fa(1.0f, fm(fm(alpha, ATM_THIRD), fa(1.0f, fm(g2, g)))));
  return fm(fm(ATM_INV_4PI, num), shape);
}

// sky.slang:169-256 integrate_single_scattered_luminance with eval_multiscattering = eval_planet_luminance = false; t_max = -1 takes the
// atmosphere's exit.  Returns the luminance and the transmittance (multiscattering_as_1 feeds no output and is not computed).  The MS
// term of sun_luminance stays as 0 * scattering_sum: it is NaN for an infinite or NaN sum and turns a -0 luminance into +0.
OXC_DI void atm_integrate(const AtmosphereParams& p, Vec3 eye_pos, Vec3 eye_dir, Vec3 sun_dir, float step_count, float t_max,
                          Vec3& luminance, Vec3& transmittance) {
  luminance = vec3(0.0f, 0.0f, 0.0f);
  transmittance = vec3(1.0f, 1.0f, 1.0f);
  const float R = p.planet_radius;
  if (vdot(eye_pos, eye_pos) <= fm(R, R)) return;
  float planet_t = 0.0f, atmos_t = 0.0f;
  const bool planet_hit = atm_ray_sphere_nearest(eye_pos, eye_dir, R, planet_t);
  float integration_length;
  if (t_max == -1.0f) {
    if (!atm_ray_sphere_nearest(eye_pos, eye_dir, p.atmos_radius, atmos_t)) return;
    integration_length = planet_hit ? vmax(0.0f, planet_t) : atmos_t;
  } else {
    integration_length = t_max;
  }
  const float cos_theta = vdot(sun_dir, eye_dir);
  const float rayleigh_phase = fm(ATM_RAYLEIGH_K, fa(1.0f, fm(cos_theta, cos_theta)));
  const float d0 = atm_draine(0.0f, p.hg[0], cos_theta), d1 = atm_draine(p.hg[2], p.hg[1], cos_theta);
  const float mie_phase = fa(d0, fm(fs(d1, d0), p.hg[3])); // lerp(a, b, w_d)
  float old_ray_shift = 0.0f;
  for (float step = 0.0f; step < step_count; step = fa(step, 1.0f)) {
    const float new_ray_shift = fd(fm(integration_length, fa(step, 0.3f)), step_count);
    const float step_length = fs(new_ray_shift, old_ray_shift);
    old_ray_shift = new_ray_shift;
    const Vec3 step_pos = vadd(eye_pos, vscale(eye_dir, new_ray_shift));
    const float h = vlength(step_pos);
    const float altitude = fs(h, R);
    const AtmMedium m = atm_medium(p, altitude);
    const Vec3 up_vec = vnormalize(step_pos);
    const Vec3 up_vec_scaled = vscale(up_vec, ATM_PLANET_RADIUS_OFFSET); // PLANET_RADIUS_OFFSET * up_vec
    const float sun_theta = vdot(sun_dir, up_vec);
    float mu, r;
    atm_transmittance_uv(p.atmos_radius, R, h, sun_theta, mu, r);
    const Vec3 sun_transmittance = atm_tap_transmittance(p, mu, r);
    const Vec3 scattering_phase = vadd(vscale(m.mie_scattering, mie_phase), vscale(m.rayleigh_scattering, rayleigh_phase));
    float shadow_t;
    const float earth_shadow = atm_ray_sphere_nearest(vsub(step_pos, up_vec_scaled), sun_dir, R, shadow_t) ? 0.0f : 1.0f;
    const Vec3 ms = vscale(m.scattering_sum, 0.0f); // MS * scattering_sum with MS = 0
    const Vec3 sun_luminance = vadd(vmul(vscale(sun_transmittance, earth_shadow), scattering_phase), ms);
    const Vec3 step_transmittance = vec3(canonical_exp(fm(-step_length, m.extinction_sum.x)), canonical_exp(fm(-step_length, m.extinction_sum.y)),
                                         canonical_exp(fm(-step_length, m.extinction_sum.z)));
    const Vec3 integral = vec3(fd(fs(sun_luminance.x, fm(sun_luminance.x, step_transmittance.x)), m.extinction_sum.x),
                               fd(fs(sun_luminance.y, fm(sun_luminance.y, step_transmittance.y)), m.extinction_sum.y),
                               fd(fs(sun_luminance.z, fm(sun_luminance.z, step_transmittance.z)), m.extinction_sum.z));
    luminance = vadd(luminance, vscale(vmul(integral, transmittance), p.sun_intensity));
    transmittance = vmul(transmittance, step_transmittance);
  }
}

// sky.slang:104-117 move_to_top_atmosphere
OXC_DI bool atm_move_to_top(Vec3& pos, Vec3 dir, float atmos_radius) {
  const float h = vlength(pos);
  if (h > atmos_radius) {
    float t;
    if (!atm_ray_sphere_nearest(pos, dir, atmos_radius, t)) return false;
    const Vec3 up_vec = vdiv(pos, h);
    const Vec3 up_offset = vscale(up_vec, -ATM_PLANET_RADIUS_OFFSET);
    pos = vadd(vadd(pos, vscale(dir, t)), up_offset);
  }
  return true;
}

// passes/sky_transmittance.slang:19-45 for texel (x, y): the stored RGBA (exp(-optical_depth), 1)
OXC_DI void atm_transmittance_texel(const AtmosphereParams& p, int x, int y) {
  const float u = fd(fa((float)x, 0.5f), (float)p.t_w), v = fd(fa((float)y, 0.5f), (float)p.t_h);
  const float R = p.planet_radius, A = p.atmos_radius;
  const float h = atm_safe_sqrt(fs(fm(A, A), fm(R, R)));
  const float rho = fm(h, v);
  const float lut_x = fsq(fa(fm(rho, rho), fm(R, R)));
  const float d_min = fs(A, lut_x);
  const float d_max = fa(rho, h);
  const float d = fa(d_min, fm(u, fs(d_max, d_min)));
  float lut_y = d == 0.0f ? 1.0f : fd(fs(fs(fm(h, h), fm(rho, rho)), fm(d, d)), fm(fm(2.0f, lut_x), d));
  lut_y = vmin(vmax(lut_y, -1.0f), 1.0f);
  const Vec3 sun_dir = vec3(0.0f, fsq(fs(1.0f, fm(lut_y, lut_y))), lut_y);
  Vec3 ray_pos = vec3(0.0f, 0.0f, lut_x);
  float distance = 0.0f; // Optional<f32>::value of `none` reads 0
  atm_ray_sphere_nearest(ray_pos, sun_dir, A, distance);
  const float distance_per_step = fd(distance, (float)ATM_TRANSMITTANCE_STEPS);
  Vec3 optical_depth = vec3(0.0f, 0.0f, 0.0f);
  for (int i = 0; i < ATM_TRANSMITTANCE_STEPS; i++) {
    ray_pos = vadd(ray_pos, vscale(sun_dir, distance_per_step));
    const float ray_altitude = fs(vlength(ray_pos), R);
    const AtmMedium m = atm_medium(p, ray_altitude);
    optical_depth = vadd(optical_depth, vscale(m.extinction_sum, distance_per_step));
  }
  atm_store(p.out_transmittance, (size_t)y * p.t_w + x, canonical_exp(-optical_depth.x), canonical_exp(-optical_depth.y),
            canonical_exp(-optical_depth.z), 1.0f);
}

// sky.slang:69-102 uv_to_sky_view_lut_params with the dispatch's beta / zenith_horizon_angle
OXC_DI Vec3 atm_sky_view_dir(const AtmosphereParams& p, float u, float v) {
  // from_sub_uvs_to_unit (:7-9): (uv - 0.5 / res) * (res / (res - 1))
  const float rw = (float)p.sv_w, rh = (float)p.sv_h;
  u = fm(fs(u, fd(0.5f, rw)), fd(rw, fs(rw, 1.0f)));
  v = fm(fs(v, fd(0.5f, rh)), fd(rh, fs(rh, 1.0f)));
  float view_zenith_angle;
  if (v < 0.5f) {
    float coord = fm(v, 2.0f);
    coord = fs(1.0f, coord);
    coord = fm(coord, coord);
    coord = fs(1.0f, coord);
    view_zenith_angle = fm(p.zenith_horizon, coord);
  } else {
    float coord = fs(fm(v, 2.0f), 1.0f);
    coord = fm(coord, coord);
    view_zenith_angle = fa(p.zenith_horizon, fm(p.beta, coord));
  }
  const float longitude = fm(u, ATM_TAU);
  const float vz_cos = canonical_cos(view_zenith_angle);
  const float vz_sin = fm(atm_safe_sqrt(fs(1.0f, fm(vz_cos, vz_cos))), view_zenith_angle > 0.0f ? 1.0f : -1.0f);
  const float lon_cos = canonical_cos(longitude);
  const float lon_sin = fm(atm_safe_sqrt(fs(1.0f, fm(lon_cos, lon_cos))), longitude <= PI ? 1.0f : -1.0f);
  return vec3(fm(vz_sin, lon_cos), vz_cos, fm(vz_sin, lon_sin));
}

// passes/sky_view.slang:23-51 for texel (x, y)
OXC_DI void atm_sky_view_texel(const AtmosphereParams& p, int x, int y) {
  const size_t texel = (size_t)y * p.sv_w + x;
  const float u = fd(fa((float)x, 0.5f), (float)p.sv_w), v = fd(fa((float)y, 0.5f), (float)p.sv_h);
  Vec3 eye_pos = vec3(0.0f, p.eye_y, 0.0f);
  const float h = p.eye_h;
  const Vec3 eye_dir = atm_sky_view_dir(p, u, v);
  if (!atm_move_to_top(eye_pos, eye_dir, p.atmos_radius)) {
    atm_store(p.out_sky_view, texel, 0.0f, 0.0f, 0.0f, 0.0f);
    return;
  }
  const Vec3 up_vec = vdiv(eye_pos, h); // the moved position over the height before the move, as written
  const float sun_zenith_cos = vdot(vec3(p.sun[0], p.sun[1], p.sun[2]), up_vec);
  const Vec3 sun_dir = vnormalize(vec3(atm_safe_sqrt(fs(1.0f, fm(sun_zenith_cos, sun_zenith_cos))), sun_zenith_cos, 0.0f));
  Vec3 lum, trans;
  atm_integrate(p, eye_pos, eye_dir, sun_dir, (float)ATM_SKY_VIEW_STEPS, -1.0f, lum, trans);
  // sanitize(max(luminance, 0)): max returns 0 for a NaN, sanitize replaces +-inf by 0
  float l[3] = {vmax(lum.x, 0.0f), vmax(lum.y, 0.0f), vmax(lum.z, 0.0f)};
  for (int c = 0; c < 3; c++) l[c] = fabsf(l[c]) == __uint_as_float(0x7F800000u) ? 0.0f : l[c];
  const float max_luminance = vmax(l[0], vmax(l[1], l[2]));
  const float mult = vmin(vmax(max_luminance, ATM_HALF_MIN_NORMAL), ATM_HALF_MAX);
  atm_store(p.out_sky_view, texel, fd(l[0], mult), fd(l[1], mult), fd(l[2], mult), mult);
}

// passes/sky_aerial_perspective.slang:25-79 for texel (x, y, z)
OXC_DI void atm_aerial_texel(const AtmosphereParams& p, int x, int y, int z) {
  const size_t texel = ((size_t)z * p.ap_h + y) * p.ap_w + x;
  const float u = fd(fa((float)x, 0.5f), (float)p.ap_w), v = fd(fa((float)y, 0.5f), (float)p.ap_h);
  const float cx = fs(fm(2.0f, u), 1.0f), cy = fs(fm(2.0f, v), 1.0f);
  const float hw = row_dot4(p.inv_pv_row[3], cx, cy, 1.0f, 1.0f);
  const Vec3 world_pos = vec3(fd(row_dot4(p.inv_pv_row[0], cx, cy, 1.0f, 1.0f), hw), fd(row_dot4(p.inv_pv_row[1], cx, cy, 1.0f, 1.0f), hw),
                              fd(row_dot4(p.inv_pv_row[2], cx, cy, 1.0f, 1.0f), hw));
  const Vec3 world_dir = vnormalize(vsub(world_pos, vec3(p.cam_pos[0], p.cam_pos[1], p.cam_pos[2])));
  Vec3 eye_pos = vec3(0.0f, p.eye_y, 0.0f);
  const float fz = (float)p.ap_d;
  float slice = fm(fa((float)z, 0.5f), fd(1.0f, fz));
  slice = fm(slice, slice);
  slice = fm(slice, fz);
  const float t_max = fm(slice, p.per_slice_depth);
  float t_max_max = t_max;
  const float view_height = p.eye_h;
  if (view_height >= p.atmos_radius) {
    const Vec3 prev_ray_pos = eye_pos;
    if (!atm_move_to_top(eye_pos, world_dir, p.atmos_radius)) {
      atm_store(p.out_aerial, texel, 0.0f, 0.0f, 0.0f, 0.0f);
      return;
    }
    const float length_to_atmosphere = vlength(vsub(prev_ray_pos, eye_pos));
    if (t_max_max < length_to_atmosphere) {
      atm_store(p.out_aerial, texel, 0.0f, 0.0f, 0.0f, 0.0f);
      return;
    }
    t_max_max = vmax(0.0f, fs(t_max_max, length_to_atmosphere));
  }
  const float step_count = vmax(1.0f, fm(fa((float)z, 1.0f), 2.0f));
  Vec3 lum, trans;
  atm_integrate(p, eye_pos, world_dir, vec3(p.sun[0], p.sun[1], p.sun[2]), step_count, t_max_max, lum, trans);
  atm_store(p.out_aerial, texel, lum.x, lum.y, lum.z, vdot(trans, vec3(ATM_THIRD, ATM_THIRD, ATM_THIRD)));
}

} // namespace oxc
