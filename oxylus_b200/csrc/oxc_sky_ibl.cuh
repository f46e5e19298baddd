// oxc_sky_ibl.cuh — the sky IBL cube, one texel and one sample at a time: passes/sky_ibl.slang with the sky.slang functions it calls
// (get_atmosphere_illuminance_along_ray, sky_view_params_to_lut_uv) and the common/math.slang ones they call.  Pure per-thread functions:
// no warp intrinsics, no shared memory, so tests compile this source for the host; kernels_sky_ibl.cuh lays the samples out.
// Specification: include/oxcull.h (comment above oxc_atmosphere_sky_ibl) == oracle/oxc_oracle_sky_ibl.c, operation for operation.
#pragma once
#include "oxc_atmosphere.cuh"

namespace oxc {

constexpr int SKY_IBL_RES = 32;                 // IBL_CUBE_RES, sky_ibl.slang:8
constexpr int SKY_IBL_SAMPLES = 64;             // IBL_SAMPLES_PER_FRAME, :9
constexpr int SKY_IBL_TEXELS = 6 * SKY_IBL_RES * SKY_IBL_RES;
// binary32 roundings of the shaders' literals (bits pinned by tests/test_oracle_sky_ibl.py)
constexpr float SKY_IBL_UP_LIMIT = 0x1.ff7ceep-1f;     // 0x3F7FBE77 = 0.999, :72
constexpr float SKY_IBL_IGN_X = 0x1.12e286p-4f;        // 0x3D897143 = 0.06711056, :42
constexpr float SKY_IBL_IGN_Y = 0x1.7e8b2p-8f;         // 0x3BBF4590 = 0.00583715
constexpr float SKY_IBL_IGN_Z = 0x1.a7dd04p+5f;        // 0x4253EE82 = 52.9829189
constexpr float SKY_IBL_GOLDEN = 0x1.3c6ef4p-1f;       // 0x3F1E377A = 0.61803398875, :81
constexpr float SKY_IBL_VDC_SCALE = 0x1p-32f;          // 0x2F800000 = 2.3283064365386963e-10, :38
constexpr float SKY_IBL_ALPHA = 0x1.47ae14p-6f;        // 0x3CA3D70A = 0.02, :112
constexpr float SKY_IBL_SAFE_NORMALIZE_MIN = 0x1.79ca10p-67f; // 0x1E3CE508 = 1e-20, common/math.slang:92
constexpr float SKY_IBL_SIDE_MIN = 0x1.4f8b58p-17f;    // 0x3727C5AC = 1e-5, sky.slang:309

// the kernel's parameters: the atmosphere's (eye height, beta, PI - beta, the LUT sizes) and the per-call values of this pass
struct SkyIblParams {
  AtmosphereParams atm;        // atmosphere_make_params with the call's camera; atm.transmittance is the transmittance LUT
  const uint16_t* sky_view;    // the sky-view LUT (binary16 RGBA, atm.sv_w x atm.sv_h)
  uint16_t* cube;              // 6 x 32 x 32 binary16 RGBA, read and written in place
  float up[3];                 // eye_pos / length(eye_pos), sky.slang:305
  float sun[3];                // normalize(sun_dir), sky.slang:312
  float sun_raw[3];            // the sun as given: the sun term uses it unnormalized (sky_ibl.slang:101, :107)
  float sun_cos_zenith;        // dot(sun_dir, (0, 1, 0)), :101
  float sun_intensity, sun_ambient_strength;
  float frame;                 // f32(frame_index), round to nearest even
};

// the kernel's parameters from the C ABI's arguments (oxc_atmosphere_sky_ibl, and the host build of the tests)
__host__ inline SkyIblParams sky_ibl_make_params(const OxcAtmosphere& a, const OxcPbrCamera& cam, const float sun[3], float sun_intensity,
                                                 float sun_ambient_strength, uint32_t frame_index, const uint16_t* transmittance,
                                                 const uint16_t* sky_view, uint16_t* cube) {
  SkyIblParams p{};
  p.atm = atmosphere_make_params(a, &cam, sun, sun_intensity, transmittance, nullptr, nullptr, nullptr, 0);
  p.sky_view = sky_view;
  p.cube = cube;
  // eye_pos = (0, eye_y, 0), height = length(eye_pos) = eye_h
  p.up[0] = 0.0f / p.atm.eye_h; p.up[1] = p.atm.eye_y / p.atm.eye_h; p.up[2] = 0.0f / p.atm.eye_h;
  const float sl = sqrtf((sun[0] * sun[0] + sun[1] * sun[1]) + sun[2] * sun[2]);
  for (int i = 0; i < 3; i++) { p.sun[i] = sun[i] / sl; p.sun_raw[i] = sun[i]; }
  p.sun_cos_zenith = (sun[0] * 0.0f + sun[1] * 1.0f) + sun[2] * 0.0f;
  p.sun_intensity = sun_intensity;
  p.sun_ambient_strength = sun_ambient_strength;
  p.frame = (float)frame_index;
  return p;
}

OXC_DI float sib_sanitize(float x) { return fabsf(x) < __uint_as_float(0x7F800000u) ? x : 0.0f; } // isfinite ? x : 0

// SampleLevel(linear_clamp, (u, v), 0) of a w x h binary16 RGBA plane, all four channels: the atmosphere's tap rule (include/oxcull.h,
// atmosphere item 5) for any plane
OXC_DI void sib_tap4(const uint16_t* plane, int w, int h, float u, float v, float out[4]) {
  const float x = fs(fm(u, (float)w), 0.5f), y = fs(fm(v, (float)h), 0.5f);
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = fs(x, x0), wy = fs(y, y0);
  const long long ix = sat_i32(x0), iy = sat_i32(y0);
  const int xa = clamp_index(ix, w), xb = clamp_index(ix + 1, w), ya = clamp_index(iy, h), yb = clamp_index(iy + 1, h);
  const uint2* t = reinterpret_cast<const uint2*>(plane);
  const uint2 q[4] = {__ldg(t + (size_t)ya * w + xa), __ldg(t + (size_t)ya * w + xb), __ldg(t + (size_t)yb * w + xa),
                      __ldg(t + (size_t)yb * w + xb)};
  for (int c = 0; c < 4; c++) {
    const int sh = (c & 1) * 16;
    float a[4];
    for (int k = 0; k < 4; k++) a[k] = half_float((uint16_t)(((c < 2) ? q[k].x : q[k].y) >> sh));
    const float top = fa(a[0], fm(wx, fs(a[1], a[0]))), bot = fa(a[2], fm(wx, fs(a[3], a[2])));
    out[c] = fa(top, fm(wy, fs(bot, top)));
  }
}

// sky_ibl.slang:21-30 and :67-68: the direction of texel (x, y) of `face`; the face matrices by rows, mul(M, v) row by row
OXC_DI Vec3 sky_ibl_dir(int face, int x, int y) {
  const float u = fd(fa((float)x, 0.5f), (float)SKY_IBL_RES), v = fd(fa((float)y, 0.5f), (float)SKY_IBL_RES);
  const float qx = fs(fm(u, 2.0f), 1.0f), qy = fs(fm(v, 2.0f), 1.0f), qz = -1.0f;
  float m[9];
  switch (face) {
    case 0: { const float r[9] = {0, 0, -1, 0, -1, 0, -1, 0, 0}; for (int k = 0; k < 9; k++) m[k] = r[k]; break; }
    case 1: { const float r[9] = {0, 0, 1, 0, -1, 0, 1, 0, 0}; for (int k = 0; k < 9; k++) m[k] = r[k]; break; }
    case 2: { const float r[9] = {1, 0, 0, 0, 0, -1, 0, 1, 0}; for (int k = 0; k < 9; k++) m[k] = r[k]; break; }
    case 3: { const float r[9] = {1, 0, 0, 0, 0, 1, 0, -1, 0}; for (int k = 0; k < 9; k++) m[k] = r[k]; break; }
    case 4: { const float r[9] = {1, 0, 0, 0, -1, 0, 0, 0, -1}; for (int k = 0; k < 9; k++) m[k] = r[k]; break; }
    default: { const float r[9] = {-1, 0, 0, 0, -1, 0, 0, 0, 1}; for (int k = 0; k < 9; k++) m[k] = r[k]; break; }
  }
  return vnormalize(vec3(dot3(m[0], m[1], m[2], qx, qy, qz), dot3(m[3], m[4], m[5], qx, qy, qz), dot3(m[6], m[7], m[8], qx, qy, qz)));
}

// what every sample of a texel shares: its direction and tangent frame (:72-74), its history (:76-77) and the rotation (:79-82)
struct SkyIblTexel {
  Vec3 dir, tangent, bitangent;
  float history[4];
  bool has_history;
  float rotation;
};

// sky_ibl.slang:41-44 interleaved_gradient_noise
OXC_DI float sky_ibl_ign(float px, float py) { return frac(fm(SKY_IBL_IGN_Z, frac(fa(fm(px, SKY_IBL_IGN_X), fm(py, SKY_IBL_IGN_Y))))); }

OXC_DI SkyIblTexel sky_ibl_texel(const SkyIblParams& p, int face, int x, int y) {
  SkyIblTexel t;
  t.dir = sky_ibl_dir(face, x, y);
  const Vec3 up = fabsf(t.dir.y) < SKY_IBL_UP_LIMIT ? vec3(0.0f, 1.0f, 0.0f) : vec3(1.0f, 0.0f, 0.0f);
  t.tangent = vnormalize(vcross(up, t.dir));
  t.bitangent = vcross(t.dir, t.tangent);
  const uint2 h = *reinterpret_cast<const uint2*>(p.cube + ((size_t)(face * SKY_IBL_RES + y) * SKY_IBL_RES + x) * 4);
  t.history[0] = half_float((uint16_t)h.x); t.history[1] = half_float((uint16_t)(h.x >> 16));
  t.history[2] = half_float((uint16_t)h.y); t.history[3] = half_float((uint16_t)(h.y >> 16));
  const float inf = __uint_as_float(0x7F800000u);
  t.has_history = t.history[3] > 0.0f && fabsf(t.history[0]) < inf && fabsf(t.history[1]) < inf && fabsf(t.history[2]) < inf;
  const float f = (float)face;
  const float base = sky_ibl_ign(fa((float)x, fm(f, 37.0f)), fa((float)y, fm(f, 17.0f)));
  t.rotation = t.has_history ? frac(fa(base, fm(p.frame, SKY_IBL_GOLDEN))) : base;
  return t;
}

// sky_ibl.slang:32-39: f32(bits) * 2^-32, exact for every i < 64 (the reversed bits have at most 6 significant bits)
OXC_DI float sky_ibl_radical_inverse(uint32_t bits) {
  bits = (bits << 16u) | (bits >> 16u);
  bits = ((bits & 0x55555555u) << 1u) | ((bits & 0xAAAAAAAAu) >> 1u);
  bits = ((bits & 0x33333333u) << 2u) | ((bits & 0xCCCCCCCCu) >> 2u);
  bits = ((bits & 0x0F0F0F0Fu) << 4u) | ((bits & 0xF0F0F0F0u) >> 4u);
  bits = ((bits & 0x00FF00FFu) << 8u) | ((bits & 0xFF00FF00u) >> 8u);
  return fm((float)bits, SKY_IBL_VDC_SCALE);
}

// sky.slang:39-67 sky_view_params_to_lut_uv with the call's beta and PI - beta (altitude = eye_h)
OXC_DI void sky_ibl_sky_view_uv(const AtmosphereParams& a, bool intersect_planet, float view_zenith_cos, float lx, float ly, float& u,
                                float& v) {
  const float view_zenith_angle = canonical_acos(view_zenith_cos);
  if (!intersect_planet) {
    float coord = fd(view_zenith_angle, a.zenith_horizon);
    coord = fs(1.0f, coord);
    coord = atm_safe_sqrt(coord);
    coord = fs(1.0f, coord);
    v = fm(coord, 0.5f);
  } else {
    float coord = fd(fs(view_zenith_angle, a.zenith_horizon), a.beta);
    coord = atm_safe_sqrt(coord);
    v = fa(fm(coord, 0.5f), 0.5f);
  }
  const float theta = canonical_atan2(-ly, -lx);
  u = fd(fa(theta, PI), ATM_TAU); // 2.0 * PI folds to TAU exactly
  // from_unit_to_sub_uvs (:11-13): (uv + 0.5 / res) * (res / (res + 1))
  const float rw = (float)a.sv_w, rh = (float)a.sv_h;
  u = fm(fa(u, fd(0.5f, rw)), fd(rw, fa(rw, 1.0f)));
  v = fm(fa(v, fd(0.5f, rh)), fd(rh, fa(rh, 1.0f)));
}

// sky.slang:296-322 get_atmosphere_illuminance_along_ray(sun, (0, eye_y, 0), eye_dir), its up vector and normalized sun per call
OXC_DI Vec3 sky_ibl_illuminance(const SkyIblParams& p, Vec3 eye_dir) {
  const Vec3 up = vec3(p.up[0], p.up[1], p.up[2]);
  const float view_zenith_cos = vdot(eye_dir, up);
  const Vec3 side_raw = vcross(up, eye_dir);
  const Vec3 side = vlength(side_raw) > SKY_IBL_SIDE_MIN ? vnormalize(side_raw) : vec3(1.0f, 0.0f, 0.0f);
  const Vec3 forward = vnormalize(vcross(side, up));
  const Vec3 sun = vec3(p.sun[0], p.sun[1], p.sun[2]);
  float lx = vdot(sun, forward), ly = vdot(sun, side);
  // safe_normalize (common/math.slang:90-93): len_sq > 1e-20 ? v * rsqrt(len_sq) : (1, 0), rsqrt(x) = fl(1 / fl(sqrt(x)))
  const float len_sq = fa(fm(lx, lx), fm(ly, ly));
  if (len_sq > SKY_IBL_SAFE_NORMALIZE_MIN) {
    const float rs = fd(1.0f, fsq(len_sq));
    lx = fm(lx, rs); ly = fm(ly, rs);
  } else {
    lx = 1.0f; ly = 0.0f;
  }
  float t;
  const bool intersect_planet = atm_ray_sphere_nearest(vec3(0.0f, p.atm.eye_y, 0.0f), eye_dir, p.atm.planet_radius, t);
  float u, v;
  sky_ibl_sky_view_uv(p.atm, intersect_planet, view_zenith_cos, lx, ly, u, v);
  float s[4];
  sib_tap4(p.sky_view, p.atm.sv_w, p.atm.sv_h, u, v, s);
  return vec3(sib_sanitize(fm(s[0], s[3])), sib_sanitize(fm(s[1], s[3])), sib_sanitize(fm(s[2], s[3])));
}

// sky_ibl.slang:46-52 and :86-97: sample i of a texel, sanitized
OXC_DI Vec3 sky_ibl_sample(const SkyIblParams& p, const SkyIblTexel& t, int i) {
  const float u1 = fd(fa((float)i, 0.5f), (float)SKY_IBL_SAMPLES);
  const float u2 = frac(fa(sky_ibl_radical_inverse((uint32_t)i), t.rotation));
  const float r = fsq(u1);
  const float phi = fm(ATM_TAU, u2);
  float sn, cs;
  canonical_sincos(phi, sn, cs);
  const float lx = fm(r, cs), ly = fm(r, sn), lz = fsq(vmax(0.0f, fs(1.0f, u1)));
  const Vec3 input_dir = vnormalize(vadd(vadd(vscale(t.tangent, lx), vscale(t.bitangent, ly)), vscale(t.dir, lz)));
  const Vec3 s = sky_ibl_illuminance(p, input_dir);
  return vec3(sib_sanitize(s.x), sib_sanitize(s.y), sib_sanitize(s.z));
}

// sky_ibl.slang:99-115 for a texel whose 64 samples sum (in index order, from 0) to `sum`: the sun term, the clamp, the history lerp and
// the store of (rgb, 1)
OXC_DI void sky_ibl_finish(const SkyIblParams& p, const SkyIblTexel& t, int face, int x, int y, Vec3 sum) {
  const AtmosphereParams& a = p.atm;
  float mu, rr;
  atm_transmittance_uv(a.atmos_radius, a.planet_radius, a.eye_y, p.sun_cos_zenith, mu, rr);
  float sun_color[4];
  sib_tap4(a.transmittance, a.t_w, a.t_h, mu, rr, sun_color);
  const float sun_facing = saturate(dot3(t.dir.x, t.dir.y, t.dir.z, p.sun_raw[0], p.sun_raw[1], p.sun_raw[2]));
  const float est[3] = {sum.x, sum.y, sum.z};
  float out[3];
  for (int c = 0; c < 3; c++) {
    const float sun_term = fd(fm(fm(fm(p.sun_ambient_strength, sun_color[c]), p.sun_intensity), sun_facing), PI);
    const float frame_result = vmin(vmax(sib_sanitize(fa(fd(est[c], (float)SKY_IBL_SAMPLES), sun_term)), 0.0f), ATM_HALF_MAX);
    out[c] = t.has_history ? fa(t.history[c], fm(fs(frame_result, t.history[c]), SKY_IBL_ALPHA)) : frame_result;
  }
  atm_store(p.cube, (size_t)(face * SKY_IBL_RES + y) * SKY_IBL_RES + x, out[0], out[1], out[2], 1.0f);
}

// the whole texel with its 64 samples in one serial loop, as the shader writes it
OXC_DI void sky_ibl_texel_serial(const SkyIblParams& p, int face, int x, int y) {
  const SkyIblTexel t = sky_ibl_texel(p, face, x, y);
  Vec3 sum = vec3(0.0f, 0.0f, 0.0f);
  for (int i = 0; i < SKY_IBL_SAMPLES; i++) sum = vadd(sum, sky_ibl_sample(p, t, i));
  sky_ibl_finish(p, t, face, x, y, sum);
}

} // namespace oxc
