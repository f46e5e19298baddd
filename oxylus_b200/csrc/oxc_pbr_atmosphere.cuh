// oxc_pbr_atmosphere.cuh — PBR apply of one pixel under the atmosphere (passes/pbr_apply.slang:26-184 with the sky.slang functions it
// calls: get_direct_sun_lighting, sky_view_params_to_lut_uv, sample_aerial_perspective) as pure per-thread functions.  The G-buffer
// reads, the BRDF, the light loop and the sum are oxc_pbr.cuh's (pbr_prologue, pbr_shade); the LUT taps are oxc_sky_ibl.cuh's.
// No warp intrinsics, no shared memory: tests compile this source for the host.
// Specification: include/oxcull.h (comment above oxc_apply_pbr_atmosphere) == oracle/oxc_oracle_pbr_atmosphere.c, operation for operation.
#pragma once
#include "oxc_pbr.cuh"
#include "oxc_sky_ibl.cuh"

namespace oxc {

// binary32 roundings of the shader's literals and folds (bits pinned by tests/test_oracle_pbr_atmosphere.py)
constexpr float PBRA_SUN_RADIANS = 0x1.1df46ap-6f;    // 0x3C8EFA35 = fl(fl(1 * PI) / 180), draw_sun's radius * PI / 180.0
constexpr float PBRA_HALF_SLICE = 0x1.6a09e6p-1f;     // 0x3F3504F3 = sqrt(0.5), sky.slang:276
constexpr float PBRA_NEAR_FADE = 0x1.f3fffep+9f;      // 0x4479FFFF = fl(1 / fl(0.001)), sky.slang:281, folded in binary32
constexpr float PBRA_HD_LO = -0.1f, PBRA_HD_HI = 0.3f; // smoothstep(-0.1, 0.3, sun_cos_theta), pbr_apply.slang:103

struct PbrAtmParams {
  PbrParams pbr;             // pbr_make_params of the call: base_ambient and the sky_* fields are not read
  AtmosphereParams atm;      // the record's radii and sizes, the transmittance LUT, eye_y of the camera; beta and PI - beta for
                             // altitude eye_y (sky.slang:46-48 with h = eye_pos.y)
  const uint16_t* sky_view;  // sv_w x sv_h binary16 RGBA
  const uint16_t* aerial;    // ap_w x ap_h x ap_d binary16 RGBA
  const uint16_t* cube;      // 6 x 32 x 32 binary16 RGBA
  float min_altitude;        // planet_radius + PLANET_RADIUS_OFFSET (scene.slang:230)
  float sun_cos_theta;       // dot(L, (0, 1, 0)), :102
  float horizon_darkening;   // smoothstep(-0.1, 0.3, sun_cos_theta), :103
  float min_cos;             // canonical_cos(0x3C8EFA35), draw_sun :27
  float ap_per_slice_depth;  // f32(size.x) / f32(size.z), sky.slang:266
  float ap_start, ap_exposure;
};

// the kernel's parameters from the C ABI's arguments (oxc_apply_pbr_atmosphere, and the host build of the tests)
__host__ inline PbrAtmParams pbr_atmosphere_make_params(const OxcPbrCamera& cam, const OxcPbrSettings& st, const OxcAtmosphere& a,
                                                        const OxcLight* lights, const OxcPbrInputs& in, const OxcPbrSky& sky, uint32_t w,
                                                        uint32_t h, float* out) {
  PbrAtmParams p{};
  p.pbr = pbr_make_params(cam, st, lights, in, w, h, out);
  p.atm = atmosphere_make_params(a, &cam, st.sun_direction, st.sun_intensity, sky.transmittance, nullptr, nullptr, nullptr, 0);
  // sky_view_params_to_lut_uv with altitude = eye_pos.y as pbr_apply.slang:110 passes it (not length(eye_pos))
  const float alt = p.atm.eye_y;
  const float horizon = sqrtf(vmax(0.0f, alt * alt - a.planet_radius * a.planet_radius));
  p.atm.beta = canonical_acos(horizon / alt);
  p.atm.zenith_horizon = PI - p.atm.beta;
  p.sky_view = sky.sky_view; p.aerial = sky.aerial_perspective; p.cube = sky.sky_cube;
  p.min_altitude = a.planet_radius + ATM_PLANET_RADIUS_OFFSET;
  const float* L = st.sun_direction;
  p.sun_cos_theta = (L[0] * 0.0f + L[1] * 1.0f) + L[2] * 0.0f;
  const float t = saturate((p.sun_cos_theta - PBRA_HD_LO) / (PBRA_HD_HI - PBRA_HD_LO));
  p.horizon_darkening = (t * t) * (3.0f - 2.0f * t);
  p.min_cos = canonical_cos(PBRA_SUN_RADIANS);
  p.ap_per_slice_depth = (float)a.aerial_perspective_lut_size[0] / (float)a.aerial_perspective_lut_size[2];
  p.ap_start = a.aerial_perspective_start_km;
  p.ap_exposure = a.aerial_perspective_exposure;
  return p;
}

// draw_sun(world_dir, sun_dir, 1.0) (pbr_apply.slang:26-38), one channel (the shader's three are equal)
OXC_DI float pbra_draw_sun(float min_cos, float cos_theta) {
  if (cos_theta >= min_cos) return 1.0f;
  const float offset = fs(min_cos, cos_theta);
  const float gaussian_bloom = fm(canonical_exp(fm(-offset, 50000.0f)), 0.5f);
  const float inv_bloom = fm(fd(1.0f, fa(0.02f, fm(offset, 300.0f))), 0.01f);
  return fa(gaussian_bloom, inv_bloom);
}

// one binary16 RGBA texel of a plane, read exactly
OXC_DI void pbra_texel(const uint16_t* plane, size_t texel, float o[4]) {
  const uint2 q = __ldg(reinterpret_cast<const uint2*>(plane) + texel);
  o[0] = half_float((uint16_t)q.x); o[1] = half_float((uint16_t)(q.x >> 16));
  o[2] = half_float((uint16_t)q.y); o[3] = half_float((uint16_t)(q.y >> 16));
}

// SampleLevel(linear_clamp, (u, v, w), 0) of the aerial-perspective LUT: the atmosphere's bilinear rule (item 5) in slices z0 and z0 + 1
// (z = w * D - 0.5, z0 = floor(z), wz = z - z0, the same NaN-safe clamped indices), then s0 + wz * (s1 - s0), all four channels
OXC_DI void pbra_tap3(const PbrAtmParams& p, float u, float v, float w, float out[4]) {
  const int W = p.atm.ap_w, H = p.atm.ap_h, D = p.atm.ap_d;
  const float z = fs(fm(w, (float)D), 0.5f);
  const float z0 = floorf(z);
  const float wz = fs(z, z0);
  const long long iz = sat_i32(z0);
  const int za = clamp_index(iz, D), zb = clamp_index(iz + 1, D);
  float s0[4], s1[4];
  sib_tap4(p.aerial + (size_t)za * H * W * 4, W, H, u, v, s0);
  sib_tap4(p.aerial + (size_t)zb * H * W * 4, W, H, u, v, s1);
  for (int c = 0; c < 4; c++) out[c] = fa(s0[c], fm(wz, fs(s1[c], s0[c])));
}

// sample_aerial_perspective (sky.slang:258-293) at tex_coord (u, v) and camera_relative_pos d
OXC_DI void pbra_aerial(const PbrAtmParams& p, float u, float v, Vec3 d, float out[4]) {
  const float dz = (float)p.atm.ap_d;
  const float relative_depth = vmax(0.0f, fs(fsq(vdot(d, d)), p.ap_start));
  const float linear_slice = fm(relative_depth, fd(1.0f, p.ap_per_slice_depth));
  const float linear_w = fm(linear_slice, fd(1.0f, dz));
  const float non_linear_w = fsq(linear_w);
  const float non_linear_slice = fm(non_linear_w, dz);
  float weight = 1.0f;
  if (non_linear_slice < PBRA_HALF_SLICE) weight = saturate(fm(fm(non_linear_slice, non_linear_slice), 2.0f));
  weight = fm(weight, saturate(fm(relative_depth, PBRA_NEAR_FADE)));
  pbra_tap3(p, u, v, non_linear_w, out);
  for (int c = 0; c < 3; c++) out[c] = fm(out[c], weight);
  out[3] = fs(1.0f, fm(weight, fs(1.0f, out[3])));
  for (int c = 0; c < 3; c++) out[c] = fm(out[c], p.ap_exposure);
}

// the face of direction r by the major axis (X when |x| >= |y| and |x| >= |z|, else Y when |y| >= |z|, else Z; the positive face when
// the major component is >= 0) and its (sc, tc, ma) by the Vulkan face table
OXC_DI int pbra_cube_face(float x, float y, float z, float& sc, float& tc, float& ma) {
  const float ax = fabsf(x), ay = fabsf(y), az = fabsf(z);
  if (ax >= ay && ax >= az) {
    ma = x; tc = -y;
    if (x >= 0.0f) { sc = -z; return 0; }
    sc = z; return 1;
  }
  if (ay >= az) {
    ma = y; sc = x;
    if (y >= 0.0f) { tc = z; return 2; }
    tc = -z; return 3;
  }
  ma = z; tc = -y;
  if (z >= 0.0f) { sc = x; return 4; }
  sc = -x; return 5;
}

// texel (i, j) of face f with i, j in -1..32: in the face it is the texel; one step off an edge it is the adjacent face's texel that
// shares that edge (the cube's geometry in half-texel units: the off-face coordinate, +-33, becomes that face's plane, +-32, and the old
// plane, +-32, the edge texel's centre, +-31); off both edges (a corner) it is ((inside + across i) + across j) / 3
OXC_DI size_t pbra_cube_remap(int f, int i, int j) {
  int a = 2 * i - 31, b = 2 * j - 31, m = 32;
  if (a < -32 || a > 32) { a = a < 0 ? -32 : 32; m = 31; }  // the off-face axis becomes the new plane, the old plane the edge centre
  if (b < -32 || b > 32) { b = b < 0 ? -32 : 32; m = 31; }
  // the point (sc, tc, ma) = (a, b, m) of face f in cube coordinates (the face table solved for x, y, z)
  int x, y, z;
  switch (f) {
    case 0: x = m; y = -b; z = -a; break;
    case 1: x = -m; y = -b; z = a; break;
    case 2: x = a; y = m; z = b; break;
    case 3: x = a; y = -m; z = -b; break;
    case 4: x = a; y = -b; z = m; break;
    default: x = -a; y = -b; z = -m; break;
  }
  // back to (face, sc, tc): the major axis is the unique component of magnitude 32
  int nf, sc, tc;
  if (x == 32 || x == -32) { nf = x > 0 ? 0 : 1; sc = x > 0 ? -z : z; tc = -y; }
  else if (y == 32 || y == -32) { nf = y > 0 ? 2 : 3; sc = x; tc = y > 0 ? z : -z; }
  else { nf = z > 0 ? 4 : 5; sc = z > 0 ? x : -x; tc = -y; }
  return ((size_t)nf * SKY_IBL_RES + (size_t)((tc + 31) / 2)) * SKY_IBL_RES + (size_t)((sc + 31) / 2);
}

OXC_DI void pbra_cube_fetch(const uint16_t* cube, int f, int i, int j, float o[4]) {
  const bool oi = i < 0 || i >= SKY_IBL_RES, oj = j < 0 || j >= SKY_IBL_RES;
  if (!oi && !oj) { pbra_texel(cube, ((size_t)f * SKY_IBL_RES + j) * SKY_IBL_RES + i, o); return; }
  if (!(oi && oj)) { pbra_texel(cube, pbra_cube_remap(f, i, j), o); return; }
  const int ci = i < 0 ? 0 : SKY_IBL_RES - 1, cj = j < 0 ? 0 : SKY_IBL_RES - 1;
  float t0[4], t1[4], t2[4];
  pbra_texel(cube, ((size_t)f * SKY_IBL_RES + cj) * SKY_IBL_RES + ci, t0);
  pbra_texel(cube, pbra_cube_remap(f, i, cj), t1);
  pbra_texel(cube, pbra_cube_remap(f, ci, j), t2);
  for (int c = 0; c < 4; c++) o[c] = fd(fa(fa(t0[c], t1[c]), t2[c]), 3.0f);
}

// TextureCube.SampleLevel(linear_clamp, r, 0) of the 32 x 32 cube: face and (sc, tc, ma) by pbra_cube_face, s = 0.5 * (sc / |ma|) + 0.5
// (t likewise), x = s * 32 - 0.5, x0 = floor(x), wx = x - x0 (y likewise), NaN-safe indices clamped to -1..32, the 2 x 2 footprint
// through pbra_cube_fetch, the atmosphere's bilinear order (top = a00 + wx * (a10 - a00), bottom likewise, top + wy * (bottom - top))
OXC_DI void pbra_cube_tap(const uint16_t* cube, Vec3 r, float out[4]) {
  float sc, tc, ma;
  const int f = pbra_cube_face(r.x, r.y, r.z, sc, tc, ma);
  const float s = fa(fm(0.5f, fd(sc, fabsf(ma))), 0.5f), t = fa(fm(0.5f, fd(tc, fabsf(ma))), 0.5f);
  const float x = fs(fm(s, (float)SKY_IBL_RES), 0.5f), y = fs(fm(t, (float)SKY_IBL_RES), 0.5f);
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = fs(x, x0), wy = fs(y, y0);
  const long long ix = sat_i32(x0), iy = sat_i32(y0);
  const int i0 = clamp_index(ix + 1, SKY_IBL_RES + 2) - 1, j0 = clamp_index(iy + 1, SKY_IBL_RES + 2) - 1;
  const int i1 = clamp_index(ix + 2, SKY_IBL_RES + 2) - 1, j1 = clamp_index(iy + 2, SKY_IBL_RES + 2) - 1;
  float a00[4], a10[4], a01[4], a11[4];
  pbra_cube_fetch(cube, f, i0, j0, a00);
  pbra_cube_fetch(cube, f, i1, j0, a10);
  pbra_cube_fetch(cube, f, i0, j1, a01);
  pbra_cube_fetch(cube, f, i1, j1, a11);
  for (int c = 0; c < 4; c++) {
    const float top = fa(a00[c], fm(wx, fs(a10[c], a00[c]))), bot = fa(a01[c], fm(wx, fs(a11[c], a01[c])));
    out[c] = fa(top, fm(wy, fs(bot, top)));
  }
}

// fs_main (pbr_apply.slang:40-184) of pixel (x, y) with the staged lights
OXC_DI float4 pbr_atmosphere_pixel(const PbrAtmParams& p, const PbrLight* lights, int x, int y) {
  const PbrParams& b = p.pbr;
  const size_t pix = (size_t)y * b.width + x;
  const float depth = b.depth[pix];
  if ((b.flags & PBR_FLAG_TRANSPARENT) && depth == 0.0f) return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  PbrPixel q = pbr_prologue(b, pix, depth, x, y);
  const float visibility = pbr_visibility(b, pix, (b.flags & PBR_FLAG_DIRECTIONAL) != 0);
  // :99-106: the sun's transmittance at the pixel's altitude, get_eye_pos(world_position).y
  const float world_eye_y = vmax(fa(fm(q.world.y, ATM_CAMERA_SCALE_UNIT), p.min_altitude), p.min_altitude);
  float mu, rr, T[4];
  atm_transmittance_uv(p.atm.atmos_radius, p.atm.planet_radius, world_eye_y, p.sun_cos_theta, mu, rr);
  sib_tap4(p.atm.transmittance, p.atm.t_w, p.atm.t_h, mu, rr, T);
  const Vec3 direct = vec3(fm(fm(T[0], b.sun_intensity), p.horizon_darkening), fm(fm(T[1], b.sun_intensity), p.horizon_darkening),
                           fm(fm(T[2], b.sun_intensity), p.horizon_darkening));
  if (depth == 0.0f) {
    // :108-124
    const Vec3 up = vec3(0.0f, 1.0f, 0.0f), mv = vec3(-q.s.V.x, -q.s.V.y, -q.s.V.z), L = q.Ls;
    const Vec3 right = vnormalize(vcross(up, mv));
    const Vec3 forward = vnormalize(vcross(right, up));
    float lx = vdot(L, forward), ly = vdot(L, right);
    const float ll = fsq(fa(fm(lx, lx), fm(ly, ly)));
    lx = fd(lx, ll); ly = fd(ly, ll);
    const float view_zenith_cos = vdot(mv, up);
    float t;
    const bool hit = atm_ray_sphere_nearest(vec3(0.0f, p.atm.eye_y, 0.0f), mv, p.atm.planet_radius, t);
    float u, v, s[4];
    sky_ibl_sky_view_uv(p.atm, hit, view_zenith_cos, lx, ly, u, v);
    sib_tap4(p.sky_view, p.atm.sv_w, p.atm.sv_h, u, v, s);
    if (!hit) {
      const float sun = fm(pbra_draw_sun(p.min_cos, vdot(mv, L)), b.sun_intensity);
      for (int c = 0; c < 3; c++) s[c] = fa(s[c], fm(sun, T[c]));
    }
    return make_float4(nan_canonical(fm(s[0], s[3])), nan_canonical(fm(s[1], s[3])), nan_canonical(fm(s[2], s[3])), 1.0f);
  }
  // :126-141
  float ap[4];
  pbra_aerial(p, q.u, q.v,
              vec3(fm(fs(q.world.x, b.cam_pos[0]), ATM_CAMERA_SCALE_UNIT), fm(fs(q.world.y, b.cam_pos[1]), ATM_CAMERA_SCALE_UNIT),
                   fm(fs(q.world.z, b.cam_pos[2]), ATM_CAMERA_SCALE_UNIT)),
              ap);
  const Vec3 aerial = vec3(fm(ap[0], ap[3]), fm(ap[1], ap[3]), fm(ap[2], ap[3]));
  const float k = fs(1.0f, q.roughness);
  const Vec3 N = q.s.N;
  const Vec3 rd = vnormalize(vec3(fa(N.x, fm(fs(q.R.x, N.x), k)), fa(N.y, fm(fs(q.R.y, N.y), k)), fa(N.z, fm(fs(q.R.z, N.z), k))));
  float ss[4], ds[4];
  pbra_cube_tap(p.cube, rd, ss);
  pbra_cube_tap(p.cube, N, ds);
  const float hd = p.horizon_darkening;
  const Vec3 specular_sky = vec3(fm(fm(ss[0], ss[3]), hd), fm(fm(ss[1], ss[3]), hd), fm(fm(ss[2], ss[3]), hd));
  const Vec3 diffuse_sky = vec3(fm(fm(ds[0], ds[3]), hd), fm(fm(ds[1], ds[3]), hd), fm(fm(ds[2], ds[3]), hd));
  return pbr_shade(b, lights, q, diffuse_sky, specular_sky, direct, visibility, &aerial);
}

} // namespace oxc
