// oxc_pbr.cuh — PBR apply of one pixel (passes/pbr_apply_no_atmos.slang:23-127 with the pbr.slang:1-172 functions it calls) as
// pure per-thread functions: the per-light constants the kernel stages once per CTA, and the lit colour of a pixel.
// No warp intrinsics, no shared memory: tests compile this source for the host.
// Specification: include/oxcull.h (comment above oxc_apply_pbr) == oracle/oxc_oracle_pbr.c, operation for operation.
#pragma once
#include "oxc_vsm_resolve.cuh"

namespace oxc {

constexpr uint32_t PBR_FLAG_DIRECTIONAL = 1u << 0, PBR_FLAG_ATMOSPHERE = 1u << 1, PBR_FLAG_CONTACT = 1u << 9, PBR_FLAG_SKY = 1u << 10,
                   PBR_FLAG_TRANSPARENT = 1u << 11; // SceneFlags
constexpr uint32_t PBR_LIGHT_POINT = 1u, PBR_LIGHT_SPOT = 2u;   // LightKind
constexpr float PBR_PI = 3.1415926535897932384626433832795f;     // common/math.slang PI
constexpr float PBR_INV_PI = 1.0f / PBR_PI;                      // Fd_Lambert: fl(1 / fl(pi))

struct PbrV3 { float x, y, z; };
OXC_DI PbrV3 v3(float x, float y, float z) { return PbrV3{x, y, z}; }
OXC_DI float pbr_dot(PbrV3 a, PbrV3 b) { return dot3(a.x, a.y, a.z, b.x, b.y, b.z); }
OXC_DI PbrV3 pbr_normalize(PbrV3 v) { const float l = fsq(pbr_dot(v, v)); return v3(fd(v.x, l), fd(v.y, l), fd(v.z, l)); }
OXC_DI float pbr_sat(float x) { return vmin(vmax(x, 0.0f), 1.0f); }

// a light as the kernel stages it: the record's fields plus the per-light constants of calculate_spot_light_attenuation
struct PbrLight {
  float4 pos_intensity;   // position, intensity
  float4 color_range;     // color, range
  float4 spot_cos_inner;  // normalize(direction), cos(inner_cone_angle)
  float4 cos_outer_kind;  // cos(outer_cone_angle), kind (bits), 0, 0
};

struct PbrParams {
  float4 inv_pv_row[4];   // rows of Camera::inv_projection_view
  float cam_pos[3];
  float sun[3], sun_intensity;
  float base_ambient[3];
  float4 sky_solid;
  float sky_ambient[3];
  uint32_t sky_has_texture;
  uint32_t flags, light_count;
  const float* depth;
  const float4* albedo;
  const float4* normal;   // oct(mapped normal) in .xy, oct(world normal) in .zw
  const float4* emissive;
  const float4* mro;      // metallic, roughness, occlusion
  const float* ao;        // NULL = 1
  const float* shadow;    // NULL = 1
  const float* contact;   // read under PBR_FLAG_CONTACT
  const float4* lights;   // light_count records of four float4 (OxcLight)
  float4* out;
  int width, height;
};

// the kernel's parameters from the C ABI's arguments (oxc_apply_pbr, and the host build of the tests)
__host__ inline PbrParams pbr_make_params(const OxcPbrCamera& cam, const OxcPbrSettings& st, const OxcLight* lights, const OxcPbrInputs& in,
                                          uint32_t w, uint32_t h, float* out) {
  PbrParams p{};
  for (int i = 0; i < 4; i++)
    p.inv_pv_row[i] = make_float4(cam.inv_projection_view[i], cam.inv_projection_view[4 + i], cam.inv_projection_view[8 + i],
                                  cam.inv_projection_view[12 + i]);
  for (int i = 0; i < 3; i++) {
    p.cam_pos[i] = cam.position[i]; p.sun[i] = st.sun_direction[i]; p.base_ambient[i] = st.base_ambient_color[i];
    p.sky_ambient[i] = st.sky_ambient_color[i];
  }
  p.sun_intensity = st.sun_intensity;
  p.sky_solid = make_float4(st.sky_solid_color[0], st.sky_solid_color[1], st.sky_solid_color[2], st.sky_solid_color[3]);
  p.sky_has_texture = st.sky_has_texture;
  p.flags = st.scene_flags; p.light_count = st.light_count;
  p.depth = in.depth; p.albedo = reinterpret_cast<const float4*>(in.albedo); p.normal = reinterpret_cast<const float4*>(in.normal);
  p.emissive = reinterpret_cast<const float4*>(in.emissive); p.mro = reinterpret_cast<const float4*>(in.metallic_roughness_occlusion);
  p.ao = in.ambient_occlusion; p.shadow = in.shadow;
  p.contact = (st.scene_flags & OXC_SCENE_HAS_CONTACT_SHADOWS) ? in.contact_shadow : nullptr;
  p.lights = reinterpret_cast<const float4*>(lights); p.out = reinterpret_cast<float4*>(out);
  p.width = (int)w; p.height = (int)h;
  return p;
}

// the per-light constants (pbr.slang:132-138): the same function of the same record wherever it is evaluated
OXC_DI PbrLight pbr_stage_light(float4 r0, float4 r1, float4 r2, float4 r3) {
  PbrLight l;
  l.pos_intensity = r0;
  l.color_range = r1;
  const PbrV3 sd = pbr_normalize(v3(r2.x, r2.y, r2.z));
  l.spot_cos_inner = make_float4(sd.x, sd.y, sd.z, canonical_cos(r2.w));
  l.cos_outer_kind = make_float4(canonical_cos(r3.x), r3.y, 0.0f, 0.0f);
  return l;
}

// common/encoding.slang:7-15
OXC_DI PbrV3 pbr_oct_to_vec3(float ex, float ey) {
  PbrV3 v = v3(ex, ey, fs(fs(1.0f, fabsf(ex)), fabsf(ey)));
  const float sx = v.x >= 0.0f ? 1.0f : -1.0f, sy = v.y >= 0.0f ? 1.0f : -1.0f;
  if (v.z < 0.0f) { v.x = fm(fs(1.0f, fabsf(ey)), sx); v.y = fm(fs(1.0f, fabsf(ex)), sy); }
  return pbr_normalize(v);
}

// pbr.slang:35-44, both components
OXC_DI void pbr_ggx_directional_albedo(float x, float y, float& a, float& b) {
  const float x2 = fm(x, x), y2 = fm(y, y);
  const float c[9][4] = {{0.1003f, 0.9345f, 1.0f, 1.0f},     {-0.6303f, -2.323f, -1.765f, 0.2281f}, {9.748f, 2.229f, 8.263f, 15.94f},
                         {-2.038f, -3.748f, 11.53f, -55.83f}, {29.34f, 1.424f, 28.96f, 13.08f},     {-8.245f, -0.7684f, -7.507f, 41.26f},
                         {-26.44f, 1.436f, -36.11f, 54.9f},   {19.99f, 0.2913f, 15.86f, 300.2f},    {-5.448f, 0.6286f, 33.37f, -285.1f}};
  float r[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    float s = fa(c[0][i], fm(c[1][i], x));
    s = fa(s, fm(c[2][i], y));
    s = fa(s, fm(fm(c[3][i], x), y));
    s = fa(s, fm(c[4][i], x2));
    s = fa(s, fm(c[5][i], y2));
    s = fa(s, fm(fm(c[6][i], x2), y));
    s = fa(s, fm(fm(c[7][i], x), y2));
    s = fa(s, fm(fm(c[8][i], x2), y2));
    r[i] = s;
  }
  a = pbr_sat(fd(r[0], r[2]));
  b = pbr_sat(fd(r[1], r[3]));
}

// pbr.slang:89-100
OXC_DI float pbr_attenuate_point(float dist, float cutoff) {
  if (cutoff <= 0.0f) return fd(1.0f, fa(fm(dist, dist), 0.1f));
  float win = fd(dist, cutoff);
  win = fm(fm(fm(win, win), win), win);
  win = vmax(0.0f, fs(1.0f, win));
  win = fm(win, win);
  return fd(win, fa(fm(dist, dist), 0.1f));
}

// what the BRDF (pbr.slang:61-87) shares between the lights of one pixel: F0, alpha, alpha^2, NoV and the energy compensation
struct PbrSurface {
  PbrV3 N, V, albedo, F0, energy;
  float metallic, alpha2, NoV;
};

// pbr.slang:61-87 BRDF(V, N, L, ...): diffuse and specular
OXC_DI void pbr_brdf(const PbrSurface& s, PbrV3 L, PbrV3& diffuse, PbrV3& specular) {
  const PbrV3 VL = v3(fa(s.V.x, L.x), fa(s.V.y, L.y), fa(s.V.z, L.z));
  const PbrV3 H = pbr_dot(VL, VL) > 1e-8f ? pbr_normalize(VL) : s.N;
  const float NoL = pbr_sat(pbr_dot(s.N, L));
  const float NoH = pbr_sat(pbr_dot(s.N, H));
  const float LoH = pbr_sat(pbr_dot(L, H));
  // D_GGX :11-14
  const float f = fa(fm(fs(fm(NoH, s.alpha2), NoH), NoH), 1.0f);
  const float D = fd(s.alpha2, fa(fm(fm(PBR_PI, f), f), 1e-7f));
  // V_SmithGGXCorrelated :16-20
  const float one_a2 = fs(1.0f, s.alpha2);
  const float GGXV = fm(NoL, fsq(fa(fm(fm(s.NoV, s.NoV), one_a2), s.alpha2)));
  const float GGXL = fm(s.NoV, fsq(fa(fm(fm(NoL, NoL), one_a2), s.alpha2)));
  const float Vis = pbr_sat(fd(0.5f, fa(fa(GGXV, GGXL), 1e-7f)));
  // F_Schlick :22-24
  const float p5 = canonical_pow5(pbr_sat(fs(1.0f, LoH)));
  const PbrV3 F = v3(fa(s.F0.x, fm(fs(1.0f, s.F0.x), p5)), fa(s.F0.y, fm(fs(1.0f, s.F0.y), p5)), fa(s.F0.z, fm(fs(1.0f, s.F0.z), p5)));
  const float DV = fm(D, Vis);
  specular = v3(fm(fm(DV, F.x), s.energy.x), fm(fm(DV, F.y), s.energy.y), fm(fm(DV, F.z), s.energy.z));
  const float one_m = fs(1.0f, s.metallic);
  diffuse = v3(fm(fm(fm(one_m, fs(1.0f, F.x)), s.albedo.x), PBR_INV_PI), fm(fm(fm(one_m, fs(1.0f, F.y)), s.albedo.y), PBR_INV_PI),
               fm(fm(fm(one_m, fs(1.0f, F.z)), s.albedo.z), PBR_INV_PI));
}

// point_light_contribution (pbr.slang:102-130) and calculate_spot_light_contribution (:140-172), added to `total`; other kinds add
// nothing
OXC_DI void pbr_add_light(const PbrSurface& s, PbrV3 world, const PbrLight& l, PbrV3& total) {
  const uint32_t kind = __float_as_uint(l.cos_outer_kind.y);
  if (kind != PBR_LIGHT_POINT && kind != PBR_LIGHT_SPOT) return;
  const PbrV3 lv = v3(fs(l.pos_intensity.x, world.x), fs(l.pos_intensity.y, world.y), fs(l.pos_intensity.z, world.z));
  const float dist = fsq(pbr_dot(lv, lv));
  const PbrV3 L = v3(fd(lv.x, dist), fd(lv.y, dist), fd(lv.z, dist));
  float att = pbr_attenuate_point(dist, l.color_range.w);
  if (kind == PBR_LIGHT_SPOT) {
    // calculate_spot_light_attenuation :132-138, smoothstep(cos_outer, cos_inner, dot(-L, normalize(direction)))
    const float cos_angle = dot3(-L.x, -L.y, -L.z, l.spot_cos_inner.x, l.spot_cos_inner.y, l.spot_cos_inner.z);
    const float e0 = l.cos_outer_kind.x, e1 = l.spot_cos_inner.w;
    const float t = pbr_sat(fd(fs(cos_angle, e0), fs(e1, e0)));
    att = fm(att, fm(fm(t, t), fs(3.0f, fm(2.0f, t))));
  }
  const float intensity = l.pos_intensity.w;
  if (att <= 0.0f || intensity <= 0.0f) return;
  const float NdotL = pbr_sat(pbr_dot(s.N, L));
  if (NdotL <= 0.0f) return;
  PbrV3 d, sp;
  pbr_brdf(s, L, d, sp);
  total.x = fa(total.x, fm(fm(fa(d.x, sp.x), fm(fm(l.color_range.x, att), intensity)), NdotL));
  total.y = fa(total.y, fm(fm(fa(d.y, sp.y), fm(fm(l.color_range.y, att), intensity)), NdotL));
  total.z = fa(total.z, fm(fm(fa(d.z, sp.z), fm(fm(l.color_range.z, att), intensity)), NdotL));
}

// the stored value: every NaN is written as 0x7FFFFFFF
OXC_DI float pbr_store(float v) { return v != v ? __uint_as_float(0x7FFFFFFFu) : v; }

// fs_main (pbr_apply_no_atmos.slang:23-127) of pixel (x, y) with the staged lights
OXC_DI float4 pbr_pixel(const PbrParams& p, const PbrLight* lights, int x, int y) {
  const size_t pix = (size_t)y * p.width + x;
  const float depth = p.depth[pix];
  if ((p.flags & PBR_FLAG_TRANSPARENT) && depth == 0.0f) return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  const float u = fd(fa((float)x, 0.5f), (float)p.width), v = fd(fa((float)y, 0.5f), (float)p.height);
  const float4 alb = __ldg(p.albedo + pix);
  const float4 nrm = __ldg(p.normal + pix);
  const PbrV3 mapped = pbr_oct_to_vec3(round_to_half(nrm.x), round_to_half(nrm.y));
  const PbrV3 smooth = pbr_oct_to_vec3(round_to_half(nrm.z), round_to_half(nrm.w));
  const float4 em = __ldg(p.emissive + pix);
  const float4 mro = __ldg(p.mro + pix);
  const float metallic = vmin(vmax(mro.x, 0.0f), 1.0f);
  const float roughness = vmin(vmax(mro.y, 0.045f), 1.0f);
  const float ssao = p.ao ? round_to_half(__ldg(p.ao + pix)) : 1.0f;
  const float occlusion = fm(mro.z, ssao);
  // world position :56-58
  const float nx = fs(fm(u, 2.0f), 1.0f), ny = fs(fm(v, 2.0f), 1.0f);
  float h[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const float4 r = p.inv_pv_row[i];
    h[i] = fa(fa(fa(fm(r.x, nx), fm(r.y, ny)), fm(r.z, depth)), fm(r.w, 1.0f));
  }
  const PbrV3 world = v3(fd(h[0], h[3]), fd(h[1], h[3]), fd(h[2], h[3]));
  // :63-67
  PbrSurface s;
  s.V = pbr_normalize(v3(fs(p.cam_pos[0], world.x), fs(p.cam_pos[1], world.y), fs(p.cam_pos[2], world.z)));
  s.N = pbr_normalize(mapped);
  const PbrV3 I = v3(-s.V.x, -s.V.y, -s.V.z);
  const float dIN = pbr_dot(I, s.N);
  const PbrV3 R = v3(fs(I.x, fm(fm(2.0f, s.N.x), dIN)), fs(I.y, fm(fm(2.0f, s.N.y), dIN)), fs(I.z, fm(fm(2.0f, s.N.z), dIN)));
  s.NoV = fa(fabsf(pbr_dot(s.N, s.V)), 1e-5f);
  const PbrV3 Ls = v3(p.sun[0], p.sun[1], p.sun[2]);
  const float NoL = vmax(pbr_dot(s.N, Ls), 0.0f);
  if ((p.flags & PBR_FLAG_SKY) && depth == 0.0f)
    return p.sky_has_texture ? make_float4(1.0f, 1.0f, 1.0f, 1.0f)
                             : make_float4(pbr_store(p.sky_solid.x), pbr_store(p.sky_solid.y), pbr_store(p.sky_solid.z), pbr_store(p.sky_solid.w));
  const bool has_dir = (p.flags & PBR_FLAG_DIRECTIONAL) != 0;
  const float dshadow = has_dir && p.shadow ? __ldg(p.shadow + pix) : 1.0f;
  const float cshadow = (p.flags & PBR_FLAG_CONTACT) ? __ldg(p.contact + pix) : 1.0f;
  const float visibility = fm(dshadow, cshadow);
  const float direct = has_dir ? p.sun_intensity : 0.0f;
  const bool has_sky = (p.flags & PBR_FLAG_SKY) != 0;
  const PbrV3 env = has_sky ? v3(p.sky_ambient[0], p.sky_ambient[1], p.sky_ambient[2]) : v3(p.base_ambient[0], p.base_ambient[1], p.base_ambient[2]);
  // :86-100
  s.albedo = v3(alb.x, alb.y, alb.z);
  s.metallic = metallic;
  s.F0 = v3(fa(0.04f, fm(fs(alb.x, 0.04f), metallic)), fa(0.04f, fm(fs(alb.y, 0.04f), metallic)), fa(0.04f, fm(fs(alb.z, 0.04f), metallic)));
  const float alpha = vmax(fm(roughness, roughness), 0.0025f);
  s.alpha2 = fm(alpha, alpha);
  float ABx, ABy;
  pbr_ggx_directional_albedo(s.NoV, alpha, ABx, ABy);
  const PbrV3 kS = v3(fa(fm(s.F0.x, ABx), ABy), fa(fm(s.F0.y, ABx), ABy), fa(fm(s.F0.z, ABx), ABy));
  const float one_m = fs(1.0f, metallic);
  const PbrV3 kD = v3(fm(one_m, fs(1.0f, kS.x)), fm(one_m, fs(1.0f, kS.y)), fm(one_m, fs(1.0f, kS.z)));
  // specular_occlusion_horizon :52-54
  const float spec_occ = pbr_sat(fa(fs(canonical_pow(fa(s.NoV, occlusion), canonical_pow(2.0f, fs(fm(-16.0f, roughness), 1.0f))), 1.0f), occlusion));
  const PbrV3 indirect = v3(fa(fm(fm(fm(fm(kD.x, env.x), alb.x), PBR_INV_PI), occlusion), fm(fm(kS.x, env.x), spec_occ)),
                            fa(fm(fm(fm(fm(kD.y, env.y), alb.y), PBR_INV_PI), occlusion), fm(fm(kS.y, env.y), spec_occ)),
                            fa(fm(fm(fm(fm(kD.z, env.z), alb.z), PBR_INV_PI), occlusion), fm(fm(kS.z, env.z), spec_occ)));
  // GGX_energy_compensation :46-50, which depends on no light
  const float Ess = pbr_sat(fa(ABx, ABy));
  const float one_ess = fs(1.0f, Ess), ess_den = vmax(Ess, 1e-4f);
  s.energy = v3(fa(1.0f, fd(fm(s.F0.x, one_ess), ess_den)), fa(1.0f, fd(fm(s.F0.y, one_ess), ess_den)), fa(1.0f, fd(fm(s.F0.z, one_ess), ess_den)));
  // :102-113
  PbrV3 total = v3(0.0f, 0.0f, 0.0f);
  for (uint32_t i = 0; i < p.light_count; i++) pbr_add_light(s, world, lights[i], total);
  // :115-123
  float horizon = pbr_sat(fa(1.0f, fm(1.3f, pbr_dot(R, smooth))));
  horizon = fm(horizon, horizon);
  PbrV3 surf = v3(0.0f, 0.0f, 0.0f);
  if (NoL > 0.0f) {
    PbrV3 d, sp;
    pbr_brdf(s, Ls, d, sp);
    surf = v3(fm(fm(fm(fa(d.x, fm(sp.x, horizon)), direct), NoL), visibility), fm(fm(fm(fa(d.y, fm(sp.y, horizon)), direct), NoL), visibility),
              fm(fm(fm(fa(d.z, fm(sp.z, horizon)), direct), NoL), visibility));
  }
  // :125-126
  return make_float4(pbr_store(fa(fa(fa(surf.x, total.x), indirect.x), em.x)), pbr_store(fa(fa(fa(surf.y, total.y), indirect.y), em.y)),
                     pbr_store(fa(fa(fa(surf.z, total.z), indirect.z), em.z)), 1.0f);
}

} // namespace oxc
