// oxc_pbr.cuh — PBR apply of one pixel (passes/pbr_apply_no_atmos.slang:23-127 with the pbr.slang:1-172 functions it calls) as
// pure per-thread functions: the per-light constants the kernel stages once per CTA, and the lit colour of a pixel.
// No warp intrinsics, no shared memory: tests compile this source for the host.
// Specification: include/oxcull.h (comment above oxc_apply_pbr) == oracle/oxc_oracle_pbr.c, operation for operation.
#pragma once
#include "oxc_shader_math.cuh"

namespace oxc {

constexpr uint32_t PBR_FLAG_DIRECTIONAL = 1u << 0, PBR_FLAG_ATMOSPHERE = 1u << 1, PBR_FLAG_CONTACT = 1u << 9, PBR_FLAG_SKY = 1u << 10,
                   PBR_FLAG_TRANSPARENT = 1u << 11; // SceneFlags
constexpr uint32_t PBR_LIGHT_POINT = 1u, PBR_LIGHT_SPOT = 2u;   // LightKind
constexpr float PBR_INV_PI = 1.0f / PI;                          // Fd_Lambert: fl(1 / fl(pi))

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
  const Vec3 sd = vnormalize(vec3(r2.x, r2.y, r2.z));
  l.spot_cos_inner = make_float4(sd.x, sd.y, sd.z, canonical_cos(r2.w));
  l.cos_outer_kind = make_float4(canonical_cos(r3.x), r3.y, 0.0f, 0.0f);
  return l;
}

// common/encoding.slang:7-15
OXC_DI Vec3 pbr_oct_to_vec3(float ex, float ey) {
  Vec3 v = vec3(ex, ey, fs(fs(1.0f, fabsf(ex)), fabsf(ey)));
  const float sx = v.x >= 0.0f ? 1.0f : -1.0f, sy = v.y >= 0.0f ? 1.0f : -1.0f;
  if (v.z < 0.0f) { v.x = fm(fs(1.0f, fabsf(ey)), sx); v.y = fm(fs(1.0f, fabsf(ex)), sy); }
  return vnormalize(v);
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
  a = saturate(fd(r[0], r[2]));
  b = saturate(fd(r[1], r[3]));
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
  Vec3 N, V, albedo, F0, energy;
  float metallic, alpha2, NoV;
};

// pbr.slang:61-87 BRDF(V, N, L, ...): diffuse and specular
OXC_DI void pbr_brdf(const PbrSurface& s, Vec3 L, Vec3& diffuse, Vec3& specular) {
  const Vec3 VL = vec3(fa(s.V.x, L.x), fa(s.V.y, L.y), fa(s.V.z, L.z));
  const Vec3 H = vdot(VL, VL) > 1e-8f ? vnormalize(VL) : s.N;
  const float NoL = saturate(vdot(s.N, L));
  const float NoH = saturate(vdot(s.N, H));
  const float LoH = saturate(vdot(L, H));
  // D_GGX :11-14
  const float f = fa(fm(fs(fm(NoH, s.alpha2), NoH), NoH), 1.0f);
  const float D = fd(s.alpha2, fa(fm(fm(PI, f), f), 1e-7f));
  // V_SmithGGXCorrelated :16-20
  const float one_a2 = fs(1.0f, s.alpha2);
  const float GGXV = fm(NoL, fsq(fa(fm(fm(s.NoV, s.NoV), one_a2), s.alpha2)));
  const float GGXL = fm(s.NoV, fsq(fa(fm(fm(NoL, NoL), one_a2), s.alpha2)));
  const float Vis = saturate(fd(0.5f, fa(fa(GGXV, GGXL), 1e-7f)));
  // F_Schlick :22-24
  const float p5 = canonical_pow5(saturate(fs(1.0f, LoH)));
  const Vec3 F = vec3(fa(s.F0.x, fm(fs(1.0f, s.F0.x), p5)), fa(s.F0.y, fm(fs(1.0f, s.F0.y), p5)), fa(s.F0.z, fm(fs(1.0f, s.F0.z), p5)));
  const float DV = fm(D, Vis);
  specular = vec3(fm(fm(DV, F.x), s.energy.x), fm(fm(DV, F.y), s.energy.y), fm(fm(DV, F.z), s.energy.z));
  const float one_m = fs(1.0f, s.metallic);
  diffuse = vec3(fm(fm(fm(one_m, fs(1.0f, F.x)), s.albedo.x), PBR_INV_PI), fm(fm(fm(one_m, fs(1.0f, F.y)), s.albedo.y), PBR_INV_PI),
                 fm(fm(fm(one_m, fs(1.0f, F.z)), s.albedo.z), PBR_INV_PI));
}

// point_light_contribution (pbr.slang:102-130) and calculate_spot_light_contribution (:140-172), added to `total`; other kinds add
// nothing
OXC_DI void pbr_add_light(const PbrSurface& s, Vec3 world, const PbrLight& l, Vec3& total) {
  const uint32_t kind = __float_as_uint(l.cos_outer_kind.y);
  if (kind != PBR_LIGHT_POINT && kind != PBR_LIGHT_SPOT) return;
  const Vec3 lv = vec3(fs(l.pos_intensity.x, world.x), fs(l.pos_intensity.y, world.y), fs(l.pos_intensity.z, world.z));
  const float dist = fsq(vdot(lv, lv));
  const Vec3 L = vec3(fd(lv.x, dist), fd(lv.y, dist), fd(lv.z, dist));
  float att = pbr_attenuate_point(dist, l.color_range.w);
  if (kind == PBR_LIGHT_SPOT) {
    // calculate_spot_light_attenuation :132-138, smoothstep(cos_outer, cos_inner, dot(-L, normalize(direction)))
    const float cos_angle = dot3(-L.x, -L.y, -L.z, l.spot_cos_inner.x, l.spot_cos_inner.y, l.spot_cos_inner.z);
    const float e0 = l.cos_outer_kind.x, e1 = l.spot_cos_inner.w;
    const float t = saturate(fd(fs(cos_angle, e0), fs(e1, e0)));
    att = fm(att, fm(fm(t, t), fs(3.0f, fm(2.0f, t))));
  }
  const float intensity = l.pos_intensity.w;
  if (att <= 0.0f || intensity <= 0.0f) return;
  const float NdotL = saturate(vdot(s.N, L));
  if (NdotL <= 0.0f) return;
  Vec3 d, sp;
  pbr_brdf(s, L, d, sp);
  total.x = fa(total.x, fm(fm(fa(d.x, sp.x), fm(fm(l.color_range.x, att), intensity)), NdotL));
  total.y = fa(total.y, fm(fm(fa(d.y, sp.y), fm(fm(l.color_range.y, att), intensity)), NdotL));
  total.z = fa(total.z, fm(fm(fa(d.z, sp.z), fm(fm(l.color_range.z, att), intensity)), NdotL));
}

// what both fs_main variants compute from the G-buffer before their sky tests (pbr_apply_no_atmos.slang:40-67, pbr_apply.slang:57-83):
// the surface terms that depend on no light and no sky (PbrSurface's N, V and NoV; the rest is set by pbr_shade), the world position,
// R, the smooth normal and NoL
struct PbrPixel {
  PbrSurface s;
  Vec3 world, R, smooth, Ls;
  float4 alb, em;
  float u, v, metallic, roughness, occlusion, NoL;
};

OXC_DI PbrPixel pbr_prologue(const PbrParams& p, size_t pix, float depth, int x, int y) {
  PbrPixel q;
  q.u = fd(fa((float)x, 0.5f), (float)p.width); q.v = fd(fa((float)y, 0.5f), (float)p.height);
  q.alb = __ldg(p.albedo + pix);
  const float4 nrm = __ldg(p.normal + pix);
  const Vec3 mapped = pbr_oct_to_vec3(round_to_half(nrm.x), round_to_half(nrm.y));
  q.smooth = pbr_oct_to_vec3(round_to_half(nrm.z), round_to_half(nrm.w));
  q.em = __ldg(p.emissive + pix);
  const float4 mro = __ldg(p.mro + pix);
  q.metallic = saturate(mro.x);
  q.roughness = vmin(vmax(mro.y, 0.045f), 1.0f);
  const float ssao = p.ao ? round_to_half(__ldg(p.ao + pix)) : 1.0f;
  q.occlusion = fm(mro.z, ssao);
  // world position :56-58
  const float nx = fs(fm(q.u, 2.0f), 1.0f), ny = fs(fm(q.v, 2.0f), 1.0f);
  float h[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const float4 r = p.inv_pv_row[i];
    h[i] = fa(fa(fa(fm(r.x, nx), fm(r.y, ny)), fm(r.z, depth)), fm(r.w, 1.0f));
  }
  q.world = vec3(fd(h[0], h[3]), fd(h[1], h[3]), fd(h[2], h[3]));
  // :63-67
  q.s.V = vnormalize(vec3(fs(p.cam_pos[0], q.world.x), fs(p.cam_pos[1], q.world.y), fs(p.cam_pos[2], q.world.z)));
  q.s.N = vnormalize(mapped);
  const Vec3 I = vec3(-q.s.V.x, -q.s.V.y, -q.s.V.z);
  const float dIN = vdot(I, q.s.N);
  q.R = vec3(fs(I.x, fm(fm(2.0f, q.s.N.x), dIN)), fs(I.y, fm(fm(2.0f, q.s.N.y), dIN)), fs(I.z, fm(fm(2.0f, q.s.N.z), dIN)));
  q.s.NoV = fa(fabsf(vdot(q.s.N, q.s.V)), 1e-5f);
  q.Ls = vec3(p.sun[0], p.sun[1], p.sun[2]);
  q.NoL = vmax(vdot(q.s.N, q.Ls), 0.0f);
  return q;
}

// directional_shadow * contact_shadow (pbr_apply_no_atmos.slang:73-75, pbr_apply.slang:85-87)
OXC_DI float pbr_visibility(const PbrParams& p, size_t pix, bool has_dir) {
  const float dshadow = has_dir && p.shadow ? __ldg(p.shadow + pix) : 1.0f;
  const float cshadow = (p.flags & PBR_FLAG_CONTACT) ? __ldg(p.contact + pix) : 1.0f;
  return fm(dshadow, cshadow);
}

// what both variants compute after their sky terms (pbr_apply_no_atmos.slang:86-126, pbr_apply.slang:143-183), with the variant's
// diffuse and specular sky and per-channel direct illuminance: the stored (((surface + lights) + indirect) + emission) [+ aerial], the
// aerial perspective term added only where `aerial` is given
OXC_DI float4 pbr_shade(const PbrParams& p, const PbrLight* lights, PbrPixel& q, const Vec3& diffuse_sky, const Vec3& specular_sky,
                        const Vec3& direct, float visibility, const Vec3* aerial) {
  PbrSurface& s = q.s;
  const float4 alb = q.alb;
  const float metallic = q.metallic, roughness = q.roughness, occlusion = q.occlusion;
  // :86-100
  s.albedo = vec3(alb.x, alb.y, alb.z);
  s.metallic = metallic;
  s.F0 = vec3(fa(0.04f, fm(fs(alb.x, 0.04f), metallic)), fa(0.04f, fm(fs(alb.y, 0.04f), metallic)), fa(0.04f, fm(fs(alb.z, 0.04f), metallic)));
  const float alpha = vmax(fm(roughness, roughness), 0.0025f);
  s.alpha2 = fm(alpha, alpha);
  float ABx, ABy;
  pbr_ggx_directional_albedo(s.NoV, alpha, ABx, ABy);
  const Vec3 kS = vec3(fa(fm(s.F0.x, ABx), ABy), fa(fm(s.F0.y, ABx), ABy), fa(fm(s.F0.z, ABx), ABy));
  const float one_m = fs(1.0f, metallic);
  const Vec3 kD = vec3(fm(one_m, fs(1.0f, kS.x)), fm(one_m, fs(1.0f, kS.y)), fm(one_m, fs(1.0f, kS.z)));
  // specular_occlusion_horizon :52-54
  const float spec_occ = saturate(fa(fs(canonical_pow(fa(s.NoV, occlusion), canonical_pow(2.0f, fs(fm(-16.0f, roughness), 1.0f))), 1.0f), occlusion));
  const Vec3 indirect = vec3(fa(fm(fm(fm(fm(kD.x, diffuse_sky.x), alb.x), PBR_INV_PI), occlusion), fm(fm(kS.x, specular_sky.x), spec_occ)),
                             fa(fm(fm(fm(fm(kD.y, diffuse_sky.y), alb.y), PBR_INV_PI), occlusion), fm(fm(kS.y, specular_sky.y), spec_occ)),
                             fa(fm(fm(fm(fm(kD.z, diffuse_sky.z), alb.z), PBR_INV_PI), occlusion), fm(fm(kS.z, specular_sky.z), spec_occ)));
  // GGX_energy_compensation :46-50, which depends on no light
  const float Ess = saturate(fa(ABx, ABy));
  const float one_ess = fs(1.0f, Ess), ess_den = vmax(Ess, 1e-4f);
  s.energy = vec3(fa(1.0f, fd(fm(s.F0.x, one_ess), ess_den)), fa(1.0f, fd(fm(s.F0.y, one_ess), ess_den)), fa(1.0f, fd(fm(s.F0.z, one_ess), ess_den)));
  // :102-113
  Vec3 total = vec3(0.0f, 0.0f, 0.0f);
  for (uint32_t i = 0; i < p.light_count; i++) pbr_add_light(s, q.world, lights[i], total);
  // :115-123
  float horizon = saturate(fa(1.0f, fm(1.3f, vdot(q.R, q.smooth))));
  horizon = fm(horizon, horizon);
  Vec3 surf = vec3(0.0f, 0.0f, 0.0f);
  if (q.NoL > 0.0f) {
    Vec3 d, sp;
    pbr_brdf(s, q.Ls, d, sp);
    surf = vec3(fm(fm(fm(fa(d.x, fm(sp.x, horizon)), direct.x), q.NoL), visibility), fm(fm(fm(fa(d.y, fm(sp.y, horizon)), direct.y), q.NoL), visibility),
                fm(fm(fm(fa(d.z, fm(sp.z, horizon)), direct.z), q.NoL), visibility));
  }
  // :125-126
  const float4 em = q.em;
  if (aerial)
    return make_float4(nan_canonical(fa(fa(fa(fa(surf.x, total.x), indirect.x), em.x), aerial->x)),
                       nan_canonical(fa(fa(fa(fa(surf.y, total.y), indirect.y), em.y), aerial->y)),
                       nan_canonical(fa(fa(fa(fa(surf.z, total.z), indirect.z), em.z), aerial->z)), 1.0f);
  return make_float4(nan_canonical(fa(fa(fa(surf.x, total.x), indirect.x), em.x)), nan_canonical(fa(fa(fa(surf.y, total.y), indirect.y), em.y)),
                     nan_canonical(fa(fa(fa(surf.z, total.z), indirect.z), em.z)), 1.0f);
}

// fs_main (pbr_apply_no_atmos.slang:23-127) of pixel (x, y) with the staged lights
OXC_DI float4 pbr_pixel(const PbrParams& p, const PbrLight* lights, int x, int y) {
  const size_t pix = (size_t)y * p.width + x;
  const float depth = p.depth[pix];
  if ((p.flags & PBR_FLAG_TRANSPARENT) && depth == 0.0f) return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  PbrPixel q = pbr_prologue(p, pix, depth, x, y);
  if ((p.flags & PBR_FLAG_SKY) && depth == 0.0f)
    return p.sky_has_texture ? make_float4(1.0f, 1.0f, 1.0f, 1.0f)
                             : make_float4(nan_canonical(p.sky_solid.x), nan_canonical(p.sky_solid.y), nan_canonical(p.sky_solid.z), nan_canonical(p.sky_solid.w));
  const bool has_dir = (p.flags & PBR_FLAG_DIRECTIONAL) != 0;
  const float visibility = pbr_visibility(p, pix, has_dir);
  const float direct = has_dir ? p.sun_intensity : 0.0f;
  const bool has_sky = (p.flags & PBR_FLAG_SKY) != 0;
  const Vec3 env = has_sky ? vec3(p.sky_ambient[0], p.sky_ambient[1], p.sky_ambient[2]) : vec3(p.base_ambient[0], p.base_ambient[1], p.base_ambient[2]);
  return pbr_shade(p, lights, q, env, env, vec3(direct, direct, direct), visibility, nullptr);
}

} // namespace oxc
