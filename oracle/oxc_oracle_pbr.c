/*
 * oxc_oracle_pbr.c — CPU ORACLE (test infrastructure) of PBR apply without atmosphere: RendererInstance::apply_pbr's
 * pbr_apply_no_atmos pass (Passes/PBR.cpp:435-531), passes/pbr_apply_no_atmos.slang:23-127 and the pbr.slang:1-172 functions it
 * calls, one C function per shader function, in the shader's structure (the BRDF recomputes everything per call; the kernel hoists
 * what does not depend on the light, which gives the same bits).  Same rules as oxc_oracle.c: plain C11, IEEE binary32 with round to
 * nearest, no contraction, IEEE divide / sqrt, products and sums left to right as written, dot(a, b) = (a.x*b.x + a.y*b.y) + a.z*b.z,
 * mul(M, v) row by row in the same order.  It is one translation unit with oxc_oracle_gtao.c (and so oxc_oracle_vsm_resolve.c and
 * oxc_oracle.c), included below, so that it runs the library's own sin / cos, pow and binary16 rounding.  Built into
 * liboxc_oracle_pbr.so by oracle/pyoracle_pbr.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_pbr.c -lm
 *
 * SPECIFICATION of orc_apply_pbr (include/oxcull.h oxc_apply_pbr repeats it).  Where the shader does not define an outcome, this
 * commits to one:
 *   1. pixel centre: tex_coord = ((x + 0.5) / W, (y + 0.5) / H).  SampleLevel(linear_repeat, tex_coord, 0) of the albedo at a pixel
 *      centre has bilinear weights of exactly 0: the pixel's own texel.
 *   2. the normal plane's four components are rounded to binary16 (R16G16B16A16F, round to nearest even); both oct_to_vec3 follow
 *      common/encoding.slang:7-15 (which normalizes); N = normalize(mapped_normal) is normalized a second time, as written.
 *   3. the ambient occlusion is rounded to binary16 (R16F); albedo, emissive, metallic / roughness / occlusion, shadow and contact
 *      shadow are the binary32 values given.  NULL ambient occlusion and shadow read as 1.0 (the reference clears both to White); the
 *      shadow is read under HasDirectionalLight, the contact shadow only under HasContactShadows.
 *   4. transcendentals: cos of the cone angles orc_sincos_canonical; exp2(e) = orc_pow_canonical(2, e); pow(NoV + ao, .) =
 *      orc_pow_canonical; pow(., 5.0) = orc_pow5_canonical (below).
 *   5. operations: normalize(v) = v / sqrt(dot(v, v)); length = sqrt(dot); lerp(a, b, t) = a + (b - a) * t; reflect(i, n) = i -
 *      (2 * n) * dot(i, n); max / min return the other operand for a NaN, clamp(x, a, b) = min(max(x, a), b), saturate(NaN) = 0;
 *      smoothstep(e0, e1, x) = (t * t) * (3 - 2 * t), t = saturate((x - e0) / (e1 - e0)); Fd_Lambert = fl(1 / fl(pi)); constants
 *      are the binary32 roundings of the literals; a scalar times a vector is applied per component.
 *   6. a light kind other than Point (1) or Spot (2) contributes nothing; the lights are summed in index order.
 *   7. early returns in shader order: TransparentBackground and depth == 0 -> (0, 0, 0, 0); HasSky and depth == 0 -> has_texture ?
 *      (1, 1, 1, 1) : solid_color; otherwise the full computation, also on sky pixels without HasSky.
 *   8. output: binary32 RGBA (the value before the reference's B10G11R11 / RGBA16F store); every NaN is stored as 0x7FFFFFFF.
 * orc_pow5_canonical: x2 = x * x in binary64 (exact), (x2 * x2) * x in binary64, one rounding to binary32; within 1 ulp of the
 * correctly rounded power (the proof is at oxc_exact.cuh canonical_pow5).
 */
#include "oxc_oracle_gtao.c"

#include "oxc_oracle_pbr.h"

#define P_PI 3.1415926535897932384626433832795f /* common/math.slang */
#define P_MIN_ALPHA 0.0025f                      /* pbr.slang:4 */
#define P_SCENE_DIRECTIONAL (1u << 0)
#define P_SCENE_CONTACT (1u << 9)
#define P_SCENE_SKY (1u << 10)
#define P_SCENE_TRANSPARENT (1u << 11)

typedef struct { float x, y, z; } pv3;
static pv3 pv(float x, float y, float z) { pv3 r = {x, y, z}; return r; }
static pv3 pv_s(float s) { return pv(s, s, s); }
static pv3 pv_add(pv3 a, pv3 b) { return pv(a.x + b.x, a.y + b.y, a.z + b.z); }
static pv3 pv_sub(pv3 a, pv3 b) { return pv(a.x - b.x, a.y - b.y, a.z - b.z); }
static pv3 pv_mul(pv3 a, pv3 b) { return pv(a.x * b.x, a.y * b.y, a.z * b.z); }
static pv3 pv_div(pv3 a, pv3 b) { return pv(a.x / b.x, a.y / b.y, a.z / b.z); }
static pv3 pv_neg(pv3 a) { return pv(-a.x, -a.y, -a.z); }
static float pv_dot(pv3 a, pv3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
static float pv_length(pv3 a) { return sqrtf(pv_dot(a, a)); }
static pv3 pv_normalize(pv3 a) { return pv_div(a, pv_s(sqrtf(pv_dot(a, a)))); }
static float p_max(float a, float b) { return (b != b || a > b) ? a : b; }
static float p_min(float a, float b) { return (b != b || a < b) ? a : b; }
static float p_clamp(float x, float lo, float hi) { return p_min(p_max(x, lo), hi); }
static float p_sat(float x) { return p_clamp(x, 0.0f, 1.0f); }
static pv3 pv_lerp(pv3 a, pv3 b, float t) { return pv_add(a, pv_mul(pv_sub(b, a), pv_s(t))); }
static pv3 pv_reflect(pv3 i, pv3 n) { return pv_sub(i, pv_mul(pv_mul(pv_s(2.0f), n), pv_s(pv_dot(i, n)))); }
static float p_store(float v) { return v != v ? bits2f(0x7FFFFFFFu) : v; }

float orc_pow5_canonical(float xf) {
  const double x = (double)xf;
  const double x2 = x * x;
  return (float)((x2 * x2) * x);
}

void orc_pow5_canonical_n(const float* x, float* out, uint64_t n) {
  for (uint64_t i = 0; i < n; i++) out[i] = orc_pow5_canonical(x[i]);
}

float orc_pbr_smoothstep(float e0, float e1, float x) {
  const float t = p_sat((x - e0) / (e1 - e0));
  return (t * t) * (3.0f - 2.0f * t);
}

void orc_pbr_oct_to_vec3(float ex, float ey, float out[3]) {
  pv3 v = pv(ex, ey, (1.0f - fabsf(ex)) - fabsf(ey));
  const float sx = (v.x >= 0.0f) ? 1.0f : -1.0f, sy = (v.y >= 0.0f) ? 1.0f : -1.0f;
  if (v.z < 0.0f) {
    const float nx = (1.0f - fabsf(v.y)) * sx, ny = (1.0f - fabsf(v.x)) * sy;
    v.x = nx;
    v.y = ny;
  }
  v = pv_normalize(v);
  out[0] = v.x; out[1] = v.y; out[2] = v.z;
}
static pv3 p_oct_to_vec3(float ex, float ey) {
  float o[3];
  orc_pbr_oct_to_vec3(ex, ey, o);
  return pv(o[0], o[1], o[2]);
}

/* pbr.slang:6-9 */
static float p_perceptual_roughness_to_alpha(float r) { return p_max(r * r, P_MIN_ALPHA); }

/* :11-14 */
static float p_D_GGX(float NoH, float alpha2) {
  const float f = (NoH * alpha2 - NoH) * NoH + 1.0f;
  return alpha2 / (P_PI * f * f + 1e-7f);
}

/* :16-20 */
static float p_V_SmithGGXCorrelated(float NoV, float NoL, float alpha2) {
  const float GGXV = NoL * sqrtf(NoV * NoV * (1.0f - alpha2) + alpha2);
  const float GGXL = NoV * sqrtf(NoL * NoL * (1.0f - alpha2) + alpha2);
  return p_sat(0.5f / (GGXV + GGXL + 1e-7f));
}

/* :22-24 */
static pv3 p_F_Schlick(float LoH, pv3 F0) {
  return pv_add(F0, pv_mul(pv_sub(pv_s(1.0f), F0), pv_s(orc_pow5_canonical(p_sat(1.0f - LoH)))));
}

/* :31-33 */
static float p_Fd_Lambert(void) { return 1.0f / P_PI; }

/* :35-44 */
void orc_pbr_ggx_directional_albedo(float NoV, float alpha, float out[2]) {
  static const float c[9][4] = {{0.1003f, 0.9345f, 1.0f, 1.0f},      {-0.6303f, -2.323f, -1.765f, 0.2281f}, {9.748f, 2.229f, 8.263f, 15.94f},
                                {-2.038f, -3.748f, 11.53f, -55.83f},  {29.34f, 1.424f, 28.96f, 13.08f},     {-8.245f, -0.7684f, -7.507f, 41.26f},
                                {-26.44f, 1.436f, -36.11f, 54.9f},    {19.99f, 0.2913f, 15.86f, 300.2f},    {-5.448f, 0.6286f, 33.37f, -285.1f}};
  const float x = NoV, y = alpha, x2 = x * x, y2 = y * y;
  float r[4];
  for (int i = 0; i < 4; i++)
    r[i] = c[0][i] + c[1][i] * x + c[2][i] * y + c[3][i] * x * y + c[4][i] * x2 + c[5][i] * y2 + c[6][i] * x2 * y + c[7][i] * x * y2 +
           c[8][i] * x2 * y2;
  out[0] = p_clamp(r[0] / r[2], 0.0f, 1.0f);
  out[1] = p_clamp(r[1] / r[3], 0.0f, 1.0f);
}

/* :46-50 */
static pv3 p_GGX_energy_compensation(float NoV, float alpha, pv3 Fss) {
  float AB[2];
  orc_pbr_ggx_directional_albedo(NoV, alpha, AB);
  const float Ess = p_sat(AB[0] + AB[1]);
  return pv_add(pv_s(1.0f), pv_div(pv_mul(Fss, pv_s(1.0f - Ess)), pv_s(p_max(Ess, 1e-4f))));
}

/* :52-54 */
static float p_specular_occlusion_horizon(float NoV, float ao, float perceptual_roughness) {
  return p_sat(orc_pow_canonical(NoV + ao, orc_pow_canonical(2.0f, -16.0f * perceptual_roughness - 1.0f)) - 1.0f + ao);
}

/* :61-87 */
static void p_BRDF(pv3 V, pv3 N, pv3 L, pv3 albedo, float perceptual_roughness, float metallic, pv3* diffuse, pv3* specular) {
  const pv3 VL = pv_add(V, L);
  const pv3 H = pv_dot(VL, VL) > 1e-8f ? pv_normalize(VL) : N;
  const float NoV = fabsf(pv_dot(N, V)) + 1e-5f;
  const float NoL = p_sat(pv_dot(N, L));
  const float NoH = p_sat(pv_dot(N, H));
  const float LoH = p_sat(pv_dot(L, H));
  const pv3 F0 = pv_lerp(pv_s(0.04f), albedo, metallic);
  const float alpha = p_perceptual_roughness_to_alpha(perceptual_roughness);
  const float alpha2 = alpha * alpha;
  const float D = p_D_GGX(NoH, alpha2);
  const float Vis = p_V_SmithGGXCorrelated(NoV, NoL, alpha2);
  const pv3 F = p_F_Schlick(LoH, F0);
  const pv3 energy_compensation = p_GGX_energy_compensation(NoV, alpha, F0);
  *specular = pv_mul(pv_mul(pv_s(D * Vis), F), energy_compensation);
  const pv3 kd = pv_mul(pv_s(1.0f - metallic), pv_sub(pv_s(1.0f), F));
  *diffuse = pv_mul(pv_mul(kd, albedo), pv_s(p_Fd_Lambert()));
}

/* :89-100 */
float orc_pbr_attenuate_point(float to_light_dist, float cutoff) {
  if (cutoff <= 0.0f) return 1.0f / (to_light_dist * to_light_dist + 0.1f);
  float win = to_light_dist / cutoff;
  win = win * win * win * win;
  win = p_max(0.0f, 1.0f - win);
  win = win * win;
  return win / (to_light_dist * to_light_dist + 0.1f);
}

/* :102-130 */
static pv3 p_point_light_contribution(pv3 world_position, pv3 N, pv3 V, pv3 albedo, float roughness, float metallic, pv3 light_position,
                                      const OxcLight* light) {
  const pv3 light_vector = pv_sub(light_position, world_position);
  const float light_distance = pv_length(light_vector);
  const pv3 L = pv_div(light_vector, pv_s(light_distance));
  const float attenuation = orc_pbr_attenuate_point(light_distance, light->range);
  if (attenuation <= 0.0f || light->intensity <= 0.0f) return pv_s(0.0f);
  const float NdotL = p_sat(pv_dot(N, L));
  if (NdotL <= 0.0f) return pv_s(0.0f);
  pv3 d, s;
  p_BRDF(V, N, L, albedo, roughness, metallic, &d, &s);
  const pv3 radiance = pv_mul(pv_mul(pv(light->color[0], light->color[1], light->color[2]), pv_s(attenuation)), pv_s(light->intensity));
  return pv_mul(pv_mul(pv_add(d, s), radiance), pv_s(NdotL));
}

/* :132-138 */
float orc_pbr_spot_attenuation(const float Ld[3], const float sd[3], float inner_cone_angle, float outer_cone_angle) {
  const float cos_angle = pv_dot(pv_neg(pv(Ld[0], Ld[1], Ld[2])), pv_normalize(pv(sd[0], sd[1], sd[2])));
  float s, cos_inner, cos_outer;
  orc_sincos_canonical(inner_cone_angle, &s, &cos_inner);
  orc_sincos_canonical(outer_cone_angle, &s, &cos_outer);
  return orc_pbr_smoothstep(cos_outer, cos_inner, cos_angle);
}

/* :140-172 */
static pv3 p_spot_light_contribution(pv3 world_position, pv3 N, pv3 V, pv3 albedo, float roughness, float metallic, pv3 light_position,
                                     pv3 light_direction, const OxcLight* light) {
  const pv3 light_vector = pv_sub(light_position, world_position);
  const float light_distance = pv_length(light_vector);
  const pv3 L = pv_div(light_vector, pv_s(light_distance));
  const float distance_attenuation = orc_pbr_attenuate_point(light_distance, light->range);
  const float Ld[3] = {L.x, L.y, L.z}, sd[3] = {light_direction.x, light_direction.y, light_direction.z};
  const float spot_attenuation = orc_pbr_spot_attenuation(Ld, sd, light->inner_cone_angle, light->outer_cone_angle);
  const float total_attenuation = distance_attenuation * spot_attenuation;
  if (total_attenuation <= 0.0f || light->intensity <= 0.0f) return pv_s(0.0f);
  const float NdotL = p_sat(pv_dot(N, L));
  if (NdotL <= 0.0f) return pv_s(0.0f);
  pv3 d, s;
  p_BRDF(V, N, L, albedo, roughness, metallic, &d, &s);
  const pv3 radiance = pv_mul(pv_mul(pv(light->color[0], light->color[1], light->color[2]), pv_s(total_attenuation)), pv_s(light->intensity));
  return pv_mul(pv_mul(pv_add(d, s), radiance), pv_s(NdotL));
}

/* pbr_apply_no_atmos.slang:23-127 fs_main of pixel (x, y) */
static void p_fs_main(const OxcPbrCamera* cam, const OxcPbrSettings* st, const OxcLight* lights, const float* depth_img, const float* albedo_img,
                      const float* normal_img, const float* emissive_img, const float* mro_img, const float* gtao_img, const float* shadow_img,
                      const float* contact_img, uint32_t W, uint32_t H, uint32_t x, uint32_t y, float out[4]) {
  const size_t pix = (size_t)y * W + x;
  const uint32_t flags = st->scene_flags;
  const float depth = depth_img[pix];
  if ((flags & P_SCENE_TRANSPARENT) != 0 && depth == 0.0f) {
    out[0] = out[1] = out[2] = out[3] = 0.0f;
    return;
  }
  const float tc[2] = {((float)x + 0.5f) / (float)W, ((float)y + 0.5f) / (float)H};
  const float* a = albedo_img + pix * 4;
  const pv3 albedo_color = pv(a[0], a[1], a[2]);
  const float* ms = normal_img + pix * 4;
  const pv3 mapped_normal = p_oct_to_vec3(orc_round_to_half(ms[0]), orc_round_to_half(ms[1]));
  const pv3 smooth_normal = p_oct_to_vec3(orc_round_to_half(ms[2]), orc_round_to_half(ms[3]));
  const float* e = emissive_img + pix * 4;
  const pv3 emission = pv(e[0], e[1], e[2]);
  const float* mro = mro_img + pix * 4;
  const float metallic = p_clamp(mro[0], 0.0f, 1.0f);
  const float roughness = p_clamp(mro[1], 0.045f, 1.0f);
  const float baked_occlusion = mro[2];
  const float screen_space_occlusion = gtao_img ? orc_round_to_half(gtao_img[pix]) : 1.0f;
  const float occlusion = baked_occlusion * screen_space_occlusion;
  const float ndc[4] = {tc[0] * 2.0f - 1.0f, tc[1] * 2.0f - 1.0f, depth, 1.0f};
  float wh[4];
  const float* M = cam->inv_projection_view; /* column-major: M[col * 4 + row] */
  for (int r = 0; r < 4; r++) wh[r] = M[r] * ndc[0] + M[4 + r] * ndc[1] + M[8 + r] * ndc[2] + M[12 + r] * ndc[3];
  const pv3 world_position = pv_div(pv(wh[0], wh[1], wh[2]), pv_s(wh[3]));
  const int has_directional_light = (flags & P_SCENE_DIRECTIONAL) != 0;
  const pv3 L = pv(st->sun_direction[0], st->sun_direction[1], st->sun_direction[2]);
  const pv3 V = pv_normalize(pv_sub(pv(cam->position[0], cam->position[1], cam->position[2]), world_position));
  const pv3 N = pv_normalize(mapped_normal);
  const pv3 R = pv_reflect(pv_neg(V), N);
  const float NoV = fabsf(pv_dot(N, V)) + 1e-5f;
  const float NoL = p_max(pv_dot(N, L), 0.0f);
  if ((flags & P_SCENE_SKY) != 0 && depth == 0.0f) {
    for (int i = 0; i < 4; i++) out[i] = st->sky_has_texture ? 1.0f : p_store(st->sky_solid_color[i]);
    return;
  }
  const float directional_shadow = has_directional_light ? (shadow_img ? shadow_img[pix] : 1.0f) : 1.0f;
  const float contact_shadow = (flags & P_SCENE_CONTACT) != 0 ? contact_img[pix] : 1.0f;
  const float visibility = directional_shadow * contact_shadow;
  pv3 indirect_illuminance;
  const pv3 direct_illuminance = has_directional_light ? pv_s(st->sun_intensity) : pv_s(0.0f);
  const int has_sky = (flags & P_SCENE_SKY) != 0;
  const pv3 environment_radiance = has_sky ? pv(st->sky_ambient_color[0], st->sky_ambient_color[1], st->sky_ambient_color[2])
                                           : pv(st->base_ambient_color[0], st->base_ambient_color[1], st->base_ambient_color[2]);
  const pv3 diffuse_sky = environment_radiance, specular_sky = environment_radiance;
  {
    const pv3 F0 = pv_lerp(pv_s(0.04f), albedo_color, metallic);
    const float alpha = p_perceptual_roughness_to_alpha(roughness);
    float AB[2];
    orc_pbr_ggx_directional_albedo(NoV, alpha, AB);
    const pv3 kS = pv_add(pv_mul(F0, pv_s(AB[0])), pv_s(AB[1]));
    const pv3 kD = pv_mul(pv_s(1.0f - metallic), pv_sub(pv_s(1.0f), kS));
    const float spec_occlusion = p_specular_occlusion_horizon(NoV, occlusion, roughness);
    const pv3 ibl_diffuse = pv_mul(pv_mul(pv_mul(kD, diffuse_sky), albedo_color), pv_s(p_Fd_Lambert()));
    const pv3 ibl_specular = pv_mul(pv_mul(kS, specular_sky), pv_s(spec_occlusion));
    indirect_illuminance = pv_add(pv_mul(ibl_diffuse, pv_s(occlusion)), ibl_specular);
  }
  pv3 total_lighting = pv(0.0f, 0.0f, 0.0f);
  for (uint32_t i = 0; i < st->light_count; i++) {
    const OxcLight* light = &lights[i];
    const pv3 lp = pv(light->position[0], light->position[1], light->position[2]);
    if (light->kind == 1u)
      total_lighting = pv_add(total_lighting, p_point_light_contribution(world_position, N, V, albedo_color, roughness, metallic, lp, light));
    else if (light->kind == 2u)
      total_lighting = pv_add(total_lighting, p_spot_light_contribution(world_position, N, V, albedo_color, roughness, metallic, lp,
                                                                        pv(light->direction[0], light->direction[1], light->direction[2]), light));
  }
  const float horizon_fade = 1.3f;
  float horizon = p_sat(1.0f + horizon_fade * pv_dot(R, smooth_normal));
  horizon *= horizon;
  pv3 material_surface_color = pv(0.0f, 0.0f, 0.0f);
  if (NoL > 0.0f) {
    pv3 d, s;
    p_BRDF(V, N, L, albedo_color, roughness, metallic, &d, &s);
    material_surface_color = pv_mul(pv_mul(pv_mul(pv_add(d, pv_mul(s, pv_s(horizon))), direct_illuminance), pv_s(NoL)), pv_s(visibility));
  }
  const pv3 final_color = pv_add(pv_add(pv_add(material_surface_color, total_lighting), indirect_illuminance), emission);
  out[0] = p_store(final_color.x);
  out[1] = p_store(final_color.y);
  out[2] = p_store(final_color.z);
  out[3] = 1.0f;
}

void orc_apply_pbr(const OxcPbrCamera* camera, const OxcPbrSettings* settings, const OxcLight* lights, const float* depth, const float* albedo,
                   const float* normal, const float* emissive, const float* metallic_roughness_occlusion, const float* ambient_occlusion,
                   const float* shadow, const float* contact_shadow, uint32_t width, uint32_t height, float* out) {
  for (uint32_t y = 0; y < height; y++)
    for (uint32_t x = 0; x < width; x++)
      p_fs_main(camera, settings, lights, depth, albedo, normal, emissive, metallic_roughness_occlusion, ambient_occlusion, shadow,
                contact_shadow, width, height, x, y, out + ((size_t)y * width + x) * 4);
}
