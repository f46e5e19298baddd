/*
 * oxc_oracle_pbr_atmosphere.c — CPU ORACLE (test infrastructure) of PBR apply under the atmosphere: RendererInstance::apply_pbr's
 * pbr_apply pass (Passes/PBR.cpp:312-432), passes/pbr_apply.slang:26-184 and the sky.slang functions it calls
 * (get_direct_sun_lighting :324-337, sky_view_params_to_lut_uv :39-67, sample_aerial_perspective :258-293), one C function per shader
 * function.  It is one translation unit with the PBR oracle (oxc_oracle_pbr.c: oct_to_vec3, the BRDF, GGX_directional_albedo,
 * specular_occlusion_horizon and the two light contributions) and the sky IBL oracle (oxc_oracle_sky_ibl.c and the atmosphere oracle it
 * includes: get_eye_pos, the transmittance parametrisation, the ray-sphere test, the sky-view uv, the tap rule, acos, atan2 and exp).  Both
 * include oxc_oracle_gtao.c; it is imported first (#import, GCC's include-once) so that the second inclusion is skipped and each function
 * is defined once.  Same rules as those oracles.  Built into liboxc_oracle_pbr_atmosphere.so by oracle/pyoracle_pbr_atmosphere.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_pbr_atmosphere.c -lm
 *
 * SPECIFICATION: include/oxcull.h above oxc_apply_pbr_atmosphere, items 1-7.
 */
#pragma GCC diagnostic ignored "-Wdeprecated"
#import "oxc_oracle_gtao.c"
#include "oxc_oracle_pbr.c"
#include "oxc_oracle_sky_ibl.c"

#include "oxc_oracle_pbr_atmosphere.h"

static const float PA_SUN_RADIANS = 0x1.1df46ap-6f, PA_HALF_SLICE = 0x1.6a09e6p-1f, PA_NEAR_FADE = 0x1.f3fffep+9f;

static float pa_min_cos(void) {
  float s, c;
  orc_sincos_canonical(PA_SUN_RADIANS, &s, &c);
  return c;
}

/* the constants the pass reads: the sun disc's argument and its min_cos, half_slice_depth, near_depth_fade_out */
void orc_pbra_constants(float out[4]) {
  out[0] = PA_SUN_RADIANS;
  out[1] = pa_min_cos();
  out[2] = PA_HALF_SLICE;
  out[3] = PA_NEAR_FADE;
}

/* pbr_apply.slang:26-38, one channel */
float orc_pbra_draw_sun(float cos_theta) {
  const float min_cos_theta = pa_min_cos();
  if (cos_theta >= min_cos_theta) return 1.0f;
  const float offset = min_cos_theta - cos_theta;
  const float gaussian_bloom = orc_exp_canonical(-offset * 50000.0f) * 0.5f;
  const float inv_bloom = 1.0f / (0.02f + offset * 300.0f) * 0.01f;
  return gaussian_bloom + inv_bloom;
}

/* the Vulkan face table, ties to X over Y over Z, >= 0 the positive face */
int orc_pbra_cube_face(const float r[3], float o[3]) {
  const float ax = fabsf(r[0]), ay = fabsf(r[1]), az = fabsf(r[2]);
  if (ax >= ay && ax >= az) {
    o[2] = r[0]; o[1] = -r[1];
    if (r[0] >= 0.0f) { o[0] = -r[2]; return 0; }
    o[0] = r[2]; return 1;
  }
  if (ay >= az) {
    o[2] = r[1]; o[0] = r[0];
    if (r[1] >= 0.0f) { o[1] = r[2]; return 2; }
    o[1] = -r[2]; return 3;
  }
  o[2] = r[2]; o[1] = -r[1];
  if (r[2] >= 0.0f) { o[0] = r[0]; return 4; }
  o[0] = -r[0]; return 5;
}

/* an off-face texel: the integer point of the cube (half-texel units, the face planes at +-32) moved onto the adjacent face */
uint32_t orc_pbra_cube_remap(uint32_t f, int32_t i, int32_t j) {
  int32_t a = 2 * i - 31, b = 2 * j - 31, m = 32;
  if (a < -32 || a > 32) { a = a < 0 ? -32 : 32; m = 31; }
  if (b < -32 || b > 32) { b = b < 0 ? -32 : 32; m = 31; }
  const int32_t P[6][3] = {{m, -b, -a}, {-m, -b, a}, {a, m, b}, {a, -m, -b}, {a, -b, m}, {-a, -b, -m}};
  const int32_t* p = P[f < 5 ? f : 5];
  float r[3] = {(float)p[0], (float)p[1], (float)p[2]}, o[3];
  const int nf = orc_pbra_cube_face(r, o);
  return ((uint32_t)nf * 32u + (uint32_t)(((int32_t)o[1] + 31) / 2)) * 32u + (uint32_t)(((int32_t)o[0] + 31) / 2);
}

static void pa_texel(const uint16_t* plane, size_t texel, float o[4]) {
  for (int c = 0; c < 4; c++) o[c] = g_half_float(plane[texel * 4 + c]);
}

static void pa_cube_fetch(const uint16_t* cube, uint32_t f, int32_t i, int32_t j, float o[4]) {
  const int oi = i < 0 || i > 31, oj = j < 0 || j > 31;
  if (!oi && !oj) { pa_texel(cube, ((size_t)f * 32 + (size_t)j) * 32 + (size_t)i, o); return; }
  if (!(oi && oj)) { pa_texel(cube, orc_pbra_cube_remap(f, i, j), o); return; }
  const int32_t ci = i < 0 ? 0 : 31, cj = j < 0 ? 0 : 31;
  float t0[4], t1[4], t2[4];
  pa_texel(cube, ((size_t)f * 32 + (size_t)cj) * 32 + (size_t)ci, t0);
  pa_texel(cube, orc_pbra_cube_remap(f, i, cj), t1);
  pa_texel(cube, orc_pbra_cube_remap(f, ci, j), t2);
  for (int c = 0; c < 4; c++) o[c] = ((t0[c] + t1[c]) + t2[c]) / 3.0f;
}

/* TextureCube.SampleLevel(linear_clamp, r, 0) */
void orc_pbra_cube_tap(const uint16_t* cube, const float r[3], float out[4]) {
  float o[3];
  const uint32_t f = (uint32_t)orc_pbra_cube_face(r, o);
  const float s = 0.5f * (o[0] / fabsf(o[2])) + 0.5f, t = 0.5f * (o[1] / fabsf(o[2])) + 0.5f;
  const float x = s * 32.0f - 0.5f, y = t * 32.0f - 0.5f;
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = x - x0, wy = y - y0;
  const int64_t ix = alpha_f2i(x0), iy = alpha_f2i(y0);
  const int32_t i0 = (int32_t)a_clampi(ix + 1, 34) - 1, i1 = (int32_t)a_clampi(ix + 2, 34) - 1;
  const int32_t j0 = (int32_t)a_clampi(iy + 1, 34) - 1, j1 = (int32_t)a_clampi(iy + 2, 34) - 1;
  float a00[4], a10[4], a01[4], a11[4];
  pa_cube_fetch(cube, f, i0, j0, a00);
  pa_cube_fetch(cube, f, i1, j0, a10);
  pa_cube_fetch(cube, f, i0, j1, a01);
  pa_cube_fetch(cube, f, i1, j1, a11);
  for (int c = 0; c < 4; c++) {
    const float top = a00[c] + wx * (a10[c] - a00[c]), bot = a01[c] + wx * (a11[c] - a01[c]);
    out[c] = top + wy * (bot - top);
  }
}

/* Texture3D.SampleLevel(linear_clamp, (u, v, w), 0): the 2D tap in slices z0 and z0 + 1, then a lerp in z */
void orc_pbra_tap3(const OxcAtmosphere* at, const uint16_t* lut, float u, float v, float w, float out[4]) {
  const uint32_t W = at->aerial_perspective_lut_size[0], H = at->aerial_perspective_lut_size[1], D = at->aerial_perspective_lut_size[2];
  const float z = w * (float)D - 0.5f;
  const float z0 = floorf(z);
  const float wz = z - z0;
  const int64_t iz = alpha_f2i(z0);
  float s0[4], s1[4];
  orc_sky_ibl_tap4(lut + (size_t)a_clampi(iz, D) * H * W * 4, W, H, u, v, s0);
  orc_sky_ibl_tap4(lut + (size_t)a_clampi(iz + 1, D) * H * W * 4, W, H, u, v, s1);
  for (int c = 0; c < 4; c++) out[c] = s0[c] + wz * (s1[c] - s0[c]);
}

/* sky.slang:258-293 */
void orc_pbra_aerial(const OxcAtmosphere* at, const uint16_t* lut, float u, float v, const float d[3], float out[4]) {
  const float lut_size[3] = {(float)at->aerial_perspective_lut_size[0], (float)at->aerial_perspective_lut_size[1],
                             (float)at->aerial_perspective_lut_size[2]};
  const float per_slice_depth = lut_size[0] / lut_size[2];
  const float aerial_perspective_lut_depth = lut_size[2];
  const float relative_depth = a_max(0.0f, a_length(d) - at->aerial_perspective_start_km);
  const float linear_slice = relative_depth * (1.0f / per_slice_depth);
  const float linear_w = linear_slice * (1.0f / aerial_perspective_lut_depth);
  const float non_linear_w = sqrtf(linear_w);
  const float non_linear_slice = non_linear_w * aerial_perspective_lut_depth;
  float weight = 1.0f;
  if (non_linear_slice < PA_HALF_SLICE) weight = p_sat(non_linear_slice * non_linear_slice * 2.0f);
  weight *= p_sat(relative_depth * PA_NEAR_FADE);
  orc_pbra_tap3(at, lut, u, v, non_linear_w, out);
  for (int c = 0; c < 3; c++) out[c] *= weight;
  out[3] = 1.0f - (weight * (1.0f - out[3]));
  for (int c = 0; c < 3; c++) out[c] *= at->aerial_perspective_exposure;
}

/* pbr_apply.slang:40-184 fs_main of pixel (x, y) */
static void pa_fs_main(const OxcPbrCamera* cam, const OxcPbrSettings* st, const OxcAtmosphere* at, const SkyCall* sc, const OxcLight* lights,
                       const float* depth_img, const float* albedo_img, const float* normal_img, const float* emissive_img,
                       const float* mro_img, const float* gtao_img, const float* shadow_img, const float* contact_img, const OxcPbrSky* sky,
                       uint32_t W, uint32_t H, uint32_t x, uint32_t y, float out[4]) {
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
  const float Li = st->sun_intensity;
  const pv3 cam_pos = pv(cam->position[0], cam->position[1], cam->position[2]);
  const pv3 V = pv_normalize(pv_sub(cam_pos, world_position));
  const pv3 N = pv_normalize(mapped_normal);
  const pv3 R = pv_reflect(pv_neg(V), N);
  const float NoV = fabsf(pv_dot(N, V)) + 1e-5f;
  const float NoL = p_max(pv_dot(N, L), 0.0f);
  const float directional_shadow = has_directional_light ? (shadow_img ? shadow_img[pix] : 1.0f) : 1.0f;
  const float contact_shadow = (flags & P_SCENE_CONTACT) != 0 ? contact_img[pix] : 1.0f;
  const float visibility = directional_shadow * contact_shadow;
  const float world_eye_pos_y = orc_atm_eye_y(at, world_position.y);
  const pv3 up = pv(0.0f, 1.0f, 0.0f);
  const float sun_cos_theta = pv_dot(L, up);
  const float horizon_darkening = orc_pbr_smoothstep(-0.1f, 0.3f, sun_cos_theta);
  float tuv[2], T[4];
  orc_atm_transmittance_uv(at->atmos_radius, at->planet_radius, world_eye_pos_y, sun_cos_theta, tuv);
  orc_sky_ibl_tap4(sky->transmittance, at->transmittance_lut_size[0], at->transmittance_lut_size[1], tuv[0], tuv[1], T);
  const pv3 sun_transmittance = pv(T[0], T[1], T[2]);
  const pv3 direct_illuminance = pv_mul(pv_mul(sun_transmittance, pv_s(Li)), pv_s(horizon_darkening));
  if (depth == 0.0f) {
    const float eye_pos[3] = {sc->eye[0], sc->eye[1], sc->eye[2]};
    const pv3 mV = pv_neg(V);
    float upa[3] = {0.0f, 1.0f, 0.0f}, mva[3] = {mV.x, mV.y, mV.z}, right_raw[3], right[3], fw_raw[3], forward[3], La[3] = {L.x, L.y, L.z};
    s_cross(upa, mva, right_raw);
    s_normalize(right_raw, right);
    s_cross(right, upa, fw_raw);
    s_normalize(fw_raw, forward);
    float lop[2] = {a_dot(La, forward), a_dot(La, right)};
    const float ll = sqrtf(lop[0] * lop[0] + lop[1] * lop[1]);
    lop[0] = lop[0] / ll; lop[1] = lop[1] / ll;
    const float view_zenith_cos_angle = a_dot(mva, upa);
    float t;
    const int hit = orc_atm_ray_sphere_nearest(eye_pos, mva, at->planet_radius, &t);
    float uv[2], s[4];
    s_sky_view_uv(sc, hit, view_zenith_cos_angle, lop, uv);
    orc_sky_ibl_tap4(sky->sky_view, at->sky_view_lut_size[0], at->sky_view_lut_size[1], uv[0], uv[1], s);
    if (!hit) {
      const float sun = orc_pbra_draw_sun(a_dot(mva, La)) * Li;
      for (int c = 0; c < 3; c++) s[c] += sun * T[c];
    }
    for (int c = 0; c < 3; c++) out[c] = p_store(s[c] * s[3]);
    out[3] = 1.0f;
    return;
  }
  float ap[4];
  const float crp[3] = {(world_position.x - cam_pos.x) * A_CSU, (world_position.y - cam_pos.y) * A_CSU, (world_position.z - cam_pos.z) * A_CSU};
  orc_pbra_aerial(at, sky->aerial_perspective, tc[0], tc[1], crp, ap);
  const pv3 aerial_perspective_contribution = pv_mul(pv(ap[0], ap[1], ap[2]), pv_s(ap[3]));
  const pv3 reflection_dir = pv_normalize(pv_lerp(N, R, 1.0f - roughness));
  float ss[4], ds[4];
  const float rd[3] = {reflection_dir.x, reflection_dir.y, reflection_dir.z}, nd[3] = {N.x, N.y, N.z};
  orc_pbra_cube_tap(sky->sky_cube, rd, ss);
  orc_pbra_cube_tap(sky->sky_cube, nd, ds);
  const pv3 specular_sky = pv_mul(pv_mul(pv(ss[0], ss[1], ss[2]), pv_s(ss[3])), pv_s(horizon_darkening));
  const pv3 diffuse_sky = pv_mul(pv_mul(pv(ds[0], ds[1], ds[2]), pv_s(ds[3])), pv_s(horizon_darkening));
  pv3 indirect_illuminance;
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
  const pv3 final_color =
      pv_add(pv_add(pv_add(pv_add(material_surface_color, total_lighting), indirect_illuminance), emission), aerial_perspective_contribution);
  out[0] = p_store(final_color.x);
  out[1] = p_store(final_color.y);
  out[2] = p_store(final_color.z);
  out[3] = 1.0f;
}

void orc_apply_pbr_atmosphere(const OxcPbrCamera* camera, const OxcPbrSettings* settings, const OxcAtmosphere* at, const OxcLight* lights,
                              const float* depth, const float* albedo, const float* normal, const float* emissive,
                              const float* metallic_roughness_occlusion, const float* ambient_occlusion, const float* shadow,
                              const float* contact_shadow, const OxcPbrSky* sky, uint32_t width, uint32_t height, float* out) {
  /* the camera's eye and the sky-view uv's beta / PI - beta for altitude eye.y (not length(eye)), once per call */
  SkyCall c;
  c.at = at;
  c.eye[0] = 0.0f; c.eye[1] = orc_atm_eye_y(at, camera->position[1]); c.eye[2] = 0.0f;
  c.height = c.eye[1];
  const float horizon = a_safe_sqrt(c.height * c.height - at->planet_radius * at->planet_radius);
  c.beta = orc_acos_canonical(horizon / c.height);
  c.zenith_horizon = A_PI - c.beta;
  for (uint32_t y = 0; y < height; y++)
    for (uint32_t x = 0; x < width; x++)
      pa_fs_main(camera, settings, at, &c, lights, depth, albedo, normal, emissive, metallic_roughness_occlusion, ambient_occlusion, shadow,
                 contact_shadow, sky, width, height, x, y, out + ((size_t)y * width + x) * 4);
}
