/*
 * oxc_oracle_pbr.h — CPU ORACLE of PBR apply without atmosphere (RendererInstance::apply_pbr, Passes/PBR.cpp:435-531,
 * passes/pbr_apply_no_atmos.slang:23-127, pbr.slang:1-172); the specification of include/oxcull.h oxc_apply_pbr (comment at the top
 * of oxc_oracle_pbr.c).  TEST INFRASTRUCTURE ONLY: only tests/ and tools/ load liboxc_oracle_pbr.so (oracle/pyoracle_pbr.py), which
 * also holds everything of oxc_oracle_gtao.h.
 */
#ifndef OXC_ORACLE_PBR_H_
#define OXC_ORACLE_PBR_H_

#include "oxc_oracle_gtao.h"

#ifdef __cplusplus
extern "C" {
#endif

/* pow(x, 5.0) of F_Schlick (oxc_exact.cuh canonical_pow5) */
float orc_pow5_canonical(float x);
/* element-wise orc_pow5_canonical of n values */
void orc_pow5_canonical_n(const float* x, float* out, uint64_t n);
/* GGX_directional_albedo(NoV, alpha) -> out[2] */
void orc_pbr_ggx_directional_albedo(float NoV, float alpha, float out[2]);
float orc_pbr_attenuate_point(float dist, float cutoff);
/* calculate_spot_light_attenuation(L, spot_direction, inner, outer) */
float orc_pbr_spot_attenuation(const float L[3], const float spot_direction[3], float inner_cone_angle, float outer_cone_angle);
/* smoothstep(e0, e1, x) */
float orc_pbr_smoothstep(float e0, float e1, float x);
/* oct_to_vec3(e) (common/encoding.slang:7-15) -> out[3] */
void orc_pbr_oct_to_vec3(float ex, float ey, float out[3]);

/* PBR apply of a width x height frame, all HOST arrays: depth (f32), albedo, normal, emissive, metallic_roughness_occlusion (float4
 * each), ambient_occlusion, shadow, contact_shadow (f32, NULL as in oxc_apply_pbr), lights (settings->light_count records); out
 * receives W x H float4. */
void orc_apply_pbr(const OxcPbrCamera* camera, const OxcPbrSettings* settings, const OxcLight* lights, const float* depth, const float* albedo,
                   const float* normal, const float* emissive, const float* metallic_roughness_occlusion, const float* ambient_occlusion,
                   const float* shadow, const float* contact_shadow, uint32_t width, uint32_t height, float* out);

#ifdef __cplusplus
}
#endif
#endif
