/*
 * oxc_oracle_contact_shadows.h — CPU ORACLE of the contact-shadow pass (RendererInstance.cpp:990-1020, passes/contact_shadows.slang
 * :29-78, raymarch.slang); the specification of include/oxcull.h oxc_contact_shadows (comment at the top of
 * oxc_oracle_contact_shadows.c).  TEST INFRASTRUCTURE ONLY: only tests/ and tools/ load liboxc_oracle_contact_shadows.so
 * (oracle/pyoracle_contact_shadows.py), which also holds everything of oxc_oracle_pbr.h.
 */
#ifndef OXC_ORACLE_CONTACT_SHADOWS_H_
#define OXC_ORACLE_CONTACT_SHADOWS_H_

#include "oxc_oracle_pbr.h"

#ifdef __cplusplus
extern "C" {
#endif

/* (1.0 + bias) of DepthRaymarchDistanceFn::call, as the pass uses it */
float orc_cs_bias_factor(void);
/* SampleLevel(nearest_clamp, (u, v), 0) of a W x H plane */
float orc_cs_nearest(const float* depth, uint32_t width, uint32_t height, float u, float v);
/* SampleLevel(linear_clamp, (u, v), 0) of a W x H plane */
float orc_cs_bilinear(const float* depth, uint32_t width, uint32_t height, float u, float v);
/* DepthRayMarch::to_cs_dir_impl(dir, false) after to_cs: the clipped ray from start_cs towards end_cs -> out[6] = (start, end) */
void orc_cs_clip_ray(const float start_cs[3], const float end_cs[3], float out[6]);
/* the step count of DepthRayMarch::march for a clipped ray (start, end) in a W x H frame */
uint32_t orc_cs_step_count(const float ray[6], uint32_t width, uint32_t height, uint32_t steps);
/* 1 - shadow of pixel (x, y); march_out (may be NULL) receives {step_count, hit step or -1, in contact (0/1)} */
float orc_cs_pixel(const OxcContactShadowCamera* camera, const OxcContactShadowSettings* settings, const float* depth, uint32_t width,
                   uint32_t height, uint32_t x, uint32_t y, int32_t march_out[3]);

/* The pass over a width x height frame, HOST arrays: depth (D32F) -> out (f32, 1 - shadow). */
void orc_contact_shadows(const OxcContactShadowCamera* camera, const OxcContactShadowSettings* settings, const float* depth, uint32_t width,
                         uint32_t height, float* out);

#ifdef __cplusplus
}
#endif
#endif
