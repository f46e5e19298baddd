/*
 * oxc_oracle_gbuffer.h — CPU ORACLE of the vis-buffer decode into the G-buffer (passes/visbuffer_decode.slang:88-183 with the material
 * functions of scene.slang:110-159); the specification of include/oxcull.h oxc_decode_gbuffer (comment at the top of
 * oxc_oracle_gbuffer.c).  TEST INFRASTRUCTURE ONLY: only tests/ and tools/ load liboxc_oracle_gbuffer.so (oracle/pyoracle_gbuffer.py),
 * which also holds everything of oxc_oracle.h.  Image texels are HOST pointers here.
 */
#ifndef OXC_ORACLE_GBUFFER_H_
#define OXC_ORACLE_GBUFFER_H_

#include "oxc_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the oracle's own sRGB table: out[c] = (float)EOTF(c / 255) evaluated in binary64 */
void orc_srgb_table(float out[256]);
/* texel fetches (one 32-bit word each on the device) made by the functions below since the last reset; reset != 0 zeroes the count */
uint64_t orc_gbuffer_texel_fetches(int reset);
/* one level of an image with one filter, four channels (spec step 5 conversion) */
void orc_gbuffer_sample_level(const OxcAlphaImage* image, const OxcSamplerDesc* sampler /* NULL: linear, repeat */, uint32_t level,
                              uint32_t filter, float u, float v, float out[4]);
/* SampleGrad (spec step 4) with the sampler's modes */
void orc_gbuffer_sample_grad(const OxcAlphaImage* image, const OxcSamplerDesc* sampler, float u, float v, float ddx_u, float ddx_v,
                             float ddy_u, float ddy_v, float out[4]);
/* the material half for one decoded pixel (spec steps 3-8).  px: ddx[3], ddy[3] (lambda derivatives), the three world positions [9],
 * uv[2], uv_ddx[2], uv_ddy[2] (before the uv transform), the normalized world normal [3] = 24 floats.  want: bit k = plane k.
 * out: albedo, normal, emissive, metallic_roughness_occlusion (16 floats).  Returns 0 (out untouched) when material_index lies
 * outside the table. */
int orc_gbuffer_shade(const OxcMaterialTable* table, uint32_t material_index, const float px[24], const float camera_position[3], uint32_t want,
                      float out[16]);
/* T (out[0..2]) and B (out[3..5]) of the tangent frame (spec step 7) for a pixel record, its uv gradients taken as they are */
void orc_gbuffer_tangent_frame(const float px[24], const float camera_position[3], float out[6]);
/* The geometry half per pixel: records[pix] = the 24-float record orc_gbuffer_shade takes; material[pix] = the mesh instance's
 * material_index, -1 for a discarded pixel, -2 for a vertex index >= vertex_count (records of both are zero). */
void orc_decode_gbuffer_pixels(const OrcScene* scene, const OxcMeshletInstance* meshlet_instances, uint32_t total, const OxcCullCamera* cam,
                               const uint32_t* vis32, uint32_t width, uint32_t height, float* records, int32_t* material);
/* The whole decode over a vis32 image (reference packing, id base 0).  Any plane may be NULL; discarded pixels are not written.
 * Returns the number of decoded pixels whose material_index lies outside the table (the device raises OXC_STATUS_BAD_MATERIAL). */
uint64_t orc_decode_gbuffer(const OrcScene* scene, const OxcMeshletInstance* meshlet_instances, uint32_t total, const OxcCullCamera* cam,
                            const uint32_t* vis32, uint32_t width, uint32_t height, const OxcMaterialTable* table, float* albedo, float* normal,
                            float* emissive, float* metallic_roughness_occlusion);

#ifdef __cplusplus
}
#endif
#endif
