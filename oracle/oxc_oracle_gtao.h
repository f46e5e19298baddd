/*
 * oxc_oracle_gtao.h — CPU ORACLE of the visibility-bitmask GTAO (RendererInstance::generate_ambient_occlusion, Passes/PBR.cpp:143-311,
 * passes/gtao/vbgtao_*.slang); the specification of include/oxcull.h oxc_generate_ambient_occlusion (comment at the top of
 * oxc_oracle_gtao.c).  TEST INFRASTRUCTURE ONLY: only tests/ and tools/ load liboxc_oracle_gtao.so (oracle/pyoracle_gtao.py), which
 * also holds everything of oxc_oracle_vsm_resolve.h.
 */
#ifndef OXC_ORACLE_GTAO_H_
#define OXC_ORACLE_GTAO_H_

#include "oxc_oracle_vsm_resolve.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the library's pow of binary32 arguments (oxc_exact.cuh canonical_pow) */
float orc_pow_canonical(float x, float y);
/* the reference's Hilbert index of (x, y) in the 64 x 64 table (RendererInstance.cpp:151-170) */
uint32_t orc_gtao_hilbert_index(uint32_t x, uint32_t y);
/* load_noise of pixel (x, y) */
void orc_gtao_noise(uint32_t x, uint32_t y, uint32_t noise_index, float out[2]);
float orc_gtao_fast_acos(float x);
uint32_t orc_gtao_update_sectors(float min_horizon, float max_horizon, uint32_t bitmask);
uint32_t orc_gtao_calc_sector_mask(float thickness, const float delta[3], const float view_dir[3], float sampling_direction, float n);
float orc_gtao_linearize(const float projection[16], float device_depth);
float orc_gtao_weighted_average(float d0, float d1, float d2, float d3);
/* byte offset / 4 of level k in the packed mip chain of a W x H frame, k = 0..5 (5 = total texel count) */
uint64_t orc_gtao_mip_offset(uint32_t width, uint32_t height, uint32_t level);
/* SampleLevel(linear_clamp, (u, v), lambda) of a packed W x H mip chain */
float orc_gtao_sample_level(const float* mips, uint32_t width, uint32_t height, float u, float v, float lambda);
/* the denoise of pixel (x, y) from a W x H noisy plane (binary16 bits) and edges plane */
float orc_gtao_denoise_pixel(const uint16_t* noisy, const uint32_t* edges, uint32_t width, uint32_t height, uint32_t x, uint32_t y,
                             float final_power);

/* The three passes over a width x height frame, all HOST arrays: depth (D32F), normals (float4 per pixel, oct in .zw).  Outputs: mips
 * (orc_gtao_mip_offset(W, H, 5) floats), edges, noisy (binary16 bits), ao; each W x H. */
void orc_generate_ambient_occlusion(const OxcGtaoCamera* camera, const OxcGtaoSettings* settings, const float* depth, const float* normals,
                                    uint32_t width, uint32_t height, float* mips, uint32_t* edges, uint16_t* noisy, float* ao);

#ifdef __cplusplus
}
#endif
#endif
