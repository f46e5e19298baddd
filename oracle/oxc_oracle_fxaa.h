/*
 * oxc_oracle_fxaa.h — CPU ORACLE of the FXAA pass (passes/fxaa/fxaa.slang fs_main); the specification of include/oxcull.h oxc_fxaa.
 * TEST INFRASTRUCTURE ONLY: only tests/ and tools/ load liboxc_oracle_fxaa.so (oracle/pyoracle_fxaa.py), which also holds everything
 * of oxc_oracle_post.h.  Planes are float4 per texel, row-major.
 */
#ifndef OXC_ORACLE_FXAA_H_
#define OXC_ORACLE_FXAA_H_

#include "oxc_oracle_post.h"

#ifdef __cplusplus
extern "C" {
#endif

/* item 6: EDGE_THRESHOLD_MIN, EDGE_THRESHOLD_MAX, SUBPIXEL_QUALITY, 1.0 / 12.0, formed from the literals in binary32 */
enum { ORC_FXAA_CONSTANTS = 4 };
void orc_fxaa_constants(float out[ORC_FXAA_CONSTANTS]);
/* item 5: QUALITY(i) */
float orc_fxaa_quality(int32_t i);
/* item 3 */
float orc_fxaa_luma(const float rgb[3]);
/* item 2: Sample(uv, int2(dx, dy)) (rgba) of a W x H float4 plane through LinearSamplerClamped; (0, 0) is Sample(uv) */
void orc_fxaa_tap(const float* src, uint32_t W, uint32_t H, float u, float v, int32_t dx, int32_t dy, float out[4]);
/* the pass: out receives width x height float4; taps (may be NULL) receives each pixel's bilinear tap count, 5 on the early exit and
 * 12..32 otherwise */
void orc_fxaa(const float* frame, uint32_t width, uint32_t height, float* out, uint8_t* taps);

#ifdef __cplusplus
}
#endif
#endif
