/*
 * oxc_oracle_post.h — CPU ORACLE of eye adaptation and bloom (passes/histogram_*.slang, passes/bloom_*.slang); the specification of
 * include/oxcull.h oxc_eye_adaptation and oxc_bloom.  TEST INFRASTRUCTURE ONLY: only tests/ and tools/ load liboxc_oracle_post.so
 * (oracle/pyoracle_post.py), which also holds everything of oxc_oracle_atmosphere.h.  Frames and levels are float4 per texel, row-major.
 */
#ifndef OXC_ORACLE_POST_H_
#define OXC_ORACLE_POST_H_

#include "oxc_oracle_atmosphere.h"

#ifdef __cplusplus
extern "C" {
#endif

/* item 1: pixel_count, exposure_range, time_coeff, bias_scale */
void orc_eye_adaptation_constants(const OxcEyeAdaptationSettings* s, uint32_t width, uint32_t height, float delta_time, float out[4]);
/* item 2: the bin of one pixel */
uint32_t orc_histogram_bin(const OxcEyeAdaptationSettings* s, float r, float g, float b);
/* item 3: the record after one frame from the finished bins and the item-1 constants */
void orc_histogram_average(const uint32_t bins[256], const float constants[4], float min_exposure, OxcExposure* record);
/* the pass: histogram receives the bins, record is read and written in place */
void orc_eye_adaptation(const float* frame, uint32_t width, uint32_t height, const OxcEyeAdaptationSettings* settings, float delta_time,
                        OxcExposure* record, uint32_t histogram[256]);

/* n of a width x height frame, the bit length of max(width / 2, height / 2) */
uint32_t orc_bloom_level_count(uint32_t width, uint32_t height);
/* item 1: the tap of a W x H float4 plane, border (transparent black) or clamp to edge */
void orc_bloom_tap(const float* src, uint32_t W, uint32_t H, float u, float v, int border, float out[3]);
/* the pass: both chains (oxc_bloom_chain_texels float4 each) written; upsampled level n-1 is left as it was (except n = 1) */
void orc_bloom(const float* frame, uint32_t width, uint32_t height, const OxcBloomSettings* settings, const OxcExposure* record,
               float* downsampled, float* upsampled);

#ifdef __cplusplus
}
#endif
#endif
