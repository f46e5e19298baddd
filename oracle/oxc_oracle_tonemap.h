/*
 * oxc_oracle_tonemap.h — CPU ORACLE of the tonemap pass (passes/tonemap.slang fs_main, passes/lens.slang); the specification of
 * include/oxcull.h oxc_tonemap.  TEST INFRASTRUCTURE ONLY: only tests/ and tools/ load liboxc_oracle_tonemap.so
 * (oracle/pyoracle_tonemap.py), which also holds everything of oxc_oracle_post.h.  Planes are float4 per texel, row-major.
 */
#ifndef OXC_ORACLE_TONEMAP_H_
#define OXC_ORACLE_TONEMAP_H_

#include "oxc_oracle_post.h"

#ifdef __cplusplus
extern "C" {
#endif

/* item 9: the constants of the curves and the lens that do not depend on the call, in this order (ORC_TM_* indices) */
enum {
  ORC_TM_AGX = 0,            /* 9: sRGB_to_adjusted, row-major */
  ORC_TM_AGX_INV = 9,        /* 9: inverse(sRGB_to_adjusted), row-major */
  ORC_TM_AGX_S = 18,         /* AGX_PEAK * AGX_LINEAR */
  ORC_TM_AGX_C = 19,         /* peak / (peak - S) */
  ORC_TM_AGX_PEAK_S = 20,    /* peak - S */
  ORC_TM_GT7_KA = 21,
  ORC_TM_GT7_KB = 22,
  ORC_TM_GT7_KC = 23,
  ORC_TM_GT7_LINEAR_PEAK = 24, /* linearSection_ * peakIntensity_ */
  ORC_TM_GT7_TARGET = 25,      /* framebufferLuminanceTarget_ */
  ORC_TM_GT7_TARGET_UCS = 26,  /* framebufferLuminanceTargetUcs_ */
  ORC_TM_GT7_SDR = 27,         /* sdrCorrectionFactor_ */
  ORC_TM_GT7_ONE_MINUS_BLEND = 28,
  ORC_TM_PQ_INV_M1 = 29,       /* 1 / m1 */
  ORC_TM_PQ_INV_M2 = 30,       /* 1 / m2 */
  ORC_TM_SIMPLEX_F2 = 31,
  ORC_TM_SIMPLEX_G2 = 32,
  ORC_TM_CONSTANTS = 33
};
void orc_tonemap_constants(float out[ORC_TM_CONSTANTS]);
/* item 7: red and green magnitudes of FfxLensGetRGMag */
void orc_tonemap_rg_mag(float amount, float out[2]);
/* item 3: one curve on one colour (OXC_TONEMAP_*), and GT7's Rec.2020 output before rec2020_to_rec709 */
void orc_tonemap_curve(uint32_t type, const float in[3], float out[3]);
void orc_tonemap_gt7_rec2020(const float in[3], float out[3]);
/* item 1: the Repeat tap (rgba) of a W x H float4 plane */
void orc_tonemap_tap(const float* src, uint32_t W, uint32_t H, float u, float v, float out[4]);
/* the pass: out receives width x height float4.  record is read under HasEyeAdaptation, bloom ((width / 2) x (height / 2) float4)
 * under HasBloom */
void orc_tonemap(const float* frame, uint32_t width, uint32_t height, const OxcTonemapSettings* settings, const OxcExposure* record,
                 const float* bloom, float* out);

#ifdef __cplusplus
}
#endif
#endif
