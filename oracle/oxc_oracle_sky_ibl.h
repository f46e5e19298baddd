/*
 * oxc_oracle_sky_ibl.h — CPU ORACLE of the sky IBL cube (passes/sky_ibl.slang with sky.slang's get_atmosphere_illuminance_along_ray);
 * the specification of include/oxcull.h oxc_atmosphere_sky_ibl.  TEST INFRASTRUCTURE ONLY: only tests/ and tools/ load
 * liboxc_oracle_sky_ibl.so (oracle/pyoracle_sky_ibl.py), which also holds everything of oxc_oracle_atmosphere.h.
 */
#ifndef OXC_ORACLE_SKY_IBL_H_
#define OXC_ORACLE_SKY_IBL_H_

#include "oxc_oracle_atmosphere.h"

#ifdef __cplusplus
extern "C" {
#endif

/* canonical_atan2 of oxc_exact.cuh, and its bulk form for the error checks */
float orc_atan2_canonical(float y, float x);
void orc_atan2_canonical_array(const float* y, const float* x, float* out, uint64_t n);
/* the tap rule of orc_atm_tap, all four channels */
void orc_sky_ibl_tap4(const uint16_t* lut, uint32_t width, uint32_t height, float u, float v, float out[4]);
/* the direction of texel (x, y) of a face; radical_inverse_vdc; interleaved_gradient_noise; the local cosine-hemisphere sample i */
void orc_sky_ibl_dir(uint32_t face, uint32_t x, uint32_t y, float out[3]);
float orc_sky_ibl_radical_inverse(uint32_t bits);
float orc_sky_ibl_ign(float px, float py);
void orc_sky_ibl_local_sample(uint32_t i, float rotation, float out[3]);
/* get_atmosphere_illuminance_along_ray(sun, get_eye_pos((0, camera_y, 0)), eye_dir) over a sky-view LUT at the record's size */
void orc_sky_ibl_illuminance(const OxcAtmosphere* atmosphere, float camera_y, const float sun[3], const uint16_t* sky_view,
                             const float eye_dir[3], float out[3]);
/* the pass: cube (6 x 32 x 32 binary16 RGBA, HOST) read and written in place */
void orc_atmosphere_sky_ibl(const OxcAtmosphere* atmosphere, const OxcPbrCamera* camera, const float sun_direction[3], float sun_intensity,
                            float sun_ambient_strength, uint32_t frame_index, const uint16_t* transmittance, const uint16_t* sky_view,
                            uint16_t* cube);

#ifdef __cplusplus
}
#endif
#endif
