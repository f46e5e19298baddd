/*
 * oxc_oracle_atmosphere.h — CPU ORACLE of the atmosphere's lookup tables (passes/sky_transmittance.slang, sky_view.slang,
 * sky_aerial_perspective.slang with sky.slang); the specification of include/oxcull.h oxc_atmosphere_transmittance /
 * oxc_atmosphere_sky_luts (comment at the top of oxc_oracle_atmosphere.c).  TEST INFRASTRUCTURE ONLY: only tests/ and tools/ load
 * liboxc_oracle_atmosphere.so (oracle/pyoracle_atmosphere.py), which also holds everything of oxc_oracle_gtao.h.
 */
#ifndef OXC_ORACLE_ATMOSPHERE_H_
#define OXC_ORACLE_ATMOSPHERE_H_

#include "oxc_oracle_gtao.h"

#ifdef __cplusplus
extern "C" {
#endif

/* canonical_exp / canonical_acos of oxc_exact.cuh, and their bulk forms for the error checks */
float orc_exp_canonical(float x);
void orc_exp_canonical_array(const float* x, float* out, uint64_t n);
float orc_acos_canonical(float x);
void orc_acos_canonical_array(const float* x, float* out, uint64_t n);
/* binary16 bits of a stored channel (NaN -> 0x7FFF) */
uint16_t orc_atm_half(float f);
/* ray_sphere_intersect_nearest: 1 and *t, or 0 for `none` (*t untouched) */
int orc_atm_ray_sphere_nearest(const float origin[3], const float dir[3], float radius, float* t);
/* transmittance_params_to_lut_uv(atmos_radius, planet_radius, (h, cos_theta)) */
void orc_atm_transmittance_uv(float atmos_radius, float planet_radius, float h, float cos_theta, float out[2]);
float orc_atm_rayleigh_phase(float cos_theta);
/* henyey_greenstein_draine_phase's g_hg, g_d, alpha, w_d of asymmetry g, and the phase itself */
void orc_atm_hg_draine_constants(float g, float out[4]);
float orc_atm_mie_phase(float g, float cos_theta);
/* MediumScattering(atmosphere, altitude).extinction_sum */
void orc_atm_medium_extinction(const OxcAtmosphere* atmosphere, float altitude, float out[3]);
/* SampleLevel(linear_clamp, (u, v), 0).rgb of a W x H binary16 RGBA LUT */
void orc_atm_tap(const uint16_t* lut, uint32_t width, uint32_t height, float u, float v, float out[3]);
/* get_eye_pos(position).y; uv_to_sky_view_lut_params(uv, altitude) */
float orc_atm_eye_y(const OxcAtmosphere* atmosphere, float camera_y);
void orc_atm_sky_view_dir(const OxcAtmosphere* atmosphere, float u, float v, float altitude, float out[3]);

/* the bake's (height, cos theta) of texel (x, y), and exp(-optical_depth) of its 1000-step march from there */
void orc_atm_transmittance_params(const OxcAtmosphere* atmosphere, uint32_t x, uint32_t y, float out[2]);
void orc_atm_transmittance_ray(const OxcAtmosphere* atmosphere, float height, float cos_theta, float out[3]);

/* The three passes, HOST planes of binary16 RGBA texels at the record's sizes (x fastest, then y, then z). */
void orc_atmosphere_transmittance(const OxcAtmosphere* atmosphere, uint16_t* lut);
void orc_atmosphere_sky_view(const OxcAtmosphere* atmosphere, const OxcPbrCamera* camera, const float sun_direction[3], float sun_intensity,
                             const uint16_t* transmittance, uint16_t* out);
void orc_atmosphere_aerial_perspective(const OxcAtmosphere* atmosphere, const OxcPbrCamera* camera, const float sun_direction[3],
                                       float sun_intensity, const uint16_t* transmittance, uint16_t* out);

#ifdef __cplusplus
}
#endif
#endif
