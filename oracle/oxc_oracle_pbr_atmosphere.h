/* oxc_oracle_pbr_atmosphere.h — CPU ORACLE of PBR apply under the atmosphere (oxc_oracle_pbr_atmosphere.c). */
#ifndef OXC_ORACLE_PBR_ATMOSPHERE_H_
#define OXC_ORACLE_PBR_ATMOSPHERE_H_

#include "oxc_oracle_pbr.h"
#include "oxc_oracle_sky_ibl.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the constants the pass reads: draw_sun's radius * PI / 180 and its min_cos, half_slice_depth, near_depth_fade_out: out[4] */
void orc_pbra_constants(float out[4]);
/* draw_sun(dir, sun, 1.0) of one channel for dot(dir, sun) = cos_theta */
float orc_pbra_draw_sun(float cos_theta);
/* the cube's face of direction r with (sc, tc, ma); the texel index (face * 32 + y) * 32 + x of texel (i, j) of face f, i, j in -1..32
 * with exactly one off the face; TextureCube.SampleLevel of the cube at r (rgba) */
int orc_pbra_cube_face(const float r[3], float sc_tc_ma[3]);
uint32_t orc_pbra_cube_remap(uint32_t face, int32_t i, int32_t j);
void orc_pbra_cube_tap(const uint16_t* cube, const float r[3], float out[4]);
/* the aerial-perspective LUT's 3D tap (rgba) and sample_aerial_perspective at tex_coord (u, v) and camera-relative position d */
void orc_pbra_tap3(const OxcAtmosphere* atmosphere, const uint16_t* lut, float u, float v, float w, float out[4]);
void orc_pbra_aerial(const OxcAtmosphere* atmosphere, const uint16_t* lut, float u, float v, const float d[3], float out[4]);
/* the pass over HOST planes; sky planes as OxcPbrSky (HOST pointers) */
void orc_apply_pbr_atmosphere(const OxcPbrCamera* camera, const OxcPbrSettings* settings, const OxcAtmosphere* atmosphere, const OxcLight* lights,
                              const float* depth, const float* albedo, const float* normal, const float* emissive,
                              const float* metallic_roughness_occlusion, const float* ambient_occlusion, const float* shadow,
                              const float* contact_shadow, const OxcPbrSky* sky, uint32_t width, uint32_t height, float* out);

#ifdef __cplusplus
}
#endif
#endif
