/*
 * oxc_oracle_vsm_resolve.h — CPU ORACLE of the VSM shadow resolve (RendererInstance::resolve_shadowmap, Passes/Shadowmaps.cpp:756-822,
 * passes/resolve_shadowmaps.slang); the specification of include/oxcull.h oxc_vsm_resolve_shadows (comment at the top of
 * oxc_oracle_vsm_resolve.c).  TEST INFRASTRUCTURE ONLY: only tests/ and tools/ load liboxc_oracle_vsm_resolve.so
 * (oracle/pyoracle_vsm_resolve.py), which also holds everything of oxc_oracle.h and oxc_oracle_vsm.h.
 */
#ifndef OXC_ORACLE_VSM_RESOLVE_H_
#define OXC_ORACLE_VSM_RESOLVE_H_

#include "oxc_oracle_vsm.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the library's sin / cos of a binary32 argument (oxc_exact.cuh canonical_sincos) */
void orc_sincos_canonical(float x, float* s, float* c);
/* max |error| of orc_sincos_canonical against libm's binary64 sin / cos over the binary32 values with bits lo, lo + stride, ... <= hi
 * (scan) or over n given values (list): out[0] / out[1] = max absolute error of sin / cos, out[2] / out[3] = max error in ulps of
 * the binary32 result */
void orc_sincos_error_scan(uint32_t lo_bits, uint32_t hi_bits, uint32_t stride, double out[4]);
void orc_sincos_error_list(const float* x, uint64_t n, double out[4]);
/* com::hammersley2d(i, n) */
void orc_hammersley2d(uint32_t i, uint32_t n, float out[2]);
/* hash2 of the pixel position (px, py) */
void orc_vsm_hash2(float px, float py, float out[2]);
/* perpendicular_basis(L): out = tangent.xyz, bitangent.xyz */
void orc_vsm_perpendicular_basis(const float light[3], float out[6]);
/* base_bias of pcss_shadow for a clipmap index, flat normal and the context's light / texel length */
float orc_vsm_base_bias(const OxcVsmContext* vsm, int32_t clipmap_index, const float normal[3]);
/* binary32 -> binary16 (round to nearest even) -> binary32 */
float orc_round_to_half(float f);

/* The resolve over depth_extent[0] x depth_extent[1] pixels: depth (D32F), normals (float4 per pixel, oct in .zw), page_tables
 * [clipmap][size][size], atlas (P x P), all HOST arrays; shadow receives one float per pixel.  pcf (may be NULL) receives 1 for each
 * pixel that ran the PCF loop, 0 otherwise.  Returns the number of such pixels. */
uint64_t orc_vsm_resolve_shadows(const OxcVsmContext* vsm, const float inv_projection_view[16], const float resolution[2],
                                 const OxcVirtualClipmap* clipmaps, const float* depth, const float* normals, const uint32_t* page_tables,
                                 const float* atlas, float* shadow, uint8_t* pcf);

#ifdef __cplusplus
}
#endif
#endif
