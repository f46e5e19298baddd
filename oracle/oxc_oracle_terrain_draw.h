/*
 * oxc_oracle_terrain_draw.h — CPU ORACLE of the terrain's vis-buffer draw (passes/terrain_visbuffer.slang); the specification of
 * include/oxcull.h oxc_draw_terrain (items 1-7).  TEST INFRASTRUCTURE ONLY: only tests/ and tools/ load liboxc_oracle_terrain_draw.so
 * (oracle/pyoracle_terrain_draw.py).
 */
#ifndef OXC_ORACLE_TERRAIN_DRAW_H_
#define OXC_ORACLE_TERRAIN_DRAW_H_

#include <stdint.h>

#include "../include/oxcull.h"

#ifdef __cplusplus
extern "C" {
#endif

/* item 1: projection_scale = (resolution_y * 0.5) / tan(radians(fov) * 0.5) through the canonical sin / cos */
float orc_terrain_projection_scale(float fov_degrees, float resolution_y);
/* item 2: the pin to [1, 63] (NaN -> 1) and the odd rounding */
float orc_terrain_factor_clamp(float f);
int32_t orc_terrain_round_odd(float f);
/* item 3: the n + 1 points of an edge of pinned factor f rounded to n */
void orc_terrain_edge_points(float f, int32_t n, float* out);

typedef struct OrcTerrainPatch {
  float corner[4][3];              /* p0..p3 (x, height, z) */
  float factor[6];                 /* edge_tessellation of u0, v0, u1, v1, then inner[0], inner[1] (before the pin) */
  float pinned[6];                 /* after the pin and the 1 + 2^-23 rule */
  int32_t n[6];                    /* rounded */
  uint32_t triangles;
} OrcTerrainPatch;

/* items 1-2 for one patch */
void orc_terrain_patch(const uint16_t* heightmap, uint32_t res_x, uint32_t res_y, const OxcTerrainDrawSettings* s,
                       const OxcCullCamera* cam, uint32_t patch_index, OrcTerrainPatch* out);
/* item 3: the patch's triangles as domain (u, v) triples in the order the raster receives them (item 6); tris holds capacity x 6
 * floats.  Returns the triangle count. */
uint32_t orc_terrain_patch_domain(const OrcTerrainPatch* p, float* tris, uint32_t capacity);
/* the whole pass into vis (width x height packed words); prim_bits 8 or 6.  Returns the triangles emitted (before any culling). */
uint64_t orc_draw_terrain(const uint16_t* heightmap, uint32_t res_x, uint32_t res_y, const OxcTerrainDrawSettings* s,
                          const uint32_t* visible_patches, uint32_t instance_count, const OxcCullCamera* cam, uint32_t prim_bits,
                          uint32_t width, uint32_t height, uint64_t* vis);

#ifdef __cplusplus
}
#endif
#endif
