/*
 * oxc_oracle_vsm_draw.h — CPU ORACLE of the VSM shadow raster into the physical atlas (Passes/Shadowmaps.cpp:433-754); the
 * specification of include/oxcull.h oxc_vsm_draw_pages (comment at the top of oxc_oracle_vsm_draw.c).  TEST INFRASTRUCTURE ONLY:
 * only tests/ and tools/ load liboxc_oracle_vsm_draw.so (oracle/pyoracle_vsm_draw.py), which also holds everything of
 * oxc_oracle.h and oxc_oracle_vsm.h.
 */
#ifndef OXC_ORACLE_VSM_DRAW_H_
#define OXC_ORACLE_VSM_DRAW_H_

#include "oxc_oracle_vsm.h"

#ifdef __cplusplus
extern "C" {
#endif

/* survivors: meshlet-instance indices (the HPB cull's list); coarse: the camera the HPB cull ran with (its PV . W is the triangle
 * test); page_tables: clipmap_count x size x size; table may be NULL (no alpha test; images are HOST pointers); atlas: P x P
 * floats updated in place.  Returns the fragments that reached the sink. */
uint64_t orc_vsm_draw_pages(const OrcScene* scene, const OxcMeshletInstance* meshlet_instances, const uint32_t* survivors,
                            uint32_t survivor_count, const OxcCullCamera* coarse, const OxcVsmContext* vsm, const OxcVirtualClipmap* clipmaps,
                            const uint32_t* dirty_flags, const uint32_t* page_tables, const OxcMaterialTable* table, float* atlas);

#ifdef __cplusplus
}
#endif
#endif
