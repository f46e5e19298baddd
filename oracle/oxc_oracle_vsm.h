/*
 * oxc_oracle_vsm.h — CPU ORACLE of the VSM page bookkeeping (Passes/Shadowmaps.cpp:100-430), one function per pass; the
 * specification of include/oxcull.h oxc_vsm_* (canonical free list, allocation and dirty list orders).  TEST INFRASTRUCTURE ONLY:
 * only tests/ load liboxc_oracle_vsm.so (oracle/pyoracle_vsm.py), which also holds everything of oxc_oracle.h.
 */
#ifndef OXC_ORACLE_VSM_H_
#define OXC_ORACLE_VSM_H_

#include "oxc_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

void orc_vsm_reset_page_visibility(const OxcVsmContext* vsm, int sun_moved, uint32_t* page_tables);
void orc_vsm_invalidate_pages(const OxcVsmContext* vsm, const OxcVirtualClipmap* clipmaps, const OrcScene* scene,
                              const uint32_t* dirty_mesh_instances, uint32_t dirty_count, const OxcTransformWorld* previous_transforms,
                              uint32_t* page_tables);
void orc_vsm_free_invisible_pages(const OxcVsmContext* vsm, uint32_t* page_tables);
void orc_vsm_build_free_page_list(const uint32_t* page_occupancy, uint32_t physical_page_count, OxcVsmAllocator* allocator,
                                  uint32_t* free_page_list);
void orc_vsm_allocate_pages(const OxcVsmContext* vsm, const int32_t* requests, uint32_t request_capacity, OxcVsmAllocator* allocator,
                            const uint32_t* free_page_list, uint32_t* page_tables);
void orc_vsm_mark_dirty_pages(const OxcVsmContext* vsm, const uint32_t* page_tables, OxcVsmAllocator* allocator, uint32_t* dirty_coords,
                              uint32_t* clipmap_dirty_flags);
void orc_vsm_clear_dirty_pages(const OxcVsmContext* vsm, const OxcVsmAllocator* allocator, const uint32_t* dirty_coords, float* atlas);
/* steps 0-10 of one frame in the order of Shadowmaps.cpp:143-430 around orc_mark_visible_pages and orc_build_hpb */
void orc_vsm_frame(const OxcVsmContext* vsm, const OxcVirtualClipmap* clipmaps, int sun_moved, const OrcScene* scene,
                   const uint32_t* dirty_mesh_instances, uint32_t dirty_count, const OxcTransformWorld* previous_transforms,
                   const float inv_projection_view[16], const float resolution[2], const float* depth, uint32_t* page_tables,
                   uint32_t* page_occupancy, uint32_t physical_page_count, int32_t* requests, uint32_t request_capacity,
                   OxcVsmAllocator* allocator, uint32_t* free_page_list, uint32_t* dirty_coords, uint32_t* clipmap_dirty_flags,
                   uint8_t* hpb, uint32_t hpb_levels, float* atlas);

#ifdef __cplusplus
}
#endif
#endif
