/*
 * oxc_oracle_vsm.c — CPU ORACLE (test infrastructure) of the VSM page bookkeeping: the passes of Passes/Shadowmaps.cpp:100-430
 * between the page marking and the shadow raster.  Same rules as oxc_oracle.c (see oxc_oracle.h): plain C11, canonical binary32
 * arithmetic, every function cites the shader lines it restates (paths relative to /root/reference/Oxylus/src/Render/Shaders
 * unless noted).  Built together with oxc_oracle.c into liboxc_oracle_vsm.so by oracle/pyoracle_vsm.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle.c oxc_oracle_vsm.c
 * The projection and the matrix product are oxc_oracle.c's (orc_project_aabb, orc_mat4_mul); the marking and the HPB build are
 * orc_mark_visible_pages and orc_build_hpb.
 */
#include "oxc_oracle_vsm.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

/* saturating, truncating float -> i32 (PTX cvt.rzi.s32.f32; NaN -> 0), as oxc_oracle.c */
static inline int32_t to_i32_f32(float x) {
  if (x != x) return 0;
  if (x <= -2147483648.0f) return INT32_MIN;
  if (x >= 2147483648.0f) return INT32_MAX;
  return (int32_t)x;
}

/* ------------------------------------------------------------------------------------------------
 * VSM page bookkeeping — the passes of Passes/Shadowmaps.cpp:100-430 around the marking and the HPB build.
 * Page table: layers x size x size u32, rmvsm.slang:16-28 VSMPageState (Visible 1, Dirty 2, Backed 4, Invalidated 8,
 * AllocationFailed 16), physical address in bits 16-31 (:30-34, 95-111).  Where the reference's result depends on the
 * atomics order of the marking or on the wave order of the allocation, these functions commit to one admissible outcome:
 * free list in ascending physical page order, requests ranked by the linear page table address they name.
 * ---------------------------------------------------------------------------------------------- */
#define VSM_VISIBLE 1u
#define VSM_DIRTY 2u
#define VSM_BACKED 4u
#define VSM_INVALIDATED 8u

static size_t vsm_entries(const OxcVsmContext* vsm) {
  return (size_t)vsm->clipmap_count * (size_t)vsm->page_table_size * (size_t)vsm->page_table_size;
}

/* Shadowmaps.cpp:143-148 (sun_moved: vuk::clear_image to 0) + passes/rmvsm_reset_page_visibility.slang:16-24 */
void orc_vsm_reset_page_visibility(const OxcVsmContext* vsm, int sun_moved, uint32_t* page_tables) {
  const size_t n = vsm_entries(vsm);
  for (size_t i = 0; i < n; i++)
    page_tables[i] = sun_moved ? 0u : (page_tables[i] & ~(VSM_VISIBLE | VSM_DIRTY | VSM_INVALIDATED));
}

/* rmvsm.slang:129-138 page_coords_virtual_to_wrapped with com::mod on floats (common/math.slang:99-101), as
 * orc_mark_visible_pages evaluates it; -1 (INVALID_COORDS) and any other coordinate outside the table: no page */
static int vsm_wrap(int32_t v, int32_t offset, int32_t size, int32_t* out) {
  const float fo = (float)(v + offset), fs = (float)size;
  const int32_t w = to_i32_f32(fo - fs * floorf(fo / fs));
  *out = w;
  return w >= 0 && w <= size - 1;
}

/* passes/rmvsm_invalidate_pages.slang:19-64 for one box.  Deviation: every page of the box is visited; the reference
 * visits the pages of 8 x 8 sections with section index < DIRECTIONAL_PAGE_TABLE_SIZE (Shadowmaps.cpp:189), which is the
 * whole table for the reference's size 64 (a multiple of 8, 64 sections) and misses pages for other sizes. */
static void vsm_invalidate_box(const OxcVsmContext* vsm, const OxcVirtualClipmap* clipmap, uint32_t layer, const float mvp[16],
                               const OxcMeshBounds* b, uint32_t* page_tables) {
  OrcScreenAabb sa;
  if (!orc_project_aabb(mvp, clipmap->z_near, b->aabb_center, b->aabb_extent, &sa)) return; /* :30: a failed projection invalidates nothing */
  /* :31-32 clamp(x, 0, 1) = min(max(x, 0), 1) with IEEE maxNum / minNum (a NaN operand yields the other one) */
  const float u0 = fminf(fmaxf(sa.min[0], 0.0f), 1.0f), v0 = fminf(fmaxf(sa.min[1], 0.0f), 1.0f);
  const float u1 = fminf(fmaxf(sa.max[0], 0.0f), 1.0f), v1 = fminf(fmaxf(sa.max[1], 0.0f), 1.0f);
  if (u0 >= u1 || v0 >= v1) return; /* :33-35 */
  const int32_t size = vsm->page_table_size;
  const float fsz = (float)size;
  int32_t x0 = to_i32_f32(floorf(u0 * fsz)), y0 = to_i32_f32(floorf(v0 * fsz));           /* :38 */
  int32_t x1 = to_i32_f32(ceilf(u1 * fsz)) - 1, y1 = to_i32_f32(ceilf(v1 * fsz)) - 1;     /* :39 */
  x0 = x0 < 0 ? 0 : (x0 > size - 1 ? size - 1 : x0); y0 = y0 < 0 ? 0 : (y0 > size - 1 ? size - 1 : y0);
  x1 = x1 < 0 ? 0 : (x1 > size - 1 ? size - 1 : x1); y1 = y1 < 0 ? 0 : (y1 > size - 1 ? size - 1 : y1);
  for (int32_t y = y0; y <= y1; y++)
    for (int32_t x = x0; x <= x1; x++) { /* :47-62 */
      int32_t wx, wy;
      if (!vsm_wrap(x, clipmap->page_offset[0], size, &wx) || !vsm_wrap(y, clipmap->page_offset[1], size, &wy)) continue;
      uint32_t* page = &page_tables[((size_t)layer * size + (size_t)wy) * size + (size_t)wx];
      if (*page & VSM_BACKED) *page = VSM_INVALIDATED; /* reset(), set_invalidated(true) */
    }
}

/* passes/rmvsm_invalidate_pages.slang:66-111 via Shadowmaps.cpp:167-222: per dirty mesh instance and clipmap, the mesh's
 * bounds under the previous (:96-102) and the current (:104-110) world matrix.  A dirty index outside the mesh instance table
 * or an instance whose transform_index is outside the transform table invalidates nothing. */
void orc_vsm_invalidate_pages(const OxcVsmContext* vsm, const OxcVirtualClipmap* clipmaps, const OrcScene* scene,
                              const uint32_t* dirty_mesh_instances, uint32_t dirty_count, const OxcTransformWorld* previous_transforms,
                              uint32_t* page_tables) {
  for (uint32_t d = 0; d < dirty_count; d++) {
    const uint32_t idx = dirty_mesh_instances[d];
    if (idx >= scene->mesh_instance_count) continue;
    const OxcMeshInstance* mi = &scene->mesh_instances[idx];
    if (mi->transform_index >= scene->transform_count || mi->mesh_index >= scene->mesh_count) continue;
    const OxcMeshBounds* b = &scene->meshes[mi->mesh_index].bounds;
    for (int32_t ci = 0; ci < vsm->clipmap_count; ci++) {
      float mvp[16];
      orc_mat4_mul(clipmaps[ci].projection_view_mat, previous_transforms[mi->transform_index].world, mvp);
      vsm_invalidate_box(vsm, &clipmaps[ci], (uint32_t)ci, mvp, b, page_tables);
      orc_mat4_mul(clipmaps[ci].projection_view_mat, scene->transforms[mi->transform_index].world, mvp);
      vsm_invalidate_box(vsm, &clipmaps[ci], (uint32_t)ci, mvp, b, page_tables);
    }
  }
}

/* passes/rmvsm_free_invisible_pages.slang:16-24: !Visible && Backed -> clear Backed (the address bits stay) */
void orc_vsm_free_invisible_pages(const OxcVsmContext* vsm, uint32_t* page_tables) {
  const size_t n = vsm_entries(vsm);
  for (size_t i = 0; i < n; i++)
    if (!(page_tables[i] & VSM_VISIBLE) && (page_tables[i] & VSM_BACKED)) page_tables[i] &= ~VSM_BACKED;
}

/* passes/rmvsm_build_free_page_list.slang:8-30: every physical page with occupancy 0, ascending */
void orc_vsm_build_free_page_list(const uint32_t* page_occupancy, uint32_t physical_page_count, OxcVsmAllocator* allocator,
                                  uint32_t* free_page_list) {
  uint32_t n = 0;
  for (uint32_t p = 0; p < physical_page_count; p++)
    if (page_occupancy[p] == 0u) free_page_list[n++] = p;
  allocator->free_page_count = n;
}

/* passes/rmvsm_allocate_pages.slang:9-43.  Reads the first min(active_request_count, request_capacity) requests; one naming an
 * entry outside the table is skipped (the reference would store out of bounds).  Requests are ranked by the linear address
 * (layer * size + y) * size + x of their entry: d requests for one entry take d consecutive slots, and the entry gets the
 * highest of them below free_page_count (the last store when the waves run in order).  When its first slot is already past
 * the free count, the shader sets AllocationFailed on its local copy and returns without a store (:32-35): the entry is left
 * unchanged.  alloc_cursor = slots handed out = valid requests read. */
void orc_vsm_allocate_pages(const OxcVsmContext* vsm, const int32_t* requests, uint32_t request_capacity, OxcVsmAllocator* allocator,
                            const uint32_t* free_page_list, uint32_t* page_tables) {
  const int32_t size = vsm->page_table_size;
  const size_t n_entries = vsm_entries(vsm);
  uint32_t* count = (uint32_t*)calloc(n_entries ? n_entries : 1, sizeof(uint32_t));
  const uint32_t n = allocator->active_request_count < request_capacity ? allocator->active_request_count : request_capacity;
  for (uint32_t r = 0; r < n; r++) {
    const int32_t x = requests[r * 3 + 0], y = requests[r * 3 + 1], l = requests[r * 3 + 2];
    if (x < 0 || y < 0 || l < 0 || x >= size || y >= size || l >= vsm->clipmap_count) continue;
    count[((size_t)l * size + (size_t)y) * size + (size_t)x]++;
  }
  uint32_t slot0 = 0;
  for (size_t a = 0; a < n_entries; a++) {
    const uint32_t c = count[a];
    if (!c) continue;
    if (slot0 < allocator->free_page_count) {
      const uint32_t slot = (slot0 + c < allocator->free_page_count ? slot0 + c : allocator->free_page_count) - 1u;
      const uint32_t phys = free_page_list[slot];
      page_tables[a] = (page_tables[a] & 0xFFFFu) | ((phys & 0xFFFFu) << 16) | VSM_DIRTY | VSM_BACKED; /* :39-42 */
    }
    slot0 += c;
  }
  allocator->alloc_cursor = slot0;
  free(count);
}

/* passes/rmvsm_mark_dirty_pages.slang:15-30: every Backed && Dirty entry, ascending address, pushes its physical page
 * coordinates (address % n, address / n; n = physical size / page size, rmvsm.slang:99-106); dirty_physical_page_count is the
 * clear dispatch's z; clipmap_dirty_flags[layer] = 1 for a layer with such an entry, 0 otherwise (a zeroed scratch buffer,
 * Shadowmaps.cpp:113-114). */
void orc_vsm_mark_dirty_pages(const OxcVsmContext* vsm, const uint32_t* page_tables, OxcVsmAllocator* allocator, uint32_t* dirty_coords,
                              uint32_t* clipmap_dirty_flags) {
  const size_t per_layer = (size_t)vsm->page_table_size * (size_t)vsm->page_table_size;
  const uint32_t n = (uint32_t)(vsm->physical_page_table_size / vsm->page_size);
  uint32_t k = 0;
  for (int32_t l = 0; l < vsm->clipmap_count; l++) {
    clipmap_dirty_flags[l] = 0u;
    for (size_t i = 0; i < per_layer; i++) {
      const uint32_t e = page_tables[(size_t)l * per_layer + i];
      if ((e & VSM_BACKED) && (e & VSM_DIRTY)) {
        dirty_coords[2 * k] = (e >> 16) % n;
        dirty_coords[2 * k + 1] = (e >> 16) / n;
        k++;
        clipmap_dirty_flags[l] = 1u;
      }
    }
  }
  allocator->dirty_physical_page_count = k;
}

/* passes/rmvsm_clear_dirty_pages.slang:12-25: every texel of each dirty physical page = 1.0 in the R32F atlas (row-major,
 * physical_page_table_size texels square).  A page whose coordinates lie outside the atlas is not written (an out-of-bounds
 * image store is discarded). */
void orc_vsm_clear_dirty_pages(const OxcVsmContext* vsm, const OxcVsmAllocator* allocator, const uint32_t* dirty_coords, float* atlas) {
  const uint32_t ps = (uint32_t)vsm->page_size, as = (uint32_t)vsm->physical_page_table_size, n = as / ps;
  for (uint32_t k = 0; k < allocator->dirty_physical_page_count; k++) {
    const uint32_t px = dirty_coords[2 * k], py = dirty_coords[2 * k + 1];
    if (px >= n || py >= n) continue;
    for (uint32_t y = 0; y < ps; y++)
      for (uint32_t x = 0; x < ps; x++) atlas[(size_t)(py * ps + y) * as + px * ps + x] = 1.0f;
  }
}

/* One VSM frame, Shadowmaps.cpp:143-430 steps in order: clear on sun_moved, reset visibility, invalidate (only without
 * sun_moved and with dirty instances), zero occupancy, mark visible pages, free invisible pages, free list, allocate,
 * HPB, mark dirty pages, clear dirty pages (atlas may be NULL).  allocator->active_request_count is the request counter. */
void orc_vsm_frame(const OxcVsmContext* vsm, const OxcVirtualClipmap* clipmaps, int sun_moved, const OrcScene* scene,
                   const uint32_t* dirty_mesh_instances, uint32_t dirty_count, const OxcTransformWorld* previous_transforms,
                   const float inv_projection_view[16], const float resolution[2], const float* depth, uint32_t* page_tables,
                   uint32_t* page_occupancy, uint32_t physical_page_count, int32_t* requests, uint32_t request_capacity,
                   OxcVsmAllocator* allocator, uint32_t* free_page_list, uint32_t* dirty_coords, uint32_t* clipmap_dirty_flags,
                   uint8_t* hpb, uint32_t hpb_levels, float* atlas) {
  orc_vsm_reset_page_visibility(vsm, sun_moved, page_tables);                                     /* steps 0-1 */
  if (!sun_moved && dirty_count > 0)                                                              /* step 2, :203 */
    orc_vsm_invalidate_pages(vsm, clipmaps, scene, dirty_mesh_instances, dirty_count, previous_transforms, page_tables);
  memset(page_occupancy, 0, (size_t)physical_page_count * sizeof(uint32_t));                      /* step 3 */
  allocator->active_request_count = 0;
  orc_mark_visible_pages(inv_projection_view, resolution, clipmaps, vsm, depth, page_tables, page_occupancy, /* step 4 */
                         &allocator->active_request_count, requests, request_capacity);
  orc_vsm_free_invisible_pages(vsm, page_tables);                                                /* step 5 */
  orc_vsm_build_free_page_list(page_occupancy, physical_page_count, allocator, free_page_list);  /* step 6 */
  orc_vsm_allocate_pages(vsm, requests, request_capacity, allocator, free_page_list, page_tables); /* step 7 */
  orc_build_hpb(page_tables, (uint32_t)vsm->page_table_size, (uint32_t)vsm->clipmap_count, hpb, hpb_levels); /* step 8 */
  orc_vsm_mark_dirty_pages(vsm, page_tables, allocator, dirty_coords, clipmap_dirty_flags);      /* step 9 */
  if (atlas) orc_vsm_clear_dirty_pages(vsm, allocator, dirty_coords, atlas);                      /* step 10 */
}

