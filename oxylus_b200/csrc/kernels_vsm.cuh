// kernels_vsm.cuh — VSM page bookkeeping between the page marking and the shadow raster (Passes/Shadowmaps.cpp:100-430):
//   k_vsm_begin_frame          clear on sun_moved (:143-148) + rmvsm_reset_page_visibility.slang:16-24 + zero-filled occupancy
//                              (:224-232) and request count, one pass
//   k_vsm_invalidate_pages     rmvsm_invalidate_pages.slang:19-111, one warp per (dirty instance, clipmap, previous/current)
//   k_vsm_allocate             rmvsm_free_invisible_pages, rmvsm_build_free_page_list, rmvsm_allocate_pages and
//                              rmvsm_mark_dirty_pages in one CTA
//   k_vsm_clear_dirty_pages    rmvsm_clear_dirty_pages.slang:12-25 with 128-bit stores, dirty count read on the device
// Specification: oracle/oxc_oracle_vsm.c orc_vsm_* (bit-exact; canonical order of free list, allocation and dirty list).
#pragma once
#include "oxc_exact.cuh"

namespace oxc {

constexpr uint32_t VSM_VISIBLE = 1u, VSM_DIRTY = 2u, VSM_BACKED = 4u, VSM_INVALIDATED = 8u;
constexpr int VSM_MAX_CLIPMAPS = 10;

__global__ void __launch_bounds__(256) k_vsm_begin_frame(uint32_t* __restrict__ page_tables, uint32_t entries, uint32_t* __restrict__ occupancy,
                                                         uint32_t physical_page_count, uint32_t* __restrict__ request_count, int sun_moved) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < entries) page_tables[i] = sun_moved ? 0u : (page_tables[i] & ~(VSM_VISIBLE | VSM_DIRTY | VSM_INVALIDATED));
  if (i < physical_page_count) occupancy[i] = 0u;
  if (i == 0) *request_count = 0u;
}

struct VsmInvalidateParams {
  float clip_pv[VSM_MAX_CLIPMAPS][16]; // projection_view_mat, column-major
  float z_near[VSM_MAX_CLIPMAPS];
  int page_offset[VSM_MAX_CLIPMAPS][2];
  const OxcMeshInstance* mesh_instances;
  const OxcMesh* meshes;
  const OxcTransformWorld* transforms;
  const OxcTransformWorld* previous_transforms;
  const uint32_t* dirty;
  uint32_t dirty_count, mesh_instance_count, mesh_count, transform_count;
  uint32_t* page_tables;
  int size, clipmap_count;
};

// rmvsm.slang:129-138 with com::mod on floats, as k_vsm_mark_visible_pages; false = no page (INVALID_COORDS or outside)
OXC_DI bool vsm_wrap(int v, int offset, int size, int& out) {
  const float fo = (float)(v + offset), fsz = (float)size;
  out = __float2int_rz(fs(fo, fm(fsz, floorf(fd(fo, fsz)))));
  return out >= 0 && out <= size - 1;
}

// Every lane evaluates the (warp-uniform) projection; the lanes then share the page rectangle.  Concurrent warps may store
// Invalidated into the same entry: the value is the same and an invalidated entry is no longer Backed, so the result does not
// depend on their order.
__global__ void __launch_bounds__(256) k_vsm_invalidate_pages(const __grid_constant__ VsmInvalidateParams p) {
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const uint32_t per_instance = (uint32_t)p.clipmap_count * 2u;
  if (warp >= p.dirty_count * per_instance) return;
  const uint32_t d = warp / per_instance, ci = (warp % per_instance) >> 1, current = warp & 1u;
  const uint32_t idx = __ldg(&p.dirty[d]);
  if (idx >= p.mesh_instance_count) return;
  const OxcMeshInstance mi = p.mesh_instances[idx];
  if (mi.transform_index >= p.transform_count || mi.mesh_index >= p.mesh_count) return;
  const OxcMeshBounds b = p.meshes[mi.mesh_index].bounds;
  const float* world_src = (current ? p.transforms : p.previous_transforms)[mi.transform_index].world; // :96,104
  float pv[16], w[16];
#pragma unroll
  for (int k = 0; k < 16; k++) { pv[k] = p.clip_pv[ci][k]; w[k] = world_src[k]; }
  float4 rows[4];
  mul_mm_rows(pv, w, rows);
  ScreenAabb sa;
  if (!project_aabb(rows[0], rows[1], rows[2], rows[3], p.z_near[ci], b.aabb_center[0], b.aabb_center[1], b.aabb_center[2],
                    b.aabb_extent[0], b.aabb_extent[1], b.aabb_extent[2], sa))
    return;                                                                                      // :30
  const float u0 = fminf(fmaxf(sa.minx, 0.0f), 1.0f), v0 = fminf(fmaxf(sa.miny, 0.0f), 1.0f);   // :31-32
  const float u1 = fminf(fmaxf(sa.maxx, 0.0f), 1.0f), v1 = fminf(fmaxf(sa.maxy, 0.0f), 1.0f);
  if (u0 >= u1 || v0 >= v1) return;                                                              // :33-35
  const int size = p.size;
  const float fsz = (float)size;
  const int x0 = min(max(__float2int_rz(floorf(fm(u0, fsz))), 0), size - 1);                    // :37-39
  const int y0 = min(max(__float2int_rz(floorf(fm(v0, fsz))), 0), size - 1);
  const int x1 = min(max(__float2int_rz(ceilf(fm(u1, fsz))) - 1, 0), size - 1);
  const int y1 = min(max(__float2int_rz(ceilf(fm(v1, fsz))) - 1, 0), size - 1);
  const int pw = x1 - x0 + 1, ph = y1 - y0 + 1;
  if (pw <= 0 || ph <= 0) return;
  uint32_t* layer = p.page_tables + (size_t)ci * size * size;
  for (int i = (int)lane; i < pw * ph; i += 32) {                                                // :47-62
    int wx, wy;
    if (!vsm_wrap(x0 + i % pw, p.page_offset[ci][0], size, wx) || !vsm_wrap(y0 + i / pw, p.page_offset[ci][1], size, wy)) continue;
    uint32_t* page = layer + (size_t)wy * size + wx;
    if (*page & VSM_BACKED) *page = VSM_INVALIDATED;
  }
}

constexpr int VSM_ALLOC_THREADS = 1024;
constexpr int VSM_ALLOC_ITEMS = 8; // consecutive entries per thread: a chunk of the table is 8192 entries, 5 chunks at 10 x 64 x 64

struct VsmAllocParams {
  uint32_t* page_tables;
  const uint32_t* occupancy;
  const int* requests;
  OxcVsmAllocator* allocator;
  uint32_t* free_list;
  uint32_t* dirty_coords; // u32x2 per dirty page, `entries` of them; words [entries, 2 * entries) hold the per-entry request counts.
                          // After chunks up to entry E the dirty list fills at most words [0, 2E), below the counts still to be
                          // read (from word entries + E on), so the list never overwrites a count before it is read
  uint32_t* dirty_flags;
  uint32_t entries, physical_page_count, request_capacity, phys_per_row;
  int size, clipmap_count;
};

// exclusive prefix of v over the block in thread order; `total` = block sum.  warp_s: 32 words of shared memory.
OXC_DI uint32_t vsm_block_scan(uint32_t v, uint32_t* warp_s, uint32_t& total) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= (uint32_t)o) x += y;
  }
  if (lane == 31) warp_s[warp] = x;
  __syncthreads();
  if (warp == 0) {
    uint32_t s = lane < VSM_ALLOC_THREADS / 32 ? warp_s[lane] : 0u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= (uint32_t)o) s += y;
    }
    warp_s[lane] = s;
  }
  __syncthreads();
  total = warp_s[VSM_ALLOC_THREADS / 32 - 1];
  const uint32_t prefix = x - v + (warp ? warp_s[warp - 1] : 0u);
  __syncthreads(); // warp_s is reused by the next scan
  return prefix;
}

// One CTA.  The free list, the slot of every entry and the dirty list are prefix sums in address order; in a single block
// they are plain block scans over chunks taken in order, so the result is the canonical one whatever the hardware schedules,
// and no inter-CTA protocol is needed for tables of a few ten thousand entries.
//   A  zero the per-entry request counts
//   B  free list (occupancy == 0, ascending); count the valid requests per entry (atomics: the counts do not depend on order)
//   C  per entry, in address order: free if invisible (rmvsm_free_invisible_pages), allocate (its requests take slots
//      [s, s + c); it gets free_list[min(s + c, free_count) - 1] if s < free_count, else stays unchanged), push if dirty
__global__ void __launch_bounds__(VSM_ALLOC_THREADS, 1) k_vsm_allocate(const __grid_constant__ VsmAllocParams p) {
  __shared__ uint32_t warp_s[32];
  __shared__ uint32_t flags_s[VSM_MAX_CLIPMAPS];
  uint32_t* const counts = p.dirty_coords + p.entries;
  constexpr uint32_t CHUNK = VSM_ALLOC_THREADS * VSM_ALLOC_ITEMS;
  const uint32_t t = threadIdx.x;
  if (t < VSM_MAX_CLIPMAPS) flags_s[t] = 0u;
  for (uint32_t a = t; a < p.entries; a += VSM_ALLOC_THREADS) counts[a] = 0u; // A
  __syncthreads();
  // B
  uint32_t free_count = 0;
  for (uint32_t base = 0; base < p.physical_page_count; base += CHUNK) {
    const uint32_t first = base + t * VSM_ALLOC_ITEMS;
    uint32_t bits = 0, n = 0;
#pragma unroll
    for (int j = 0; j < VSM_ALLOC_ITEMS; j++) {
      const uint32_t q = first + j;
      if (q < p.physical_page_count && __ldg(&p.occupancy[q]) == 0u) { bits |= 1u << j; n++; }
    }
    uint32_t total;
    uint32_t k = free_count + vsm_block_scan(n, warp_s, total);
#pragma unroll
    for (int j = 0; j < VSM_ALLOC_ITEMS; j++)
      if (bits >> j & 1u) p.free_list[k++] = first + j;
    free_count += total;
  }
  const uint32_t active = p.allocator->active_request_count;
  const uint32_t n_req = active < p.request_capacity ? active : p.request_capacity;
  for (uint32_t r = t; r < n_req; r += VSM_ALLOC_THREADS) {
    const int x = p.requests[r * 3 + 0], y = p.requests[r * 3 + 1], l = p.requests[r * 3 + 2];
    if (x < 0 || y < 0 || l < 0 || x >= p.size || y >= p.size || l >= p.clipmap_count) continue;
    atomicAdd(&counts[((uint32_t)l * p.size + (uint32_t)y) * p.size + (uint32_t)x], 1u);
  }
  __syncthreads();
  // C
  const uint32_t per_layer = (uint32_t)p.size * (uint32_t)p.size;
  uint32_t slots = 0, dirty = 0;
  for (uint32_t base = 0; base < p.entries; base += CHUNK) {
    const uint32_t first = base + t * VSM_ALLOC_ITEMS;
    uint32_t e[VSM_ALLOC_ITEMS], c[VSM_ALLOC_ITEMS], orig[VSM_ALLOC_ITEMS];
    uint32_t n = 0;
#pragma unroll
    for (int j = 0; j < VSM_ALLOC_ITEMS; j++) {
      const uint32_t a = first + j;
      e[j] = orig[j] = 0u; c[j] = 0u;
      if (a < p.entries) {
        e[j] = orig[j] = p.page_tables[a];
        c[j] = counts[a];
        if (!(e[j] & VSM_VISIBLE) && (e[j] & VSM_BACKED)) e[j] &= ~VSM_BACKED; // rmvsm_free_invisible_pages.slang:21-24
      }
      n += c[j];
    }
    uint32_t total;
    uint32_t s = slots + vsm_block_scan(n, warp_s, total);
    uint32_t nd = 0;
#pragma unroll
    for (int j = 0; j < VSM_ALLOC_ITEMS; j++) {
      if (c[j]) {
        if (s < free_count) {                                                        // rmvsm_allocate_pages.slang:32-42
          const uint32_t slot = (s + c[j] < free_count ? s + c[j] : free_count) - 1u;
          e[j] = (e[j] & 0xFFFFu) | ((p.free_list[slot] & 0xFFFFu) << 16) | VSM_DIRTY | VSM_BACKED;
        }
        s += c[j];
      }
      nd += (e[j] & VSM_BACKED) && (e[j] & VSM_DIRTY);
    }
    slots += total;
    uint32_t k = dirty + vsm_block_scan(nd, warp_s, total);
#pragma unroll
    for (int j = 0; j < VSM_ALLOC_ITEMS; j++) {
      const uint32_t a = first + j;
      if (a >= p.entries) break;
      if (e[j] != orig[j]) p.page_tables[a] = e[j];
      if ((e[j] & VSM_BACKED) && (e[j] & VSM_DIRTY)) {                               // rmvsm_mark_dirty_pages.slang:24-29
        const uint32_t phys = e[j] >> 16;
        reinterpret_cast<uint2*>(p.dirty_coords)[k++] = make_uint2(phys % p.phys_per_row, phys / p.phys_per_row);
        flags_s[a / per_layer] = 1u;
      }
    }
    dirty += total;
  }
  __syncthreads();
  if (t < (uint32_t)p.clipmap_count) p.dirty_flags[t] = flags_s[t];
  if (t == 0) {
    OxcVsmAllocator* al = p.allocator;
    al->dirty_physical_page_count = dirty;
    al->free_page_count = free_count;
    al->alloc_cursor = slots;
    al->requests = const_cast<int32_t*>(p.requests);
    al->dirty_physical_page_coords = p.dirty_coords;
    al->free_page_list = p.free_list;
  }
}

struct VsmClearParams {
  const OxcVsmAllocator* allocator;
  const uint2* dirty_coords;
  float* atlas;
  uint32_t page_size, atlas_size, phys_per_row;
  int row_shift; // log2(page_size / 4) when page_size / 4 is a power of two and the atlas is 16-byte aligned, -1 otherwise
  int vec4;      // page_size % 4 == 0 and the atlas 16-byte aligned: 128-bit stores
};

// One CTA per dirty page at a time (grid-stride over the device-side count): a page row is page_size / 4 float4 stores.
__global__ void __launch_bounds__(256) k_vsm_clear_dirty_pages(const __grid_constant__ VsmClearParams p) {
  const uint32_t count = p.allocator->dirty_physical_page_count;
  const uint32_t ps = p.page_size;
  for (uint32_t k = blockIdx.x; k < count; k += gridDim.x) {
    const uint2 pc = p.dirty_coords[k];
    if (pc.x >= p.phys_per_row || pc.y >= p.phys_per_row) continue; // an out-of-bounds image store is discarded
    float* page = p.atlas + (size_t)pc.y * ps * p.atlas_size + (size_t)pc.x * ps;
    if (p.vec4) {
      const uint32_t q = ps >> 2, n = ps * q;
      const float4 one = make_float4(1.0f, 1.0f, 1.0f, 1.0f);
      if (p.row_shift >= 0) {
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x)
          reinterpret_cast<float4*>(page + (size_t)(i >> p.row_shift) * p.atlas_size)[i & (q - 1)] = one;
      } else {
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x)
          reinterpret_cast<float4*>(page + (size_t)(i / q) * p.atlas_size)[i % q] = one;
      }
    } else {
      for (uint32_t i = threadIdx.x; i < ps * ps; i += blockDim.x) page[(size_t)(i / ps) * p.atlas_size + i % ps] = 1.0f;
    }
  }
}

} // namespace oxc
