// kernels_terrain.cuh — the terrain's vis-buffer draw (oxc_draw_terrain).  The per-patch and per-triangle arithmetic is oxc_terrain.cuh's;
// this file schedules it.
//   k_draw_terrain  one CTA per patch slot at a time (grid-stride over the slots; the instance count is read on the device, so the call
//                   needs no read-back).  Thread 0 sets the patch up in shared memory; then each thread takes every 256th triangle of
//                   the patch, forms its three clip positions and sets it up.  A triangle whose pixel box holds at most
//                   TERRAIN_SMALL_PIXELS pixels is drawn by its own thread.  Larger ones (near the camera, and pieces of the clip path)
//                   gather in the patch around the camera, so they go to the meshlet raster's chunk queue (kernels_tri.cuh big_push)
//                   and k_raster_big, launched after this kernel, spreads their 64 x 32-pixel chunks over every warp of the GPU; a
//                   triangle the full queue cannot take is drawn by its thread.
#pragma once
#include "kernels_tri.cuh"
#include "oxc_terrain.cuh"

namespace oxc {

constexpr int TERRAIN_THREADS = 256, TERRAIN_SMALL_PIXELS = 512;

OXC_DI void terrain_raster(const TerrainDrawParams& p, const TriParams& chunks, const TriSetup& s) {
  if ((s.px1 - s.px0 + 1) * (s.py1 - s.py0 + 1) > TERRAIN_SMALL_PIXELS && big_push(chunks, s, p.data)) return;
  raster_small(s, p.data, p.vis, p.width);
}

__global__ void __launch_bounds__(TERRAIN_THREADS) k_draw_terrain(const __grid_constant__ TerrainDrawParams p, uint4* big_queue,
                                                                  uint32_t* big_counters, uint32_t big_capacity) {
  __shared__ TerrainPatch patch;
  TriParams chunks; // big_push reads only the queue's three fields
  chunks.big_queue = big_queue;
  chunks.big_counters = big_counters;
  chunks.big_capacity = big_capacity;
  const uint32_t n = p.draw_cmd->instance_count, count = n < p.patch_total ? n : p.patch_total; // item 7
  for (uint32_t slot = blockIdx.x; slot < count; slot += gridDim.x) {
    const uint32_t idx = terrain_slot_patch(p, slot, count);
    if (idx >= p.patch_total) continue; // uniform over the CTA
    if (threadIdx.x == 0) terrain_patch_setup(p, idx, patch);
    __syncthreads();
    const TerrainPatch t = patch;
    __syncthreads(); // every thread holds its copy before thread 0 sets up the next patch
    for (uint32_t k = threadIdx.x; k < t.tri_count; k += TERRAIN_THREADS) {
      float2 d[3];
      terrain_triangle_domain(t, k, d);
      const float4 c0 = terrain_clip(p, t, d[0]), c1 = terrain_clip(p, t, d[1]), c2 = terrain_clip(p, t, d[2]);
      TriSetup s;
      const int why = tri_setup(to_screen(c0, p.fW, p.fH), to_screen(c1, p.fW, p.fH), to_screen(c2, p.fW, p.fH), p.width, p.height, s);
      if (why == TRI_DRAW) {
        terrain_raster(p, chunks, s);
      } else if (why == TRI_INVALID_VERTEX) { // item 5: a vertex at w <= 0 or beyond the snap range takes the clip path
        float4 poly[2][12];
        int cur;
        const int m = clip_polygon(c0, c1, c2, poly, cur);
        for (int i = 1; i + 1 < m; i++) {
          TriSetup ps;
          if (tri_setup(to_screen(poly[cur][0], p.fW, p.fH), to_screen(poly[cur][i], p.fW, p.fH), to_screen(poly[cur][i + 1], p.fW, p.fH),
                        p.width, p.height, ps) != TRI_DRAW)
            continue;
          ps.narrow = false; // pieces may be large: 64-bit edge functions
          terrain_raster(p, chunks, ps);
        }
      }
    }
  }
}

} // namespace oxc
