// kernels_fxaa.cuh — the FXAA pass (RendererInstance.cpp:1225-1255), one launch.  The per-pixel arithmetic is oxc_fxaa.cuh's; this file
// lays the pixels out.
//   k_fxaa  one thread per pixel, an 8 x 4 pixel tile per warp, 32 x 8 pixels per CTA (the other screen passes' layout).  The 3 x 3
//           taps and the edge walk read the frame through L1; a warp's edge pixels walk while its flat ones have returned.
#pragma once
#include "oxc_fxaa.cuh"

namespace oxc {

constexpr int FXAA_TILE_X = 32, FXAA_TILE_Y = 8, FXAA_THREADS = 256;

__global__ void __launch_bounds__(FXAA_THREADS) k_fxaa(const __grid_constant__ FxaaParams p) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int x = blockIdx.x * FXAA_TILE_X + (int)((warp & 3u) * 8u + (lane & 7u));
  const int y = blockIdx.y * FXAA_TILE_Y + (int)((warp >> 2) * 4u + (lane >> 3));
  if (x >= p.width || y >= p.height) return;
  int taps;
  p.out[(size_t)y * p.width + x] = fxaa_pixel(p, x, y, taps);
}

} // namespace oxc
