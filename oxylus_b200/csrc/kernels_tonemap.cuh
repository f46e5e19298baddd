// kernels_tonemap.cuh — the tonemap pass (PostProcess.cpp:205-247), one launch.  The per-pixel arithmetic is oxc_tonemap.cuh's; this
// file lays the pixels out.
//   k_tonemap<TYPE>  one thread per pixel, an 8 x 4 pixel tile per warp, 32 x 8 pixels per CTA (the other screen passes' layout); one
//                    instantiation per curve (the reference's specialization constant), the exposure, bloom and lens flags are uniform
//                    branches on the kernel parameters.
#pragma once
#include "oxc_tonemap.cuh"

namespace oxc {

constexpr int TONEMAP_TILE_X = 32, TONEMAP_TILE_Y = 8, TONEMAP_THREADS = 256;

template <uint32_t TYPE>
__global__ void __launch_bounds__(TONEMAP_THREADS) k_tonemap(const __grid_constant__ TonemapParams p) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int x = blockIdx.x * TONEMAP_TILE_X + (int)((warp & 3u) * 8u + (lane & 7u));
  const int y = blockIdx.y * TONEMAP_TILE_Y + (int)((warp >> 2) * 4u + (lane >> 3));
  if (x >= p.width || y >= p.height) return;
  p.out[(size_t)y * p.width + x] = tonemap_pixel<TYPE>(p, x, y);
}

} // namespace oxc
