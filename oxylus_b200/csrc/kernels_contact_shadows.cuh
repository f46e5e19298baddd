// kernels_contact_shadows.cuh — the contact-shadow pass (RendererInstance.cpp:990-1020, passes/contact_shadows.slang), one launch.  The
// per-pixel arithmetic is oxc_contact_shadows.cuh's; this file lays the pixels out.
//   k_contact_shadows  one thread per pixel, an 8 x 4 pixel tile per warp, 32 x 8 pixels per CTA.  The sun direction is the same for
//                      every pixel, so neighbouring rays are parallel and a warp's taps fall on few depth lines.
#pragma once
#include "oxc_contact_shadows.cuh"

namespace oxc {

constexpr int CONTACT_TILE_X = 32, CONTACT_TILE_Y = 8, CONTACT_THREADS = 256;

__global__ void __launch_bounds__(CONTACT_THREADS) k_contact_shadows(const __grid_constant__ ContactShadowParams p) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int x = blockIdx.x * CONTACT_TILE_X + (int)((warp & 3u) * 8u + (lane & 7u));
  const int y = blockIdx.y * CONTACT_TILE_Y + (int)((warp >> 2) * 4u + (lane >> 3));
  if (x >= p.width || y >= p.height) return;
  p.out[(size_t)y * p.width + x] = cs_pixel(p, cs_constants(p), x, y);
}

} // namespace oxc
