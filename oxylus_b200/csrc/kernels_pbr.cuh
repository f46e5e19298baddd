// kernels_pbr.cuh — PBR apply (RendererInstance::apply_pbr, pbr_apply_no_atmos variant, Passes/PBR.cpp:435-531), one launch.  The
// per-pixel arithmetic is oxc_pbr.cuh's; this file lays the pixels out and stages the lights.
//   k_apply_pbr  one thread per pixel, an 8 x 4 pixel tile per warp, 32 x 8 pixels per CTA.  The CTA first stages every light in
//                shared memory (at most OXC_MAX_LIGHTS x 64 B = 16 KiB) with its per-light constants (normalized spot direction,
//                cone cosines), then each thread sums the lights in index order.
#pragma once
#include "oxc_pbr.cuh"

namespace oxc {

constexpr int PBR_TILE_X = 32, PBR_TILE_Y = 8, PBR_THREADS = 256, PBR_MAX_LIGHTS = 256;

__global__ void __launch_bounds__(PBR_THREADS) k_apply_pbr(const __grid_constant__ PbrParams p) {
  __shared__ PbrLight lights[PBR_MAX_LIGHTS];
  for (uint32_t i = threadIdx.x; i < p.light_count; i += PBR_THREADS) {
    const float4* r = p.lights + (size_t)i * 4;
    lights[i] = pbr_stage_light(__ldg(r), __ldg(r + 1), __ldg(r + 2), __ldg(r + 3));
  }
  __syncthreads();
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int x = blockIdx.x * PBR_TILE_X + (int)((warp & 3u) * 8u + (lane & 7u));
  const int y = blockIdx.y * PBR_TILE_Y + (int)((warp >> 2) * 4u + (lane >> 3));
  if (x >= p.width || y >= p.height) return;
  p.out[(size_t)y * p.width + x] = pbr_pixel(p, lights, x, y);
}

} // namespace oxc
