// kernels_pbr_atmosphere.cuh — PBR apply under the atmosphere (RendererInstance::apply_pbr, pbr_apply variant, Passes/PBR.cpp:312-432),
// one launch.  The per-pixel arithmetic is oxc_pbr_atmosphere.cuh's; the layout is k_apply_pbr's.
//   k_apply_pbr_atmosphere  one thread per pixel, an 8 x 4 pixel tile per warp, 32 x 8 pixels per CTA, the lights staged once per CTA in
//                           shared memory with their per-light constants, then summed in index order.  The sky LUTs and the 48 KiB
//                           cube are read through the read-only cache.
#pragma once
#include "kernels_pbr.cuh"
#include "oxc_pbr_atmosphere.cuh"

namespace oxc {

__global__ void __launch_bounds__(PBR_THREADS) k_apply_pbr_atmosphere(const __grid_constant__ PbrAtmParams p) {
  __shared__ PbrLight lights[PBR_MAX_LIGHTS];
  for (uint32_t i = threadIdx.x; i < p.pbr.light_count; i += PBR_THREADS) {
    const float4* r = p.pbr.lights + (size_t)i * 4;
    lights[i] = pbr_stage_light(__ldg(r), __ldg(r + 1), __ldg(r + 2), __ldg(r + 3));
  }
  __syncthreads();
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int x = blockIdx.x * PBR_TILE_X + (int)((warp & 3u) * 8u + (lane & 7u));
  const int y = blockIdx.y * PBR_TILE_Y + (int)((warp >> 2) * 4u + (lane >> 3));
  if (x >= p.pbr.width || y >= p.pbr.height) return;
  p.pbr.out[(size_t)y * p.pbr.width + x] = pbr_atmosphere_pixel(p, lights, x, y);
}

} // namespace oxc
