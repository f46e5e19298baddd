// kernels_vsm_resolve.cuh — the VSM shadow resolve (RendererInstance::resolve_shadowmap, Passes/Shadowmaps.cpp:756-822,
// passes/resolve_shadowmaps.slang), one thread per pixel.  The per-pixel arithmetic is oxc_vsm_resolve.cuh's; this file only
// lays the pixels out.  Each warp takes an 8 x 4 pixel tile, so its taps land on few page-table entries and atlas lines; a CTA
// of 8 warps covers 32 x 8 pixels.  The tangent basis depends only on the light direction and is computed once per CTA.
#pragma once
#include "oxc_vsm_resolve.cuh"

namespace oxc {

constexpr int VSM_RESOLVE_TILE_X = 32, VSM_RESOLVE_TILE_Y = 8, VSM_RESOLVE_THREADS = 256;

__global__ void __launch_bounds__(VSM_RESOLVE_THREADS) k_vsm_resolve_shadows(const __grid_constant__ VsmResolveParams p) {
  __shared__ VsmBasis basis;
  if (threadIdx.x == 0) basis = vsm_perpendicular_basis(p.light[0], p.light[1], p.light[2]);
  __syncthreads();
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int x = blockIdx.x * VSM_RESOLVE_TILE_X + (int)((warp & 3u) * 8u + (lane & 7u));
  const int y = blockIdx.y * VSM_RESOLVE_TILE_Y + (int)((warp >> 2) * 4u + (lane >> 3));
  if (x >= p.width || y >= p.height) return;
  bool pcf = false;
  const VsmBasis b = basis;
  p.shadow[(size_t)y * p.width + x] = vsm_resolve_pixel(p, b, x, y, &pcf);
}

} // namespace oxc
