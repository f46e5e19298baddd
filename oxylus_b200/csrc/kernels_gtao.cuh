// kernels_gtao.cuh — the visibility-bitmask GTAO (RendererInstance::generate_ambient_occlusion, Passes/PBR.cpp:143-311), three
// launches in stream order.  The per-pixel arithmetic is oxc_gtao.cuh's; this file lays the pixels out.
//   k_gtao_prefilter  the reference's layout (vbgtao_prefilter.slang): a CTA of 8 x 8 threads covers 16 x 16 pixels, each thread
//                     linearizes a 2 x 2 quad of depth (mip 0) and averages it (mip 1); mips 2..4 are reduced in shared memory.
//                     Threads beyond the extent compute too (their clamped values reach stored texels of small frames) and store
//                     only inside each level's extent.
//   k_gtao_main       edges and the noisy occlusion, one thread per pixel, an 8 x 4 pixel tile per warp, 32 x 8 pixels per CTA.
//   k_gtao_denoise    the 3 x 3 edge-aware denoise and the final power, same layout.
#pragma once
#include "oxc_gtao.cuh"

namespace oxc {

constexpr int GTAO_PREFILTER_SIDE = 8, GTAO_TILE_X = 32, GTAO_TILE_Y = 8, GTAO_THREADS = 256;

__global__ void __launch_bounds__(GTAO_PREFILTER_SIDE * GTAO_PREFILTER_SIDE) k_gtao_prefilter(const __grid_constant__ GtaoParams p) {
  __shared__ float prev[GTAO_PREFILTER_SIDE][GTAO_PREFILTER_SIDE];
  const int lx = threadIdx.x, ly = threadIdx.y;
  const int bx = blockIdx.x * GTAO_PREFILTER_SIDE + lx, by = blockIdx.y * GTAO_PREFILTER_SIDE + ly;
  const int x0 = 2 * bx, y0 = 2 * by;
  const float d00 = gtao_level0(p, x0, y0), d10 = gtao_level0(p, x0 + 1, y0);
  const float d01 = gtao_level0(p, x0, y0 + 1), d11 = gtao_level0(p, x0 + 1, y0 + 1);
  const int W = p.width, H = p.height;
  if (y0 < H) {
    if (x0 < W) p.mips[(size_t)y0 * W + x0] = nan_canonical(d00);
    if (x0 + 1 < W) p.mips[(size_t)y0 * W + x0 + 1] = nan_canonical(d10);
  }
  if (y0 + 1 < H) {
    if (x0 < W) p.mips[(size_t)(y0 + 1) * W + x0] = nan_canonical(d01);
    if (x0 + 1 < W) p.mips[(size_t)(y0 + 1) * W + x0 + 1] = nan_canonical(d11);
  }
  float d = gtao_weighted_average(d00, d10, d01, d11);
  if (bx < p.mip_w[1] && by < p.mip_h[1]) p.mips[p.mip_off[1] + (size_t)by * p.mip_w[1] + bx] = nan_canonical(d);
  prev[lx][ly] = d;
#pragma unroll
  for (int k = 2; k < GTAO_LEVELS; k++) {
    // distance in threads between the level k-1 texels of one quad.  The writers of level k (multiples of 2 * step) are not among
    // the slots this level reads, so one barrier per level orders everything.
    const int step = 1 << (k - 2);
    __syncthreads();
    if ((lx & (2 * step - 1)) == 0 && (ly & (2 * step - 1)) == 0) {
      d = gtao_weighted_average(d, prev[lx + step][ly], prev[lx][ly + step], prev[lx + step][ly + step]);
      const int tx = bx >> (k - 1), ty = by >> (k - 1);
      if (tx < p.mip_w[k] && ty < p.mip_h[k]) p.mips[p.mip_off[k] + (size_t)ty * p.mip_w[k] + tx] = nan_canonical(d);
      prev[lx][ly] = d;
    }
  }
}

OXC_DI bool gtao_pixel(const GtaoParams& p, int& x, int& y) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  x = blockIdx.x * GTAO_TILE_X + (int)((warp & 3u) * 8u + (lane & 7u));
  y = blockIdx.y * GTAO_TILE_Y + (int)((warp >> 2) * 4u + (lane >> 3));
  return x < p.width && y < p.height;
}

__global__ void __launch_bounds__(GTAO_THREADS) k_gtao_main(const __grid_constant__ GtaoParams p) {
  int x, y;
  if (!gtao_pixel(p, x, y)) return;
  float centre;
  const size_t pix = (size_t)y * p.width + x;
  p.edges[pix] = gtao_edges(p, x, y, &centre);
  p.noisy[pix] = half_bits(gtao_occlusion(p, x, y, centre));
}

__global__ void __launch_bounds__(GTAO_THREADS) k_gtao_denoise(const __grid_constant__ GtaoParams p) {
  int x, y;
  if (!gtao_pixel(p, x, y)) return;
  p.ao[(size_t)y * p.width + x] = gtao_denoise(p, x, y);
}

} // namespace oxc
