// kernels_atmosphere.cuh — the atmosphere's lookup tables (RendererInstance.cpp:203-226 bake, Passes/PBR.cpp:11-50 and :96-140 per
// frame).  The per-texel arithmetic is oxc_atmosphere.cuh's; this file lays the texels out.
//   k_atmosphere_transmittance  one thread per texel, row-major, 1000 serial march steps each (an init-time bake: 16.4 M steps at 256 x 64).
//   k_atmosphere_sky_luts       the sky view and the aerial perspective in one launch: CTAs [0, sky_view_blocks) take sky-view texels,
//                               the rest aerial-perspective texels, x fastest, so a warp of the 32-wide aerial perspective shares one
//                               slice and its trip count 2 (z + 1).  Each LUT alone fills under a quarter of the H100's resident
//                               thread slots (59,904 and 32,768 threads of 270,336); side by side they fill a third.
#pragma once
#include "oxc_atmosphere.cuh"

namespace oxc {

constexpr int ATMOSPHERE_THREADS = 256;

__global__ void __launch_bounds__(ATMOSPHERE_THREADS) k_atmosphere_transmittance(const __grid_constant__ AtmosphereParams p) {
  const size_t i = (size_t)blockIdx.x * ATMOSPHERE_THREADS + threadIdx.x;
  if (i >= (size_t)p.t_w * p.t_h) return;
  atm_transmittance_texel(p, (int)(i % (size_t)p.t_w), (int)(i / (size_t)p.t_w));
}

__global__ void __launch_bounds__(ATMOSPHERE_THREADS) k_atmosphere_sky_luts(const __grid_constant__ AtmosphereParams p) {
  if (blockIdx.x < p.sky_view_blocks) {
    const size_t i = (size_t)blockIdx.x * ATMOSPHERE_THREADS + threadIdx.x;
    if (i >= (size_t)p.sv_w * p.sv_h) return;
    atm_sky_view_texel(p, (int)(i % (size_t)p.sv_w), (int)(i / (size_t)p.sv_w));
    return;
  }
  const size_t i = (size_t)(blockIdx.x - p.sky_view_blocks) * ATMOSPHERE_THREADS + threadIdx.x;
  const size_t row = (size_t)p.ap_w * p.ap_h;
  if (i >= row * p.ap_d) return;
  const size_t r = i % row;
  atm_aerial_texel(p, (int)(r % (size_t)p.ap_w), (int)(r / (size_t)p.ap_w), (int)(i / row));
}

} // namespace oxc
