// kernels_sky_ibl.cuh — the sky IBL cube (Passes/PBR.cpp:52-94, passes/sky_ibl.slang).  The per-texel and per-sample arithmetic is
// oxc_sky_ibl.cuh's; this file lays the samples out.
//   k_atmosphere_sky_ibl  one thread per (texel, sample): a CTA of 256 threads holds 4 texels of one face, 64 threads each.  Every thread
//                         forms its texel's frame and rotation (the same function, so the same bits in all 64), evaluates its one sample
//                         and leaves it in shared memory; after the barrier the texel's first thread sums the 64 values in index order
//                         from 0, as the shader's serial loop does, and finishes the texel.  6,144 texels alone would fill about 2 % of
//                         the H100's 270,336 resident thread slots; 393,216 sample threads fill them.
#pragma once
#include "oxc_sky_ibl.cuh"

namespace oxc {

constexpr int SKY_IBL_THREADS = 256;
constexpr int SKY_IBL_TEXELS_PER_CTA = SKY_IBL_THREADS / SKY_IBL_SAMPLES;
constexpr int SKY_IBL_BLOCKS = SKY_IBL_TEXELS / SKY_IBL_TEXELS_PER_CTA;

__global__ void __launch_bounds__(SKY_IBL_THREADS) k_atmosphere_sky_ibl(const __grid_constant__ SkyIblParams p) {
  __shared__ float s_sample[3][SKY_IBL_THREADS];
  const int i = (int)threadIdx.x % SKY_IBL_SAMPLES;
  const int texel = (int)blockIdx.x * SKY_IBL_TEXELS_PER_CTA + (int)threadIdx.x / SKY_IBL_SAMPLES;
  const int face = texel / (SKY_IBL_RES * SKY_IBL_RES), y = texel / SKY_IBL_RES % SKY_IBL_RES, x = texel % SKY_IBL_RES;
  const SkyIblTexel t = sky_ibl_texel(p, face, x, y); // reads the history before the first thread of the texel overwrites it
  const Vec3 s = sky_ibl_sample(p, t, i);
  s_sample[0][threadIdx.x] = s.x;
  s_sample[1][threadIdx.x] = s.y;
  s_sample[2][threadIdx.x] = s.z;
  __syncthreads();
  if (i != 0) return;
  Vec3 sum = vec3(0.0f, 0.0f, 0.0f);
  for (int k = 0; k < SKY_IBL_SAMPLES; k++)
    sum = vadd(sum, vec3(s_sample[0][threadIdx.x + k], s_sample[1][threadIdx.x + k], s_sample[2][threadIdx.x + k]));
  sky_ibl_finish(p, t, face, x, y, sum);
}

} // namespace oxc
