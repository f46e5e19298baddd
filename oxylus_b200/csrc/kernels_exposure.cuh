// kernels_exposure.cuh — eye adaptation (PostProcess.cpp:7-77).  The per-pixel bin and the record's update are oxc_exposure.cuh's; this
// file counts and reduces.
//   k_histogram         grid-stride over the pixels at a few CTAs per SM.  Each warp groups its 32 lanes by bin (__match_any_sync)
//                       and one lane per group adds the group's size to the CTA's shared histogram; each CTA then adds its non-zero
//                       bins to the global histogram once.  A uniform frame (every pixel in one bin) costs one shared atomic per warp
//                       per step instead of 32 global ones.  Counts are integers, so the order of the atomics cannot change a bit.
//   k_exposure_average  one CTA of 256 threads, one per bin: weighted = sum of bins[i] * i, added mod 2^32 (any order gives the same
//                       u32), then thread 0 updates the record.
#pragma once
#include "oxc_exposure.cuh"

namespace oxc {

constexpr int HISTOGRAM_THREADS = 256, HISTOGRAM_CTAS_PER_SM = 4;

__global__ void __launch_bounds__(HISTOGRAM_THREADS) k_histogram(const __grid_constant__ EyeAdaptationParams p) {
  __shared__ uint32_t s_bins[HISTOGRAM_BINS];
  for (int i = threadIdx.x; i < HISTOGRAM_BINS; i += HISTOGRAM_THREADS) s_bins[i] = 0;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t stride = (uint64_t)gridDim.x * HISTOGRAM_THREADS;
  // the warp's base index is the same in all its lanes, so every lane runs every step and takes part in the match
  for (uint64_t base = (uint64_t)blockIdx.x * HISTOGRAM_THREADS + (threadIdx.x & ~31u); base < p.pixels; base += stride) {
    const uint64_t i = base + lane;
    const int bin = i < p.pixels ? histogram_bin(p, __ldg(p.frame + i)) : HISTOGRAM_BINS; // HISTOGRAM_BINS: past the frame
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, bin);
    if (bin < HISTOGRAM_BINS && lane == (uint32_t)(__ffs((int)peers) - 1)) atomicAdd(&s_bins[bin], (uint32_t)__popc(peers));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < HISTOGRAM_BINS; i += HISTOGRAM_THREADS)
    if (s_bins[i]) atomicAdd(p.histogram + i, s_bins[i]);
}

__global__ void __launch_bounds__(HISTOGRAM_BINS) k_exposure_average(const __grid_constant__ EyeAdaptationParams p) {
  __shared__ uint32_t s_warp[HISTOGRAM_BINS / 32];
  const uint32_t gid = threadIdx.x;
  uint32_t v = p.histogram[gid] * gid;
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
  if ((gid & 31u) == 0) s_warp[gid >> 5] = v;
  __syncthreads();
  if (gid != 0) return;
  uint32_t weighted = 0;
  for (int w = 0; w < HISTOGRAM_BINS / 32; w++) weighted += s_warp[w];
  *p.record = exposure_update(p, weighted, p.histogram[0], *p.record);
}

} // namespace oxc
