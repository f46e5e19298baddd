// kernels_bloom.cuh — bloom (PostProcess.cpp:79-203).  The per-texel arithmetic is oxc_bloom.cuh's; this file decides which launch
// writes which level.
//   k_bloom_prefilter   downsampled level 0 from the frame, one thread per texel, 16 x 16 texels per CTA.
//   k_bloom_downsample  one level, one launch, for the levels above BLOOM_TAIL_TEXELS texels;
//   k_bloom_upsample    likewise, for the upsample destinations above BLOOM_TAIL_TEXELS texels.
//   k_bloom_tail        one CTA for every level from the first one of at most BLOOM_TAIL_TEXELS texels down to 1 x 1 and back up to
//                       it, with a barrier between levels; the levels pass through global memory (L2-resident) with plain loads.  The
//                       reference's chain is one dependent launch per level (19 at 1080p, 21 at 4K), and below about 32 x 32 a level is
//                       launch latency only.  For a single-level chain it writes item 6's black.
// Every path calls the same texel function, so the bits do not depend on the split (tools/ubench/bloom_per_level.cu runs every level as
// its own launch for comparison).
#pragma once
#include "oxc_bloom.cuh"

namespace oxc {

constexpr int BLOOM_TILE = 16, BLOOM_THREADS = BLOOM_TILE * BLOOM_TILE;
constexpr int BLOOM_TAIL_TEXELS = 1024, BLOOM_TAIL_THREADS = 512;

// the first level the tail runs: the first of at most BLOOM_TAIL_TEXELS texels (the last level, 1 x 1, always qualifies)
inline int bloom_tail_level(const BloomParams& p) {
  int t = 0;
  while ((long long)p.w[t] * p.h[t] > BLOOM_TAIL_TEXELS) t++;
  return t;
}

__global__ void __launch_bounds__(BLOOM_THREADS) k_bloom_prefilter(const __grid_constant__ BloomParams p) {
  const int x = blockIdx.x * BLOOM_TILE + (int)(threadIdx.x % BLOOM_TILE), y = blockIdx.y * BLOOM_TILE + (int)(threadIdx.x / BLOOM_TILE);
  if (x < p.w[0] && y < p.h[0]) bloom_prefilter_texel(p, x, y);
}

__global__ void __launch_bounds__(BLOOM_THREADS) k_bloom_downsample(const __grid_constant__ BloomParams p, int level) {
  const int x = blockIdx.x * BLOOM_TILE + (int)(threadIdx.x % BLOOM_TILE), y = blockIdx.y * BLOOM_TILE + (int)(threadIdx.x / BLOOM_TILE);
  if (x < p.w[level] && y < p.h[level]) bloom_downsample_texel(p, level, x, y);
}

// writes upsampled level `level` - 1
__global__ void __launch_bounds__(BLOOM_THREADS) k_bloom_upsample(const __grid_constant__ BloomParams p, int level) {
  const int x = blockIdx.x * BLOOM_TILE + (int)(threadIdx.x % BLOOM_TILE), y = blockIdx.y * BLOOM_TILE + (int)(threadIdx.x / BLOOM_TILE);
  if (x < p.w[level - 1] && y < p.h[level - 1]) bloom_upsample_texel(p, level, x, y);
}

// downsample levels max(first, 1)..n-1, then the upsample destinations n-2..first; item 6 when n = 1
__global__ void __launch_bounds__(BLOOM_TAIL_THREADS) k_bloom_tail(const __grid_constant__ BloomParams p, int first) {
  for (int i = first > 1 ? first : 1; i < p.levels; i++) {
    for (int t = threadIdx.x; t < p.w[i] * p.h[i]; t += BLOOM_TAIL_THREADS) bloom_downsample_texel(p, i, t % p.w[i], t / p.w[i]);
    __syncthreads();
  }
  for (int i = p.levels - 1; i >= 1 && i - 1 >= first; i--) {
    const int w = p.w[i - 1];
    for (int t = threadIdx.x; t < w * p.h[i - 1]; t += BLOOM_TAIL_THREADS) bloom_upsample_texel(p, i, t % w, t / w);
    __syncthreads();
  }
  if (p.levels == 1)
    for (int t = threadIdx.x; t < p.w[0] * p.h[0]; t += BLOOM_TAIL_THREADS) bloom_black_texel(p, t % p.w[0], t / p.w[0]);
}

inline dim3 bloom_grid(const BloomParams& p, int level) {
  return dim3((unsigned)(p.w[level] + BLOOM_TILE - 1) / BLOOM_TILE, (unsigned)(p.h[level] + BLOOM_TILE - 1) / BLOOM_TILE);
}

} // namespace oxc
