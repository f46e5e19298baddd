// bloom_per_level.cu — bloom with every level as its own launch, the comparison point of oxc_bloom's fused single-CTA tail: the
// prefilter, one launch per downsample level and one per upsample level, as the reference dispatches them (n = 1: one launch of the
// black).  The texel functions are oxc_bloom.cuh's, so the bits equal the library's.  tools/bench_post.py compiles it into a temporary
// directory with the library's flags and loads it through ctypes; the library does not contain it.
#include "../../oxylus_b200/csrc/kernels_bloom.cuh"

namespace {
__global__ void __launch_bounds__(oxc::BLOOM_THREADS) k_bloom_black(const __grid_constant__ oxc::BloomParams p) {
  const int x = blockIdx.x * oxc::BLOOM_TILE + (int)(threadIdx.x % oxc::BLOOM_TILE);
  const int y = blockIdx.y * oxc::BLOOM_TILE + (int)(threadIdx.x / oxc::BLOOM_TILE);
  if (x < p.w[0] && y < p.h[0]) oxc::bloom_black_texel(p, x, y);
}
} // namespace

// oxc_bloom's arguments, without its checks; returns the last launch's cudaError_t
extern "C" int bloom_per_level(const float* frame_dev, uint32_t width, uint32_t height, const OxcBloomSettings* settings,
                               const OxcExposure* exposure_dev, const OxcBloomTargets* targets, void* stream) {
  using namespace oxc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const BloomParams p = bloom_make_params(frame_dev, width, height, *settings, exposure_dev, *targets);
  k_bloom_prefilter<<<bloom_grid(p, 0), BLOOM_THREADS, 0, s>>>(p);
  for (int i = 1; i < p.levels; i++) k_bloom_downsample<<<bloom_grid(p, i), BLOOM_THREADS, 0, s>>>(p, i);
  for (int i = p.levels - 1; i >= 1; i--) k_bloom_upsample<<<bloom_grid(p, i - 1), BLOOM_THREADS, 0, s>>>(p, i);
  if (p.levels == 1) k_bloom_black<<<bloom_grid(p, 0), BLOOM_THREADS, 0, s>>>(p);
  return (int)cudaGetLastError();
}
