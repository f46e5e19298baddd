// post_vs_oracle.cpp — HOST run of the eye adaptation's and bloom's device sources (oxylus_b200/csrc/oxc_exposure.cuh, oxc_bloom.cuh),
// for the comparison with the oracle's specification (oracle/oxc_oracle_post.c) that tests/test_post_source_cpu.py makes bin for bin,
// texel for texel and record for record, without a GPU.  The device headers are compiled for the host through tests/host_shim/ (each
// __f*_rn intrinsic = one IEEE binary32 operation under -ffp-contract=off).  The parameters come from the headers' builders, as in
// oxc_eye_adaptation and oxc_bloom.  Test infrastructure only.
//
//   post_vs_oracle <inputs.bin> <outputs.bin>
// inputs.bin: width u32, height u32, OxcEyeAdaptationSettings, delta_time f32, OxcExposure, OxcBloomSettings, the frame (width x height
// float4), the upsampled chain's content before the call (bloom_chain_texels float4; only width, height >= 2).  outputs.bin receives
// the 256 u32 bins, the record after eye adaptation, then (width, height >= 2) the downsampled and upsampled chains; the bloom reads the
// record as eye adaptation left it.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "oxc_bloom.cuh"
#include "oxc_exposure.cuh"

using namespace oxc;

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s inputs.bin outputs.bin\n", argv[0]); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  uint32_t wh[2];
  OxcEyeAdaptationSettings es;
  float dt;
  OxcExposure record;
  OxcBloomSettings bs;
  if (std::fread(wh, 4, 2, f) != 2 || std::fread(&es, sizeof es, 1, f) != 1 || std::fread(&dt, 4, 1, f) != 1 ||
      std::fread(&record, sizeof record, 1, f) != 1 || std::fread(&bs, sizeof bs, 1, f) != 1)
    return 2;
  const uint32_t w = wh[0], h = wh[1];
  const bool bloom = w >= 2 && h >= 2;
  const size_t chain = bloom ? (size_t)bloom_chain_texels(w, h) : 0;
  std::vector<float> frame((size_t)w * h * 4), down(chain * 4), up(chain * 4);
  if (std::fread(frame.data(), 4, frame.size(), f) != frame.size() || std::fread(up.data(), 4, up.size(), f) != up.size()) return 2;
  std::fclose(f);

  std::vector<uint32_t> bins(HISTOGRAM_BINS, 0);
  const EyeAdaptationParams ep = eye_adaptation_make_params(frame.data(), w, h, es, dt, &record, bins.data());
  for (uint64_t i = 0; i < ep.pixels; i++) bins[histogram_bin(ep, ep.frame[i])]++;
  uint32_t weighted = 0;
  for (uint32_t i = 0; i < (uint32_t)HISTOGRAM_BINS; i++) weighted += bins[i] * i;
  record = exposure_update(ep, weighted, bins[0], record);

  if (bloom) {
    const OxcBloomTargets t{down.data(), up.data()};
    const BloomParams p = bloom_make_params(frame.data(), w, h, bs, &record, t);
    for (int y = 0; y < p.h[0]; y++)
      for (int x = 0; x < p.w[0]; x++) bloom_prefilter_texel(p, x, y);
    for (int i = 1; i < p.levels; i++)
      for (int y = 0; y < p.h[i]; y++)
        for (int x = 0; x < p.w[i]; x++) bloom_downsample_texel(p, i, x, y);
    for (int i = p.levels - 1; i >= 1; i--)
      for (int y = 0; y < p.h[i - 1]; y++)
        for (int x = 0; x < p.w[i - 1]; x++) bloom_upsample_texel(p, i, x, y);
    if (p.levels == 1)
      for (int y = 0; y < p.h[0]; y++)
        for (int x = 0; x < p.w[0]; x++) bloom_black_texel(p, x, y);
  }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o || std::fwrite(bins.data(), 4, bins.size(), o) != bins.size() || std::fwrite(&record, sizeof record, 1, o) != 1 ||
      std::fwrite(down.data(), 4, down.size(), o) != down.size() || std::fwrite(up.data(), 4, up.size(), o) != up.size())
    return 2;
  std::fclose(o);
  return 0;
}
