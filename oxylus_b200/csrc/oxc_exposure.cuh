// oxc_exposure.cuh — eye adaptation (PostProcess.cpp:7-77, passes/histogram_generate.slang, passes/histogram_average.slang): the bin of
// one pixel and the exposure record's update from the finished histogram, as include/oxcull.h oxc_eye_adaptation specifies them (items
// 1-3) and oracle/oxc_oracle_post.c computes them.  kernels_exposure.cuh lays the pixels and bins out.
// No warp intrinsics, no shared memory: tests compile this source for the host.
#pragma once
#include "oxc_shader_math.cuh"

namespace oxc {

constexpr int HISTOGRAM_BINS = 256;
constexpr float HISTOGRAM_LUM_R = 0x1.b39c0ep-3f;  // 0.2127, 0x3E59CE07
constexpr float HISTOGRAM_LUM_G = 0x1.6e2eb2p-1f;  // 0.7152, 0x3F371759
constexpr float HISTOGRAM_LUM_B = 0x1.27bb3p-4f;   // 0.0722, 0x3D93DD98
constexpr float LUMINANCE_EPSILON = 0x1.0624dep-10f; // 0.001, 0x3A83126F
constexpr float EXPOSURE_K = 0x1.333334p+0f;       // 1.2, 0x3F99999A

struct EyeAdaptationParams {
  const float4* frame;
  uint32_t width, height;
  uint64_t pixels;
  float min_exposure, exposure_range; // histogram_generate's remap and histogram_average's push constants
  float pixel_count, time_coeff, bias_scale;
  OxcExposure* record;
  uint32_t* histogram;
};

// item 1: the per-call values, formed once on the host (the ABI and tests/post_vs_oracle.cpp call it)
inline EyeAdaptationParams eye_adaptation_make_params(const float* frame, uint32_t width, uint32_t height, const OxcEyeAdaptationSettings& s,
                                                      float delta_time, OxcExposure* record, uint32_t* histogram) {
  EyeAdaptationParams p;
  p.frame = reinterpret_cast<const float4*>(frame);
  p.width = width;
  p.height = height;
  p.pixels = (uint64_t)width * height;
  p.min_exposure = s.min_exposure;
  p.exposure_range = hd_sub(s.max_exposure, s.min_exposure);
  p.pixel_count = (float)(uint32_t)(width * height);
  p.time_coeff = hd_sub(1.0f, canonical_exp(hd_mul(-s.adaptation_speed, delta_time)));
  p.bias_scale = hd_mul(100.0f, s.ev100_bias) / 12.5f; // ISO * ev100_bias / K, one IEEE division in the host build
  p.record = record;
  p.histogram = histogram;
  return p;
}

// item 2: bin_lum(dot(rgb, (0.2127, 0.7152, 0.0722))); alpha is not read
OXC_DI int histogram_bin(const EyeAdaptationParams& p, float4 c) {
  const float lum = dot3(c.x, c.y, c.z, HISTOGRAM_LUM_R, HISTOGRAM_LUM_G, HISTOGRAM_LUM_B);
  if (lum < LUMINANCE_EPSILON) return 0;
  const float mapped = fa(fm(fd(fs(canonical_log2(lum), p.min_exposure), p.exposure_range), 254.0f), 1.0f);
  const int b = sat_i32(mapped);
  return b < 0 ? 0 : (b > HISTOGRAM_BINS - 1 ? HISTOGRAM_BINS - 1 : b);
}

// item 3: the record after one frame, from weighted = sum bins[i] * i mod 2^32 and the dark bin
OXC_DI OxcExposure exposure_update(const EyeAdaptationParams& p, uint32_t weighted, uint32_t dark, OxcExposure last) {
  const float avg = fs(fd((float)weighted, vmax(fs(p.pixel_count, (float)dark), 1.0f)), 1.0f);
  const float desired = canonical_pow(2.0f, fa(fm(fd(avg, 254.0f), p.exposure_range), p.min_exposure));
  const float adapted = fa(last.adapted_luminance, fm(fs(desired, last.adapted_luminance), p.time_coeff));
  const float ev100 = canonical_log2(fm(adapted, p.bias_scale));
  OxcExposure out;
  out.adapted_luminance = nan_canonical(adapted);
  out.exposure = nan_canonical(fd(1.0f, fm(canonical_pow(2.0f, ev100), EXPOSURE_K)));
  return out;
}

} // namespace oxc
