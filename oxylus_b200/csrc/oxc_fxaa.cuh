// oxc_fxaa.cuh — FXAA (RendererInstance.cpp:1225-1255, passes/fxaa/fxaa.slang fs_main): the value of one output pixel, as
// include/oxcull.h oxc_fxaa specifies it (items 1-7) and oracle/oxc_oracle_fxaa.c computes it.  kernels_fxaa.cuh lays the pixels out.
// The luma weights are bloom's (com::luminance's 0.299 / 0.587 / 0.114), hence the include.
// No warp intrinsics, no shared memory: tests compile this source for the host.
#pragma once
#include "oxc_bloom.cuh"
#include "oxc_shader_math.cuh"

namespace oxc {

// item 6: the binary32 roundings of the shader's literals (tests/test_oracle_fxaa.py checks the bits)
constexpr float FXAA_EDGE_THRESHOLD_MIN = 0x1.ff2e48p-6f; // 0.0312, 0x3CFF9724
constexpr float FXAA_EDGE_THRESHOLD_MAX = 0x1p-3f;        // 0.125, 0x3E000000
constexpr float FXAA_SUBPIXEL_QUALITY = 0x1.8p-1f;        // 0.75, 0x3F400000
constexpr float FXAA_ONE_TWELFTH = 0x1.555556p-4f;        // 1.0 / 12.0, 0x3DAAAAAB
constexpr int FXAA_ITERATIONS = 12;
constexpr int FXAA_MAX_TAPS = 32; // 1 centre, 4 cross, 4 corners, 2 first ends, 2 x 10 in the walk, 1 final

struct FxaaParams {
  const float4* frame;
  float4* out;
  int width, height;
  float inv_x, inv_y; // item 1: the push constant inverse_screen_size = 1 / f32(extent), formed once per call
};

inline FxaaParams fxaa_make_params(const float* frame, uint32_t width, uint32_t height, float* out) {
  FxaaParams p;
  p.frame = reinterpret_cast<const float4*>(frame);
  p.out = reinterpret_cast<float4*>(out);
  p.width = (int)width;
  p.height = (int)height;
  p.inv_x = 1.0f / (float)width; // one IEEE division in the host build
  p.inv_y = 1.0f / (float)height;
  return p;
}

// item 5: QUALITY(i) = 1 for i <= 4, 1.5 at 5, 2 for 6..9, 4 at 10, 8 at 11
OXC_DI float fxaa_quality(int i) { return i < 5 ? 1.0f : (i > 5 ? (i < 10 ? 2.0f : (i < 11 ? 4.0f : 8.0f)) : 1.5f); }

// item 3: sqrt((r * 0.299 + g * 0.587) + b * 0.114); a negative sum gives NaN
OXC_DI float fxaa_luma(float4 c) { return fsq(dot3(c.x, c.y, c.z, BLOOM_LUM_R, BLOOM_LUM_G, BLOOM_LUM_B)); }

// item 2: Sample(uv) and Sample(uv, int2(dx, dy)) through LinearSamplerClamped
OXC_DI float4 fxaa_tap(const FxaaParams& p, float u, float v) { return bilinear_tap<CLAMP_TO_EDGE>(p.frame, p.width, p.height, u, v); }
OXC_DI float fxaa_luma_at(const FxaaParams& p, float u, float v, int dx, int dy) {
  return fxaa_luma(bilinear_tap<CLAMP_TO_EDGE>(p.frame, p.width, p.height, u, v, dx, dy));
}

// items 2-5: the filtered colour of pixel (x, y); taps receives the bilinear taps taken (5 on the early exit, 12..32 otherwise).  The
// walk advances only the moving axis: the other component's offset is 0, and uv - 0 * QUALITY(i) is uv itself (item 5).
OXC_DI float4 fxaa_filter(const FxaaParams& p, int x, int y, int& taps) {
  const float u = fd(fa((float)x, 0.5f), (float)p.width), v = fd(fa((float)y, 0.5f), (float)p.height);
  const float4 color_center = fxaa_tap(p, u, v);
  const float luma_center = fxaa_luma(color_center);
  const float luma_down = fxaa_luma_at(p, u, v, 0, -1), luma_up = fxaa_luma_at(p, u, v, 0, 1);
  const float luma_left = fxaa_luma_at(p, u, v, -1, 0), luma_right = fxaa_luma_at(p, u, v, 1, 0);
  const float luma_min = vmin(luma_center, vmin(vmin(luma_down, luma_up), vmin(luma_left, luma_right)));
  const float luma_max = vmax(luma_center, vmax(vmax(luma_down, luma_up), vmax(luma_left, luma_right)));
  const float luma_range = fs(luma_max, luma_min);
  taps = 5;
  if (luma_range < vmax(FXAA_EDGE_THRESHOLD_MIN, fm(luma_max, FXAA_EDGE_THRESHOLD_MAX))) return color_center; // item 4
  const float luma_down_left = fxaa_luma_at(p, u, v, -1, -1), luma_up_right = fxaa_luma_at(p, u, v, 1, 1);
  const float luma_up_left = fxaa_luma_at(p, u, v, -1, 1), luma_down_right = fxaa_luma_at(p, u, v, 1, -1);
  const float luma_down_up = fa(luma_down, luma_up), luma_left_right = fa(luma_left, luma_right);
  const float luma_left_corners = fa(luma_down_left, luma_up_left), luma_down_corners = fa(luma_down_left, luma_down_right);
  const float luma_right_corners = fa(luma_down_right, luma_up_right), luma_up_corners = fa(luma_up_right, luma_up_left);
  const float edge_horizontal = fa(fa(fabsf(fa(fm(-2.0f, luma_left), luma_left_corners)), fm(fabsf(fa(fm(-2.0f, luma_center), luma_down_up)), 2.0f)),
                                   fabsf(fa(fm(-2.0f, luma_right), luma_right_corners)));
  const float edge_vertical = fa(fa(fabsf(fa(fm(-2.0f, luma_up), luma_up_corners)), fm(fabsf(fa(fm(-2.0f, luma_center), luma_left_right)), 2.0f)),
                                 fabsf(fa(fm(-2.0f, luma_down), luma_down_corners)));
  const bool is_horizontal = edge_horizontal >= edge_vertical;
  float step_length = is_horizontal ? p.inv_y : p.inv_x;
  const float luma1 = is_horizontal ? luma_down : luma_left, luma2 = is_horizontal ? luma_up : luma_right;
  const float gradient1 = fs(luma1, luma_center), gradient2 = fs(luma2, luma_center);
  const bool is1_steepest = fabsf(gradient1) >= fabsf(gradient2);
  const float gradient_scaled = fm(0.25f, vmax(fabsf(gradient1), fabsf(gradient2)));
  float luma_local_average;
  if (is1_steepest) {
    step_length = -step_length;
    luma_local_average = fm(0.5f, fa(luma1, luma_center));
  } else {
    luma_local_average = fm(0.5f, fa(luma2, luma_center));
  }
  // the walk runs along `along` (u for a horizontal edge, v otherwise) at the fixed `across`, shifted half a pixel toward the edge
  const float along = is_horizontal ? u : v, across = fa(is_horizontal ? v : u, fm(step_length, 0.5f));
  const float offset = is_horizontal ? p.inv_x : p.inv_y;
  float a1 = fs(along, fm(offset, fxaa_quality(0))), a2 = fa(along, fm(offset, fxaa_quality(0)));
  float luma_end1 = fs(is_horizontal ? fxaa_luma(fxaa_tap(p, a1, across)) : fxaa_luma(fxaa_tap(p, across, a1)), luma_local_average);
  float luma_end2 = fs(is_horizontal ? fxaa_luma(fxaa_tap(p, a2, across)) : fxaa_luma(fxaa_tap(p, across, a2)), luma_local_average);
  taps = 11;
  bool reached1 = fabsf(luma_end1) >= gradient_scaled, reached2 = fabsf(luma_end2) >= gradient_scaled;
  if (!reached1) a1 = fs(a1, fm(offset, fxaa_quality(1)));
  if (!reached2) a2 = fa(a2, fm(offset, fxaa_quality(1)));
  if (!(reached1 && reached2)) {
    for (int i = 2; i < FXAA_ITERATIONS; i++) {
      if (!reached1) {
        luma_end1 = fs(is_horizontal ? fxaa_luma(fxaa_tap(p, a1, across)) : fxaa_luma(fxaa_tap(p, across, a1)), luma_local_average);
        taps++;
      }
      if (!reached2) {
        luma_end2 = fs(is_horizontal ? fxaa_luma(fxaa_tap(p, a2, across)) : fxaa_luma(fxaa_tap(p, across, a2)), luma_local_average);
        taps++;
      }
      reached1 = fabsf(luma_end1) >= gradient_scaled;
      reached2 = fabsf(luma_end2) >= gradient_scaled;
      if (!reached1) a1 = fs(a1, fm(offset, fxaa_quality(i)));
      if (!reached2) a2 = fa(a2, fm(offset, fxaa_quality(i)));
      if (reached1 && reached2) break; // after this step's advance, as the shader writes it
    }
  }
  const float distance1 = fs(along, a1), distance2 = fs(a2, along);
  const bool is_direction1 = distance1 < distance2;
  const float distance_final = vmin(distance1, distance2);
  const float edge_thickness = fa(distance1, distance2);
  const bool is_luma_center_smaller = luma_center < luma_local_average;
  const bool correct_variation1 = (luma_end1 < 0.0f) != is_luma_center_smaller;
  const bool correct_variation2 = (luma_end2 < 0.0f) != is_luma_center_smaller;
  const bool correct_variation = is_direction1 ? correct_variation1 : correct_variation2;
  const float pixel_offset = fa(fd(-distance_final, edge_thickness), 0.5f);
  float final_offset = correct_variation ? pixel_offset : 0.0f;
  const float luma_average = fm(FXAA_ONE_TWELFTH, fa(fa(fm(2.0f, fa(luma_down_up, luma_left_right)), luma_left_corners), luma_right_corners));
  const float sub_pixel_offset1 = saturate(fd(fabsf(fs(luma_average, luma_center)), luma_range));
  const float sub_pixel_offset2 = fm(fm(fa(fm(-2.0f, sub_pixel_offset1), 3.0f), sub_pixel_offset1), sub_pixel_offset1);
  const float sub_pixel_offset_final = fm(fm(sub_pixel_offset2, sub_pixel_offset2), FXAA_SUBPIXEL_QUALITY);
  final_offset = vmax(final_offset, sub_pixel_offset_final);
  const float shift = fm(final_offset, step_length);
  taps++;
  return is_horizontal ? fxaa_tap(p, u, fa(v, shift)) : fxaa_tap(p, fa(u, shift), v);
}

// item 7: the stored pixel, every NaN as 0x7FFFFFFF
OXC_DI float4 fxaa_pixel(const FxaaParams& p, int x, int y, int& taps) {
  const float4 c = fxaa_filter(p, x, y, taps);
  return make_float4(nan_canonical(c.x), nan_canonical(c.y), nan_canonical(c.z), nan_canonical(c.w));
}

} // namespace oxc
