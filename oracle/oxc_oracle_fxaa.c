/*
 * oxc_oracle_fxaa.c — CPU ORACLE (test infrastructure) of the FXAA pass (passes/fxaa/fxaa.slang fs_main, RendererInstance.cpp:1225-1255),
 * written line by line from fs_main with both uv components carried through the walk.  One translation unit with oxc_oracle_post.c,
 * included below, for bloom's luminance weights (P_CLUM_*), the NaN rules of max / min (a_max, a_min), the saturating float -> int
 * conversion (alpha_f2i) and the edge clamp (a_clampi).  Built into liboxc_oracle_fxaa.so by oracle/pyoracle_fxaa.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_fxaa.c -lm
 *
 * SPECIFICATION: include/oxcull.h above oxc_fxaa (items 1-7).  binary32, no contraction, each expression in the shader's written order;
 * max / min take the other operand for a NaN; every stored NaN is 0x7FFFFFFF.
 */
#include "oxc_oracle_post.c"

#include "oxc_oracle_fxaa.h"

#define F_EDGE_THRESHOLD_MIN 0.0312f
#define F_EDGE_THRESHOLD_MAX 0.125f
#define F_SUBPIXEL_QUALITY 0.75f
#define F_ITERATIONS 12

void orc_fxaa_constants(float out[ORC_FXAA_CONSTANTS]) {
  out[0] = F_EDGE_THRESHOLD_MIN;
  out[1] = F_EDGE_THRESHOLD_MAX;
  out[2] = F_SUBPIXEL_QUALITY;
  out[3] = 1.0f / 12.0f;
}

float orc_fxaa_quality(int32_t q) { return q < 5 ? 1.0f : (q > 5 ? (q < 10 ? 2.0f : (q < 11 ? 4.0f : 8.0f)) : 1.5f); }

float orc_fxaa_luma(const float rgb[3]) { return sqrtf((rgb[0] * P_CLUM_R + rgb[1] * P_CLUM_G) + rgb[2] * P_CLUM_B); }

void orc_fxaa_tap(const float* src, uint32_t W, uint32_t H, float u, float v, int32_t dx, int32_t dy, float out[4]) {
  /* (u * W + dx) - 0.5: with dx = 0 the sum is u * W itself (or +0 for -0, which the - 0.5 cannot tell apart) */
  const float x = (u * (float)W + (float)dx) - 0.5f, y = (v * (float)H + (float)dy) - 0.5f;
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = x - x0, wy = y - y0;
  const int64_t ix = alpha_f2i(x0), iy = alpha_f2i(y0);
  const float* q[4];
  for (int k = 0; k < 4; k++) q[k] = src + ((size_t)a_clampi(iy + (k >> 1), H) * W + (size_t)a_clampi(ix + (k & 1), W)) * 4;
  for (int c = 0; c < 4; c++) {
    const float top = q[0][c] + wx * (q[1][c] - q[0][c]), bot = q[2][c] + wx * (q[3][c] - q[2][c]);
    out[c] = top + wy * (bot - top);
  }
}

typedef struct {
  const float* src;
  uint32_t W, H;
  int taps;
} FxaaImage;

static void f_sample(FxaaImage* im, const float uv[2], int32_t dx, int32_t dy, float out[4]) {
  orc_fxaa_tap(im->src, im->W, im->H, uv[0], uv[1], dx, dy, out);
  im->taps++;
}
static float f_luma_at(FxaaImage* im, const float uv[2], int32_t dx, int32_t dy) {
  float c[4];
  f_sample(im, uv, dx, dy, c);
  return orc_fxaa_luma(c);
}

/* fs_main at tex_coord; inverse_screen_size = inv */
static void f_fs_main(FxaaImage* im, const float tex_coord[2], const float inv[2], float result[4]) {
  float color_center[4];
  f_sample(im, tex_coord, 0, 0, color_center);
  const float luma_center = orc_fxaa_luma(color_center);
  const float luma_down = f_luma_at(im, tex_coord, 0, -1);
  const float luma_up = f_luma_at(im, tex_coord, 0, 1);
  const float luma_left = f_luma_at(im, tex_coord, -1, 0);
  const float luma_right = f_luma_at(im, tex_coord, 1, 0);
  const float luma_min = a_min(luma_center, a_min(a_min(luma_down, luma_up), a_min(luma_left, luma_right)));
  const float luma_max = a_max(luma_center, a_max(a_max(luma_down, luma_up), a_max(luma_left, luma_right)));
  const float luma_range = luma_max - luma_min;
  if (luma_range < a_max(F_EDGE_THRESHOLD_MIN, luma_max * F_EDGE_THRESHOLD_MAX)) {
    memcpy(result, color_center, sizeof color_center);
    return;
  }
  const float luma_down_left = f_luma_at(im, tex_coord, -1, -1);
  const float luma_up_right = f_luma_at(im, tex_coord, 1, 1);
  const float luma_up_left = f_luma_at(im, tex_coord, -1, 1);
  const float luma_down_right = f_luma_at(im, tex_coord, 1, -1);
  const float luma_down_up = luma_down + luma_up;
  const float luma_left_right = luma_left + luma_right;
  const float luma_left_corners = luma_down_left + luma_up_left;
  const float luma_down_corners = luma_down_left + luma_down_right;
  const float luma_right_corners = luma_down_right + luma_up_right;
  const float luma_up_corners = luma_up_right + luma_up_left;
  const float edge_horizontal = fabsf(-2.0f * luma_left + luma_left_corners) + fabsf(-2.0f * luma_center + luma_down_up) * 2.0f +
                                fabsf(-2.0f * luma_right + luma_right_corners);
  const float edge_vertical = fabsf(-2.0f * luma_up + luma_up_corners) + fabsf(-2.0f * luma_center + luma_left_right) * 2.0f +
                              fabsf(-2.0f * luma_down + luma_down_corners);
  const int is_horizontal = edge_horizontal >= edge_vertical;
  float step_length = is_horizontal ? inv[1] : inv[0];
  const float luma1 = is_horizontal ? luma_down : luma_left;
  const float luma2 = is_horizontal ? luma_up : luma_right;
  const float gradient1 = luma1 - luma_center;
  const float gradient2 = luma2 - luma_center;
  const int is1_steepest = fabsf(gradient1) >= fabsf(gradient2);
  const float gradient_scaled = 0.25f * a_max(fabsf(gradient1), fabsf(gradient2));
  float luma_local_average;
  if (is1_steepest) {
    step_length = -step_length;
    luma_local_average = 0.5f * (luma1 + luma_center);
  } else {
    luma_local_average = 0.5f * (luma2 + luma_center);
  }
  float current_uv[2] = {tex_coord[0], tex_coord[1]};
  if (is_horizontal) current_uv[1] += step_length * 0.5f;
  else current_uv[0] += step_length * 0.5f;
  const float offset[2] = {is_horizontal ? inv[0] : 0.0f, is_horizontal ? 0.0f : inv[1]};
  float uv1[2], uv2[2];
  for (int k = 0; k < 2; k++) {
    uv1[k] = current_uv[k] - offset[k] * orc_fxaa_quality(0);
    uv2[k] = current_uv[k] + offset[k] * orc_fxaa_quality(0);
  }
  float luma_end1 = f_luma_at(im, uv1, 0, 0);
  float luma_end2 = f_luma_at(im, uv2, 0, 0);
  luma_end1 -= luma_local_average;
  luma_end2 -= luma_local_average;
  int reached1 = fabsf(luma_end1) >= gradient_scaled;
  int reached2 = fabsf(luma_end2) >= gradient_scaled;
  int reached_both = reached1 && reached2;
  if (!reached1)
    for (int k = 0; k < 2; k++) uv1[k] -= offset[k] * orc_fxaa_quality(1);
  if (!reached2)
    for (int k = 0; k < 2; k++) uv2[k] += offset[k] * orc_fxaa_quality(1);
  if (!reached_both) {
    for (int i = 2; i < F_ITERATIONS; i++) {
      if (!reached1) {
        luma_end1 = f_luma_at(im, uv1, 0, 0);
        luma_end1 = luma_end1 - luma_local_average;
      }
      if (!reached2) {
        luma_end2 = f_luma_at(im, uv2, 0, 0);
        luma_end2 = luma_end2 - luma_local_average;
      }
      reached1 = fabsf(luma_end1) >= gradient_scaled;
      reached2 = fabsf(luma_end2) >= gradient_scaled;
      reached_both = reached1 && reached2;
      if (!reached1)
        for (int k = 0; k < 2; k++) uv1[k] -= offset[k] * orc_fxaa_quality(i);
      if (!reached2)
        for (int k = 0; k < 2; k++) uv2[k] += offset[k] * orc_fxaa_quality(i);
      if (reached_both) break;
    }
  }
  const float distance1 = is_horizontal ? (tex_coord[0] - uv1[0]) : (tex_coord[1] - uv1[1]);
  const float distance2 = is_horizontal ? (uv2[0] - tex_coord[0]) : (uv2[1] - tex_coord[1]);
  const int is_direction1 = distance1 < distance2;
  const float distance_final = a_min(distance1, distance2);
  const float edge_thickness = (distance1 + distance2);
  const int is_luma_center_smaller = luma_center < luma_local_average;
  const int correct_variation1 = (luma_end1 < 0.0f) != is_luma_center_smaller;
  const int correct_variation2 = (luma_end2 < 0.0f) != is_luma_center_smaller;
  const int correct_variation = is_direction1 ? correct_variation1 : correct_variation2;
  const float pixel_offset = -distance_final / edge_thickness + 0.5f;
  float final_offset = correct_variation ? pixel_offset : 0.0f;
  const float luma_average = (1.0f / 12.0f) * (2.0f * (luma_down_up + luma_left_right) + luma_left_corners + luma_right_corners);
  const float sub_pixel_offset1 = a_min(a_max(fabsf(luma_average - luma_center) / luma_range, 0.0f), 1.0f);
  const float sub_pixel_offset2 = (-2.0f * sub_pixel_offset1 + 3.0f) * sub_pixel_offset1 * sub_pixel_offset1;
  const float sub_pixel_offset_final = sub_pixel_offset2 * sub_pixel_offset2 * F_SUBPIXEL_QUALITY;
  final_offset = a_max(final_offset, sub_pixel_offset_final);
  float final_uv[2] = {tex_coord[0], tex_coord[1]};
  if (is_horizontal) final_uv[1] += final_offset * step_length;
  else final_uv[0] += final_offset * step_length;
  f_sample(im, final_uv, 0, 0, result);
}

void orc_fxaa(const float* frame, uint32_t width, uint32_t height, float* out, uint8_t* taps) {
  const float inv[2] = {1.0f / (float)width, 1.0f / (float)height};
  for (uint32_t y = 0; y < height; y++)
    for (uint32_t x = 0; x < width; x++) {
      const float tex_coord[2] = {((float)x + 0.5f) / (float)width, ((float)y + 0.5f) / (float)height};
      FxaaImage im = {frame, width, height, 0};
      float c[4];
      f_fs_main(&im, tex_coord, inv, c);
      float* o = out + ((size_t)y * width + x) * 4;
      for (int k = 0; k < 4; k++) o[k] = p_nan(c[k]);
      if (taps) taps[(size_t)y * width + x] = (uint8_t)im.taps;
    }
}
