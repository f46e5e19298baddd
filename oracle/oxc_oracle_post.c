/*
 * oxc_oracle_post.c — CPU ORACLE (test infrastructure) of the post-processing inputs of the tonemap: eye adaptation
 * (passes/histogram_generate.slang, histogram_average.slang, PostProcess.cpp:7-77) and bloom (passes/bloom_prefilter.slang,
 * bloom_downsample.slang, bloom_upsample.slang, PostProcess.cpp:79-203), one C function per shader function.  One translation unit with
 * oxc_oracle_atmosphere.c, included below, so that it runs the library's own log2 (orc_log2_canonical), exp (orc_exp_canonical), pow
 * (orc_pow_canonical) and the saturating float -> int conversion (alpha_f2i).  Built into liboxc_oracle_post.so by oracle/pyoracle_post.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_post.c -lm
 *
 * SPECIFICATION: include/oxcull.h above oxc_eye_adaptation (items 1-3) and oxc_bloom (items 1-6).  binary32, no contraction, each
 * expression in the shader's written order; max / min take the other operand for a NaN; every stored NaN is 0x7FFFFFFF.
 */
#include "oxc_oracle_atmosphere.c"

#include "oxc_oracle_post.h"

static const float P_LUM_R = 0x1.b39c0ep-3f, P_LUM_G = 0x1.6e2eb2p-1f, P_LUM_B = 0x1.27bb3p-4f, P_EPSILON = 0x1.0624dep-10f,
                   P_K = 0x1.333334p+0f, P_CLUM_R = 0x1.322d0ep-2f, P_CLUM_G = 0x1.2c8b44p-1f, P_CLUM_B = 0x1.d2f1aap-4f,
                   P_EPS5 = 0x1.4f8b58p-17f;

static float p_nan(float v) { return v != v ? bits2f(0x7FFFFFFFu) : v; }

/* ---------------------------------------------------------------- eye adaptation */

/* item 1, PostProcess.cpp:44-66: the histogram_average push constants and bin_lum's remap range */
void orc_eye_adaptation_constants(const OxcEyeAdaptationSettings* s, uint32_t width, uint32_t height, float delta_time, float out[4]) {
  out[0] = (float)(width * height);                                   /* pixel_count */
  out[1] = s->max_exposure - s->min_exposure;                         /* exposure_range */
  out[2] = 1.0f - orc_exp_canonical(-s->adaptation_speed * delta_time); /* time_coeff */
  out[3] = (100.0f * s->ev100_bias) / 12.5f;                          /* ISO * ev100_bias / K */
}

/* histogram_generate.slang bin_lum(dot(color, (0.2127, 0.7152, 0.0722))) */
uint32_t orc_histogram_bin(const OxcEyeAdaptationSettings* s, float r, float g, float b) {
  const float luminance = (r * P_LUM_R + g * P_LUM_G) + b * P_LUM_B;
  if (luminance < P_EPSILON) return 0;
  /* com::remap(log2(luminance), min, max, 1, 255): (val - start1) / (end1 - start1) * (end2 - start2) + start2 */
  const float mapped = ((orc_log2_canonical(luminance) - s->min_exposure) / (s->max_exposure - s->min_exposure)) * 254.0f + 1.0f;
  const int i = alpha_f2i(mapped);
  return (uint32_t)(i < 0 ? 0 : (i > 255 ? 255 : i));
}

/* histogram_average.slang cs_main at gid 0, after the group's u32 InterlockedAdd of bins[i] * i */
void orc_histogram_average(const uint32_t bins[256], const float constants[4], float min_exposure, OxcExposure* record) {
  uint32_t weighted_sum = 0;
  for (uint32_t gid = 0; gid < 256; gid++) weighted_sum += bins[gid] * gid; /* mod 2^32 */
  const float dark_pixel_count = (float)bins[0];
  const float weighted_average_log2 = ((float)weighted_sum / a_max(constants[0] - dark_pixel_count, 1.0f)) - 1.0f;
  const float desired_luminance = orc_pow_canonical(2.0f, ((weighted_average_log2 / 254.0f) * constants[1]) + min_exposure);
  const float last_luminance = record->adapted_luminance;
  const float adapted_luminance = last_luminance + (desired_luminance - last_luminance) * constants[2];
  const float ev100 = orc_log2_canonical(adapted_luminance * constants[3]);
  record->adapted_luminance = p_nan(adapted_luminance);
  record->exposure = p_nan(1.0f / (orc_pow_canonical(2.0f, ev100) * P_K));
}

void orc_eye_adaptation(const float* frame, uint32_t width, uint32_t height, const OxcEyeAdaptationSettings* settings, float delta_time,
                        OxcExposure* record, uint32_t histogram[256]) {
  float constants[4];
  orc_eye_adaptation_constants(settings, width, height, delta_time, constants);
  memset(histogram, 0, 256 * sizeof(uint32_t));
  const uint64_t n = (uint64_t)width * height;
  for (uint64_t i = 0; i < n; i++) histogram[orc_histogram_bin(settings, frame[i * 4], frame[i * 4 + 1], frame[i * 4 + 2])]++;
  orc_histogram_average(histogram, constants, settings->min_exposure, record);
}

/* ---------------------------------------------------------------- bloom */

uint32_t orc_bloom_level_count(uint32_t width, uint32_t height) {
  uint32_t m = width / 2 > height / 2 ? width / 2 : height / 2, n = 0;
  for (; m; m >>= 1) n++;
  return n;
}

/* SampleLevel(sampler, uv, 0).rgb of a W x H float4 plane: LinearSamplerBorder (transparent black) or LinearSamplerClamped */
void orc_bloom_tap(const float* src, uint32_t W, uint32_t H, float u, float v, int border, float out[3]) {
  const float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = x - x0, wy = y - y0;
  const int64_t ix = alpha_f2i(x0), iy = alpha_f2i(y0);
  float q[4][3];
  for (int k = 0; k < 4; k++) {
    const int64_t xi = ix + (k & 1), yi = iy + (k >> 1);
    const int outside = xi < 0 || xi >= (int64_t)W || yi < 0 || yi >= (int64_t)H;
    for (int c = 0; c < 3; c++)
      q[k][c] = (border && outside) ? 0.0f : src[((size_t)a_clampi(yi, H) * W + (size_t)a_clampi(xi, W)) * 4 + c];
  }
  for (int c = 0; c < 3; c++) {
    const float top = q[0][c] + wx * (q[1][c] - q[0][c]), bot = q[2][c] + wx * (q[3][c] - q[2][c]);
    out[c] = top + wy * (bot - top);
  }
}

/* sample_color(src, sampler, uv, texel_size * offset) */
static void b_sample(const float* src, uint32_t W, uint32_t H, const float uv[2], const float ts[2], float dx, float dy, int border,
                     float out[3]) {
  orc_bloom_tap(src, W, H, uv[0] + ts[0] * dx, uv[1] + ts[1] * dy, border, out);
}

static void b_store(float* dst, const float v[3]) {
  for (int c = 0; c < 3; c++) dst[c] = p_nan(v[c]);
  dst[3] = 1.0f;
}

/* the 13 taps of bloom_prefilter.slang and bloom_downsample.slang, a..m */
static const float B_OFF13[13][2] = {{-2, 2}, {0, 2}, {2, 2}, {-2, 0}, {0, 0}, {2, 0}, {-2, -2}, {0, -2}, {2, -2},
                                     {-1, 1}, {1, 1}, {-1, -1}, {1, -1}};
enum { A_, B_, C_, D_, E_, F_, G_, H_, I_, J_, K_, L_, M_ };

static void b_coord(uint32_t x, uint32_t y, uint32_t w, uint32_t h, float uv[2], float ts[2]) {
  uv[0] = ((float)x + 0.5f) / (float)w;
  uv[1] = ((float)y + 0.5f) / (float)h;
  ts[0] = 1.0f / (float)w;
  ts[1] = 1.0f / (float)h;
}

/* bloom_prefilter.slang prefilter() */
static void b_prefilter(const float color[3], float threshold, float soft_threshold, float out[3]) {
  const float brightness = a_max(color[0], a_max(color[1], color[2]));
  const float knee = threshold * soft_threshold;
  float soft = brightness - threshold + knee;
  soft = a_min(a_max(soft, 0.0f), 2.0f * knee);
  soft = soft * soft * 0.25f / (knee + 1.0e-5f);
  float contribution = a_max(soft, brightness - threshold);
  contribution /= a_max(brightness, P_EPS5);
  for (int c = 0; c < 3; c++) out[c] = color[c] * contribution;
}

static void b_prefilter_texel(const float* frame, uint32_t fw, uint32_t fh, uint32_t w, uint32_t h, uint32_t x, uint32_t y,
                              const OxcBloomSettings* s, float exposure, float* dst) {
  float uv[2], ts[2], t[13][3];
  b_coord(x, y, w, h, uv, ts);
  for (int k = 0; k < 13; k++) b_sample(frame, fw, fh, uv, ts, B_OFF13[k][0], B_OFF13[k][1], 1, t[k]);
  static const int G[5][4] = {{A_, B_, D_, E_}, {B_, C_, E_, F_}, {D_, E_, G_, H_}, {E_, F_, H_, I_}, {J_, K_, L_, M_}};
  float color_sum[3] = {0.0f, 0.0f, 0.0f}, weight_sum = 0.0f;
  for (int gid = 0; gid < 5; gid++) {
    float group[3], pre[3];
    for (int c = 0; c < 3; c++) {
      group[c] = (t[G[gid][0]][c] + t[G[gid][1]][c] + t[G[gid][2]][c] + t[G[gid][3]][c]) * 0.25f * exposure;
      group[c] = a_min(group[c], s->clamp_value);
    }
    const float weight = 1.0f / (1.0f + ((group[0] * P_CLUM_R + group[1] * P_CLUM_G) + group[2] * P_CLUM_B)); /* karis_average */
    b_prefilter(group, s->threshold, s->soft_threshold, pre);
    for (int c = 0; c < 3; c++) color_sum[c] += pre[c] * weight;
    weight_sum += weight;
  }
  float r[3];
  for (int c = 0; c < 3; c++) r[c] = color_sum[c] / (weight_sum + 1.0e-5f);
  b_store(dst, r);
}

static void b_downsample_texel(const float* src, uint32_t sw, uint32_t sh, uint32_t w, uint32_t h, uint32_t x, uint32_t y, float* dst) {
  float uv[2], ts[2], t[13][3], r[3];
  b_coord(x, y, w, h, uv, ts);
  for (int k = 0; k < 13; k++) b_sample(src, sw, sh, uv, ts, B_OFF13[k][0], B_OFF13[k][1], 1, t[k]);
  for (int c = 0; c < 3; c++)
    r[c] = (t[A_][c] + t[C_][c] + t[G_][c] + t[I_][c]) * 0.03125f + (t[B_][c] + t[D_][c] + t[F_][c] + t[H_][c]) * 0.0625f +
           (t[E_][c] + t[J_][c] + t[K_][c] + t[L_][c] + t[M_][c]) * 0.125f;
  b_store(dst, r);
}

static void b_upsample_texel(const float* up_src, uint32_t sw, uint32_t sh, const float* down, uint32_t w, uint32_t h, uint32_t x,
                             uint32_t y, float radius, float* dst) {
  static const float OFF9[9][2] = {{-1, 1}, {0, 1}, {1, 1}, {-1, 0}, {0, 0}, {1, 0}, {-1, -1}, {0, -1}, {1, -1}};
  float uv[2], ts[2], t[9][3], src[3], r[3];
  b_coord(x, y, w, h, uv, ts);
  for (int k = 0; k < 9; k++) b_sample(up_src, sw, sh, uv, ts, OFF9[k][0], OFF9[k][1], 0, t[k]);
  orc_bloom_tap(down, w, h, uv[0], uv[1], 0, src);
  for (int c = 0; c < 3; c++) {
    const float color_sum = t[4][c] * 0.25f + (t[1][c] + t[3][c] + t[5][c] + t[7][c]) * 0.125f + (t[0][c] + t[2][c] + t[6][c] + t[8][c]) * 0.0625f;
    r[c] = src[c] + (color_sum - src[c]) * radius; /* lerp */
  }
  b_store(dst, r);
}

void orc_bloom(const float* frame, uint32_t width, uint32_t height, const OxcBloomSettings* settings, const OxcExposure* record,
               float* downsampled, float* upsampled) {
  const uint32_t n = orc_bloom_level_count(width, height);
  uint32_t w[32], h[32];
  size_t off[32];
  size_t o = 0;
  for (uint32_t k = 0; k < n; k++) {
    w[k] = (width / 2) >> k ? (width / 2) >> k : 1;
    h[k] = (height / 2) >> k ? (height / 2) >> k : 1;
    off[k] = o;
    o += (size_t)w[k] * h[k];
  }
  const float exposure = (settings->scene_flags & OXC_SCENE_HAS_EYE_ADAPTATION) ? record->exposure : 1.0f;
  for (uint32_t y = 0; y < h[0]; y++)
    for (uint32_t x = 0; x < w[0]; x++)
      b_prefilter_texel(frame, width, height, w[0], h[0], x, y, settings, exposure, downsampled + ((size_t)y * w[0] + x) * 4);
  for (uint32_t i = 1; i < n; i++)
    for (uint32_t y = 0; y < h[i]; y++)
      for (uint32_t x = 0; x < w[i]; x++)
        b_downsample_texel(downsampled + off[i - 1] * 4, w[i - 1], h[i - 1], w[i], h[i], x, y, downsampled + (off[i] + (size_t)y * w[i] + x) * 4);
  for (int i = (int)n - 1; i > 0; i--) {
    const float* src = (i == (int)n - 1 ? downsampled : upsampled) + off[i] * 4;
    for (uint32_t y = 0; y < h[i - 1]; y++)
      for (uint32_t x = 0; x < w[i - 1]; x++)
        b_upsample_texel(src, w[i], h[i], downsampled + off[i - 1] * 4, w[i - 1], h[i - 1], x, y, settings->radius,
                         upsampled + (off[i - 1] + (size_t)y * w[i - 1] + x) * 4);
  }
  if (n == 1) /* the reference's per-frame clear, vuk::Black<float> */
    for (size_t t = 0; t < (size_t)w[0] * h[0]; t++) {
      const float black[3] = {0.0f, 0.0f, 0.0f};
      b_store(upsampled + t * 4, black);
    }
}
