// oxc_bloom.cuh — bloom (PostProcess.cpp:79-203, passes/bloom_prefilter.slang, bloom_downsample.slang, bloom_upsample.slang): the
// value of one texel of each pass, as include/oxcull.h oxc_bloom specifies it (items 1-6) and oracle/oxc_oracle_post.c computes it.
// kernels_bloom.cuh decides which launch writes which texel; every path calls these functions, so the bits do not depend on it.
// The planes are read with plain loads: the fused tail reads levels the same kernel wrote before a barrier.
// No warp intrinsics, no shared memory: tests compile this source for the host.
#pragma once
#include "oxc_shader_math.cuh"

namespace oxc {

constexpr int BLOOM_MAX_LEVELS = (int)OXC_BLOOM_MAX_LEVELS;
constexpr float BLOOM_LUM_R = 0x1.322d0ep-2f;  // 0.299, 0x3E991687 (com::luminance, not the histogram's weights)
constexpr float BLOOM_LUM_G = 0x1.2c8b44p-1f;  // 0.587, 0x3F1645A2
constexpr float BLOOM_LUM_B = 0x1.d2f1aap-4f;  // 0.114, 0x3DE978D5
constexpr float BLOOM_EPS = 0x1.4f8b58p-17f;   // 1e-5, 0x3727C5AC

struct BloomParams {
  const float4* frame;
  int frame_w, frame_h;
  int levels;                    // n
  int w[BLOOM_MAX_LEVELS], h[BLOOM_MAX_LEVELS];
  uint64_t offset[BLOOM_MAX_LEVELS]; // first texel of each level in both chains
  float4* down;
  float4* up;
  float threshold, soft_threshold, clamp_value, radius;
  const OxcExposure* record;     // read under HasEyeAdaptation only, else nullptr
};

// n = the bit length of max(width / 2, height / 2) (Texture::calculate_mip_count), and the texels of one chain
inline int bloom_level_count(uint32_t width, uint32_t height) {
  uint32_t m = (width / 2u) > (height / 2u) ? (width / 2u) : (height / 2u);
  int n = 0;
  for (; m; m >>= 1) n++;
  return n;
}
inline uint64_t bloom_chain_texels(uint32_t width, uint32_t height) {
  uint64_t t = 0;
  for (int k = 0; k < bloom_level_count(width, height); k++) {
    const uint32_t w = (width / 2u) >> k, h = (height / 2u) >> k;
    t += (uint64_t)(w ? w : 1u) * (h ? h : 1u);
  }
  return t;
}

inline BloomParams bloom_make_params(const float* frame, uint32_t width, uint32_t height, const OxcBloomSettings& s, const OxcExposure* record,
                                     const OxcBloomTargets& t) {
  BloomParams p;
  p.frame = reinterpret_cast<const float4*>(frame);
  p.frame_w = (int)width;
  p.frame_h = (int)height;
  p.levels = bloom_level_count(width, height);
  uint64_t off = 0;
  for (int k = 0; k < BLOOM_MAX_LEVELS; k++) {
    const uint32_t w = (width / 2u) >> k, h = (height / 2u) >> k;
    p.w[k] = w ? (int)w : 1;
    p.h[k] = h ? (int)h : 1;
    p.offset[k] = off;
    if (k < p.levels) off += (uint64_t)p.w[k] * p.h[k];
  }
  p.down = reinterpret_cast<float4*>(t.downsampled);
  p.up = reinterpret_cast<float4*>(t.upsampled);
  p.threshold = s.threshold;
  p.soft_threshold = s.soft_threshold;
  p.clamp_value = s.clamp_value;
  p.radius = s.radius;
  p.record = (s.scene_flags & OXC_SCENE_HAS_EYE_ADAPTATION) ? record : nullptr;
  return p;
}

// item 1: SampleLevel(sampler, (u, v), 0).rgb of a W x H float4 plane; border = ClampToBorder with transparent black, else ClampToEdge
OXC_DI Vec3 bloom_tap(const float4* src, int W, int H, float u, float v, bool border) {
  const float x = fs(fm(u, (float)W), 0.5f), y = fs(fm(v, (float)H), 0.5f);
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = fs(x, x0), wy = fs(y, y0);
  const long long ix = sat_i32(x0), iy = sat_i32(y0);
  float4 q[4];
  for (int k = 0; k < 4; k++) {
    const long long xi = ix + (k & 1), yi = iy + (k >> 1);
    if (border && (xi < 0 || xi >= W || yi < 0 || yi >= H)) q[k] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    else q[k] = src[(size_t)clamp_index(yi, H) * W + clamp_index(xi, W)];
  }
  const float a00[3] = {q[0].x, q[0].y, q[0].z}, a10[3] = {q[1].x, q[1].y, q[1].z};
  const float a01[3] = {q[2].x, q[2].y, q[2].z}, a11[3] = {q[3].x, q[3].y, q[3].z};
  float out[3];
  for (int c = 0; c < 3; c++) {
    const float top = fa(a00[c], fm(wx, fs(a10[c], a00[c]))), bot = fa(a01[c], fm(wx, fs(a11[c], a01[c])));
    out[c] = fa(top, fm(wy, fs(bot, top)));
  }
  return vec3(out[0], out[1], out[2]);
}

// item 2: the tap at uv + texel_size * (dx, dy)
struct BloomCoord {
  float u, v, tu, tv;
};
OXC_DI BloomCoord bloom_coord(int x, int y, int w, int h) {
  return BloomCoord{fd(fa((float)x, 0.5f), (float)w), fd(fa((float)y, 0.5f), (float)h), fd(1.0f, (float)w), fd(1.0f, (float)h)};
}
OXC_DI Vec3 bloom_tap_at(const float4* src, int W, int H, const BloomCoord& c, float dx, float dy, bool border) {
  return bloom_tap(src, W, H, fa(c.u, fm(c.tu, dx)), fa(c.v, fm(c.tv, dy)), border);
}

OXC_DI void bloom_store(float4* dst, Vec3 v) { *dst = make_float4(nan_canonical(v.x), nan_canonical(v.y), nan_canonical(v.z), 1.0f); }

// ((a + b) + c) + d per component
OXC_DI Vec3 bloom_sum4(Vec3 a, Vec3 b, Vec3 c, Vec3 d) { return vadd(vadd(vadd(a, b), c), d); }

// the 13 taps of the prefilter and the downsample: a..i at offsets -2, 0, 2, j..m at -1, 1 (y up first, as the shaders list them)
struct BloomTaps13 {
  Vec3 a, b, c, d, e, f, g, h, i, j, k, l, m;
};
OXC_DI BloomTaps13 bloom_taps13(const float4* src, int W, int H, const BloomCoord& c) {
  BloomTaps13 t;
  t.a = bloom_tap_at(src, W, H, c, -2.0f, 2.0f, true);
  t.b = bloom_tap_at(src, W, H, c, 0.0f, 2.0f, true);
  t.c = bloom_tap_at(src, W, H, c, 2.0f, 2.0f, true);
  t.d = bloom_tap_at(src, W, H, c, -2.0f, 0.0f, true);
  t.e = bloom_tap_at(src, W, H, c, 0.0f, 0.0f, true);
  t.f = bloom_tap_at(src, W, H, c, 2.0f, 0.0f, true);
  t.g = bloom_tap_at(src, W, H, c, -2.0f, -2.0f, true);
  t.h = bloom_tap_at(src, W, H, c, 0.0f, -2.0f, true);
  t.i = bloom_tap_at(src, W, H, c, 2.0f, -2.0f, true);
  t.j = bloom_tap_at(src, W, H, c, -1.0f, 1.0f, true);
  t.k = bloom_tap_at(src, W, H, c, 1.0f, 1.0f, true);
  t.l = bloom_tap_at(src, W, H, c, -1.0f, -1.0f, true);
  t.m = bloom_tap_at(src, W, H, c, 1.0f, -1.0f, true);
  return t;
}

// item 3: one group's contribution to color_sum and weight_sum
OXC_DI void bloom_group(const BloomParams& p, Vec3 g, float exposure, Vec3& color_sum, float& weight_sum) {
  g = vscale(vscale(g, 0.25f), exposure);
  g = vec3(vmin(g.x, p.clamp_value), vmin(g.y, p.clamp_value), vmin(g.z, p.clamp_value));
  const float weight = fd(1.0f, fa(1.0f, dot3(g.x, g.y, g.z, BLOOM_LUM_R, BLOOM_LUM_G, BLOOM_LUM_B)));
  const float brightness = vmax(g.x, vmax(g.y, g.z));
  const float knee = fm(p.threshold, p.soft_threshold);
  float soft = fa(fs(brightness, p.threshold), knee);
  soft = vmin(vmax(soft, 0.0f), fm(2.0f, knee));
  soft = fd(fm(fm(soft, soft), 0.25f), fa(knee, BLOOM_EPS));
  const float contribution = fd(vmax(soft, fs(brightness, p.threshold)), vmax(brightness, BLOOM_EPS));
  color_sum = vadd(color_sum, vscale(vscale(g, contribution), weight));
  weight_sum = fa(weight_sum, weight);
}

// item 3: texel (x, y) of downsampled level 0
OXC_DI void bloom_prefilter_texel(const BloomParams& p, int x, int y) {
  const BloomCoord c = bloom_coord(x, y, p.w[0], p.h[0]);
  const BloomTaps13 t = bloom_taps13(p.frame, p.frame_w, p.frame_h, c);
  const float exposure = p.record ? p.record->exposure : 1.0f;
  Vec3 color_sum = vec3(0.0f, 0.0f, 0.0f);
  float weight_sum = 0.0f;
  bloom_group(p, bloom_sum4(t.a, t.b, t.d, t.e), exposure, color_sum, weight_sum);
  bloom_group(p, bloom_sum4(t.b, t.c, t.e, t.f), exposure, color_sum, weight_sum);
  bloom_group(p, bloom_sum4(t.d, t.e, t.g, t.h), exposure, color_sum, weight_sum);
  bloom_group(p, bloom_sum4(t.e, t.f, t.h, t.i), exposure, color_sum, weight_sum);
  bloom_group(p, bloom_sum4(t.j, t.k, t.l, t.m), exposure, color_sum, weight_sum);
  bloom_store(p.down + (size_t)y * p.w[0] + x, vdiv(color_sum, fa(weight_sum, BLOOM_EPS)));
}

// item 4: texel (x, y) of downsampled level i >= 1, from level i - 1
OXC_DI void bloom_downsample_texel(const BloomParams& p, int i, int x, int y) {
  const BloomCoord c = bloom_coord(x, y, p.w[i], p.h[i]);
  const BloomTaps13 t = bloom_taps13(p.down + p.offset[i - 1], p.w[i - 1], p.h[i - 1], c);
  const Vec3 r = vadd(vadd(vscale(bloom_sum4(t.a, t.c, t.g, t.i), 0.03125f), vscale(bloom_sum4(t.b, t.d, t.f, t.h), 0.0625f)),
                      vscale(vadd(bloom_sum4(t.e, t.j, t.k, t.l), t.m), 0.125f));
  bloom_store(p.down + p.offset[i] + (size_t)y * p.w[i] + x, r);
}

// item 5: texel (x, y) of upsampled level i - 1, i in 1..n-1
OXC_DI void bloom_upsample_texel(const BloomParams& p, int i, int x, int y) {
  const int d = i - 1;
  const BloomCoord c = bloom_coord(x, y, p.w[d], p.h[d]);
  const float4* src = (i == p.levels - 1 ? p.down : p.up) + p.offset[i];
  const int W = p.w[i], H = p.h[i];
  const Vec3 a = bloom_tap_at(src, W, H, c, -1.0f, 1.0f, false), b = bloom_tap_at(src, W, H, c, 0.0f, 1.0f, false);
  const Vec3 cc = bloom_tap_at(src, W, H, c, 1.0f, 1.0f, false), dd = bloom_tap_at(src, W, H, c, -1.0f, 0.0f, false);
  const Vec3 e = bloom_tap_at(src, W, H, c, 0.0f, 0.0f, false), f = bloom_tap_at(src, W, H, c, 1.0f, 0.0f, false);
  const Vec3 g = bloom_tap_at(src, W, H, c, -1.0f, -1.0f, false), h = bloom_tap_at(src, W, H, c, 0.0f, -1.0f, false);
  const Vec3 ii = bloom_tap_at(src, W, H, c, 1.0f, -1.0f, false);
  const Vec3 sum = vadd(vadd(vscale(e, 0.25f), vscale(bloom_sum4(b, dd, f, h), 0.125f)), vscale(bloom_sum4(a, cc, g, ii), 0.0625f));
  const Vec3 s = bloom_tap(p.down + p.offset[d], p.w[d], p.h[d], c.u, c.v, false);
  bloom_store(p.up + p.offset[d] + (size_t)y * p.w[d] + x, vadd(s, vscale(vsub(sum, s), p.radius)));
}

// item 6: a single-level chain's output, the reference's per-frame clear
OXC_DI void bloom_black_texel(const BloomParams& p, int x, int y) {
  p.up[(size_t)y * p.w[0] + x] = make_float4(0.0f, 0.0f, 0.0f, 1.0f);
}

} // namespace oxc
