// oxc_tonemap.cuh — the tonemap pass (PostProcess.cpp:205-247, passes/tonemap.slang fs_main, passes/lens.slang): the value of one output
// pixel, as include/oxcull.h oxc_tonemap specifies it (items 1-10) and oracle/oxc_oracle_tonemap.c computes it.  kernels_tonemap.cuh
// lays the pixels out.  The constants that do not depend on the call (item 9) are kept here as hex; tests recompute them.
// No warp intrinsics, no shared memory: tests compile this source for the host.
#pragma once
#include "oxc_shader_math.cuh"

namespace oxc {

// item 9, formed once in binary32 in shader order (oracle/oxc_oracle_tonemap.c orc_tonemap_constants; tests/test_oracle_tonemap.py
// recomputes them); kept in the kernel parameters, so every thread reads them from the constant bank
struct TonemapConstants {
  float agx[9];     // AgX_DS sRGB_to_adjusted = mul(sRGB_to_XYZ, XYZ_to_adjusted), row-major
  float agx_inv[9]; // inverse(sRGB_to_adjusted)
  float agx_s, agx_c, agx_peak_s;                     // color_DualSection(x, 0.1, 1): S, C = peak / (peak - S), peak - S
  float gt7_ka, gt7_kb, gt7_kc, gt7_linear_peak;      // GTToneMappingCurveV2::initializeCurve(2.5, 0.25, 0.538, 0.444, 1.280)
  float gt7_target, gt7_target_ucs, gt7_sdr, gt7_one_minus_blend; // GT7ToneMapping::initializeAsSDR
  float pq_inv_m1, pq_inv_m2;                         // eotfSt2084's 1 / m1, 1 / m2
  float simplex_f2, simplex_g2;                       // lens.slang simplex: (sqrt(3) - 1) / 2, (3 - sqrt(3)) / 6
};

inline TonemapConstants tonemap_constants() {
  return TonemapConstants{
      {0x1.cb371ep-1f, 0x1.803f0ep-5f, 0x1.803ef8p-5f, 0x1.944652p-5f, 0x1.cc77ap-1f, 0x1.944672p-5f, 0x1.b8475cp-5f, 0x1.b84774p-5f,
       0x1.ceb7aep-1f},
      {0x1.1f0cc2p+0f, -0x1.c40dfp-5f, -0x1.c40dd8p-5f, -0x1.db9e04p-5f, 0x1.1e5038p+0f, -0x1.db9e22p-5f, -0x1.02fcccp-4f, -0x1.02fcd4p-4f,
       0x1.1cfd5ep+0f},
      0x1.99999ap-4f,  // 0.1, 0x3DCCCCCD
      0x1.1c71c8p+0f,  // 0x3F8E38E4
      0x1.ccccccp-1f,  // 0x3F666666
      0x1.7b4e8p+1f,   // kA 0x403DA740
      -0x1.afc9f8p+1f, // kB 0xC057E4FC
      -0x1.14424ep-1f, // kC 0xBF0A2127
      0x1.1c28f6p+0f,  // 1.11, 0x3F8E147B
      0x1.4p+1f,       // 2.5
      0x1.3482d8p-1f,  // 0x3F1A416C
      0x1.99999ap-2f,  // 0.4, 0x3ECCCCCD
      0x1.999998p-2f,  // 1 - 0.6, 0x3ECCCCCC
      0x1.91c0d6p+2f,  // 0x40C8E06B
      0x1.9f9b58p-7f,  // 0x3C4FCDAC
      0x1.76cf5cp-2f,  // 0x3EBB67AE
      0x1.b0cb18p-3f,  // 0x3E58658C
  };
}

struct TonemapParams {
  const float4* frame;
  const float4* bloom;        // read under HasBloom only, else nullptr
  const OxcExposure* record;  // read under HasEyeAdaptation only, else nullptr
  float4* out;
  int width, height, bloom_w, bloom_h, cx, cy; // cx, cy = screen_size / 2
  uint32_t flags;
  float exposure, bloom_intensity, vignette_amount, grain_scale, grain_amount;
  uint32_t grain_seed;
  int grain_divisor;          // item 6: sat_i32(scale / 8)
  float red_mag, green_mag;   // item 4: FfxLensGetRGMag(amount)
  float rcp_x, rcp_y;         // item 4: 1 / f32(2 * c)
  TonemapConstants k;
};

// item 4: FfxLensGetRGMag, once per call on the host
inline void tonemap_rg_mag(float amount, float& red, float& green) {
  const float A = 1.5220f, B = hd_mul(0.00459f, amount);
  const float ri = hd_add(A, B / hd_mul(0.612f, 0.612f)), gi = hd_add(A, B / hd_mul(0.549f, 0.549f)), bi = hd_add(A, B / hd_mul(0.464f, 0.464f));
  red = hd_sub(ri, 1.0f) / hd_sub(bi, 1.0f);
  green = hd_sub(gi, 1.0f) / hd_sub(bi, 1.0f);
}

// the per-call values, formed once on the host (the ABI and tests/tonemap_vs_oracle.cpp call it)
inline TonemapParams tonemap_make_params(const float* frame, uint32_t width, uint32_t height, const OxcTonemapSettings& s,
                                         const OxcExposure* record, const float* bloom, float* out) {
  TonemapParams p;
  p.frame = reinterpret_cast<const float4*>(frame);
  p.flags = s.scene_flags;
  p.bloom = (s.scene_flags & OXC_SCENE_HAS_BLOOM) ? reinterpret_cast<const float4*>(bloom) : nullptr;
  p.record = (s.scene_flags & OXC_SCENE_HAS_EYE_ADAPTATION) ? record : nullptr;
  p.out = reinterpret_cast<float4*>(out);
  p.width = (int)width;
  p.height = (int)height;
  p.bloom_w = (int)(width / 2u);
  p.bloom_h = (int)(height / 2u);
  p.cx = p.width / 2;
  p.cy = p.height / 2;
  p.exposure = s.exposure;
  p.bloom_intensity = s.bloom_intensity;
  p.vignette_amount = s.vignette_amount;
  p.grain_scale = s.film_grain_scale;
  p.grain_amount = s.film_grain_amount;
  p.grain_seed = s.film_grain_seed;
  const float q = s.film_grain_scale / 8.0f; // one IEEE division in the host build; then sat_i32's rule
  p.grain_divisor = !(q == q) ? 0 : (q >= 2147483648.0f ? INT_MAX : (q <= -2147483648.0f ? INT_MIN : (int)q));
  tonemap_rg_mag(s.chromatic_aberration_amount, p.red_mag, p.green_mag);
  p.rcp_x = 1.0f / (float)(2 * p.cx);
  p.rcp_y = 1.0f / (float)(2 * p.cy);
  p.k = tonemap_constants();
  return p;
}

// mul(M, v) of a row-major 3 x 3: row . v
OXC_DI Vec3 mat_vec(const float* m, Vec3 c) { return vec3(vdot(vec3(m[0], m[1], m[2]), c), vdot(vec3(m[3], m[4], m[5]), c), vdot(vec3(m[6], m[7], m[8]), c)); }
OXC_DI float clamp01(float x) { return vmin(vmax(x, 0.0f), 1.0f); }

// ---------------------------------------------------------------- item 3: the curves

OXC_DI float aces_fit(float v) { // RRTAndODTFit
  const float a = fs(fm(v, fa(v, 0.0245786f)), 0.000090537f);
  const float b = fa(fm(v, fa(fm(0.983729f, v), 0.4329510f)), 0.238081f);
  return fd(a, b);
}
OXC_DI Vec3 aces_fitted(Vec3 c) {
  constexpr float IN0 = 0.59719f, IN1 = 0.35458f, IN2 = 0.04823f, IN3 = 0.07600f, IN4 = 0.90834f, IN5 = 0.01566f, IN6 = 0.02840f,
                  IN7 = 0.13383f, IN8 = 0.83777f;
  constexpr float OUT0 = 1.60475f, OUT1 = -0.53108f, OUT2 = -0.07367f, OUT3 = -0.10208f, OUT4 = 1.10813f, OUT5 = -0.00605f,
                  OUT6 = -0.00327f, OUT7 = -0.07276f, OUT8 = 1.07602f;
  const float in[9] = {IN0, IN1, IN2, IN3, IN4, IN5, IN6, IN7, IN8}, out[9] = {OUT0, OUT1, OUT2, OUT3, OUT4, OUT5, OUT6, OUT7, OUT8};
  c = mat_vec(in, c);
  c = mat_vec(out, vec3(aces_fit(c.x), aces_fit(c.y), aces_fit(c.z)));
  return vec3(saturate(c.x), saturate(c.y), saturate(c.z));
}

OXC_DI float agx_dual_section(const TonemapConstants& k, float x) {
  return clamp01(x < k.agx_s ? x : fs(1.0f, fm(k.agx_peak_s, canonical_exp(fd(fm(-k.agx_c, fs(x, k.agx_s)), 1.0f)))));
}
OXC_DI Vec3 agx_ds(const TonemapConstants& k, Vec3 c) {
  c = mat_vec(k.agx, vec3(vmax(c.x, 0.0f), vmax(c.y, 0.0f), vmax(c.z, 0.0f)));
  c = vec3(agx_dual_section(k, c.x), agx_dual_section(k, c.y), agx_dual_section(k, c.z));
  const float d = vdot(c, vec3(0.2126729f, 0.7151522f, 0.0721750f));
  c = vec3(clamp01(fa(d, fm(fs(c.x, d), 1.3f))), clamp01(fa(d, fm(fs(c.y, d), 1.3f))), clamp01(fa(d, fm(fs(c.z, d), 1.3f))));
  return mat_vec(k.agx_inv, c);
}

OXC_DI float gt7_smooth_step(float x, float e0, float e1) {
  const float t = fd(fs(x, e0), fs(e1, e0));
  if (x < e0) return 0.0f;
  if (x > e1) return 1.0f;
  return fm(fm(t, t), fs(3.0f, fm(2.0f, t)));
}
OXC_DI float gt7_curve(const TonemapConstants& k, float x) { // GTToneMappingCurveV2::evaluateCurve
  constexpr float MID = 0.538f, TOE = 1.280f;
  if (x < 0.0f) return 0.0f;
  const float wl = gt7_smooth_step(x, 0.0f, MID);
  if (x < k.gt7_linear_peak) return fa(fm(fs(1.0f, wl), fm(MID, canonical_pow(fd(x, MID), TOE))), fm(wl, x));
  return fa(k.gt7_ka, fm(k.gt7_kb, canonical_exp(fm(x, k.gt7_kc))));
}
OXC_DI float pq_inverse_eotf(float v) { // inverseEotfSt2084(v, 1)
  const float y = fd(fm(v, 100.0f), 10000.0f);
  const float ym = canonical_pow(y, 0.1593017578125f);
  return canonical_pow(2.0f, fm(78.84375f, fs(canonical_log2(fa(0.8359375f, fm(18.8515625f, ym))), canonical_log2(fa(1.0f, fm(18.6875f, ym))))));
}
OXC_DI float pq_eotf(const TonemapConstants& k, float n) { // eotfSt2084(n, 1)
  if (n < 0.0f) n = 0.0f;
  if (n > 1.0f) n = 1.0f;
  const float np = canonical_pow(n, k.pq_inv_m2);
  float l = fs(np, 0.8359375f);
  if (l < 0.0f) l = 0.0f;
  l = fd(l, fs(18.8515625f, fm(18.6875f, np)));
  return fd(fm(canonical_pow(l, k.pq_inv_m1), 10000.0f), 100.0f);
}
OXC_DI Vec3 rgb_to_ictcp(Vec3 c) {
  const float l = fd(fa(fa(fm(c.x, 1688.0f), fm(c.y, 2146.0f)), fm(c.z, 262.0f)), 4096.0f);
  const float m = fd(fa(fa(fm(c.x, 683.0f), fm(c.y, 2951.0f)), fm(c.z, 462.0f)), 4096.0f);
  const float s = fd(fa(fa(fm(c.x, 99.0f), fm(c.y, 309.0f)), fm(c.z, 3688.0f)), 4096.0f);
  const float L = pq_inverse_eotf(l), M = pq_inverse_eotf(m), S = pq_inverse_eotf(s);
  return vec3(fd(fa(fm(2048.0f, L), fm(2048.0f, M)), 4096.0f), fd(fa(fs(fm(6610.0f, L), fm(13613.0f, M)), fm(7003.0f, S)), 4096.0f),
              fd(fs(fs(fm(17933.0f, L), fm(17390.0f, M)), fm(543.0f, S)), 4096.0f));
}
OXC_DI Vec3 ictcp_to_rgb(const TonemapConstants& k, Vec3 u) {
  const float L = pq_eotf(k, fa(fa(u.x, fm(0.00860904f, u.y)), fm(0.11103f, u.z)));
  const float M = pq_eotf(k, fs(fs(u.x, fm(0.00860904f, u.y)), fm(0.11103f, u.z)));
  const float S = pq_eotf(k, fs(fa(u.x, fm(0.560031f, u.y)), fm(0.320627f, u.z)));
  return vec3(vmax(fa(fs(fm(3.43661f, L), fm(2.50645f, M)), fm(0.0698454f, S)), 0.0f),
              vmax(fs(fa(fm(-0.79133f, L), fm(1.9836f, M)), fm(0.192271f, S)), 0.0f),
              vmax(fa(fs(fm(-0.0259499f, L), fm(0.0989137f, M)), fm(1.12486f, S)), 0.0f));
}
// GT7ToneMapping::applyToneMapping on linear Rec.2020, after initializeAsSDR
OXC_DI Vec3 gt7_rec2020(const TonemapConstants& k, Vec3 rgb) {
  const Vec3 ucs = rgb_to_ictcp(rgb);
  const Vec3 skewed = vec3(gt7_curve(k, rgb.x), gt7_curve(k, rgb.y), gt7_curve(k, rgb.z));
  const Vec3 skewed_ucs = rgb_to_ictcp(skewed);
  const float chroma = fs(1.0f, gt7_smooth_step(fd(ucs.x, k.gt7_target_ucs), 0.98f, 1.16f));
  const Vec3 scaled = ictcp_to_rgb(k, vec3(skewed_ucs.x, fm(ucs.y, chroma), fm(ucs.z, chroma)));
  return vec3(fm(k.gt7_sdr, vmin(fa(fm(k.gt7_one_minus_blend, skewed.x), fm(0.6f, scaled.x)), k.gt7_target)),
              fm(k.gt7_sdr, vmin(fa(fm(k.gt7_one_minus_blend, skewed.y), fm(0.6f, scaled.y)), k.gt7_target)),
              fm(k.gt7_sdr, vmin(fa(fm(k.gt7_one_minus_blend, skewed.z), fm(0.6f, scaled.z)), k.gt7_target)));
}
OXC_DI Vec3 gt7(const TonemapConstants& k, Vec3 c) {
  const float to_xyz[9] = {0.4124564f, 0.3575761f, 0.1804375f, 0.2126729f, 0.7151522f, 0.0721750f, 0.0193339f, 0.1191920f, 0.9503041f};
  const float xyz_to_2020[9] = {1.7166512f, -0.3556708f, -0.2533663f, -0.6666844f, 1.6164812f, 0.0157685f, 0.0176399f, -0.0427706f, 0.9421031f};
  const float from_2020[9] = {0.636958f, 0.1446169f, 0.168881f, 0.2627002f, 0.6779981f, 0.0593017f, 0.0f, 0.0280727f, 1.0609851f};
  const float xyz_to_709[9] = {3.2404542f, -1.5371385f, -0.4985314f, -0.9692660f, 1.8760108f, 0.0415560f, 0.0556434f, -0.2040259f, 1.0572252f};
  const Vec3 o = gt7_rec2020(k, mat_vec(xyz_to_2020, mat_vec(to_xyz, c)));
  return mat_vec(xyz_to_709, mat_vec(from_2020, o));
}

template <uint32_t TYPE>
OXC_DI Vec3 tonemap_curve(const TonemapConstants& k, Vec3 c) {
  if (TYPE == OXC_TONEMAP_ACES) return aces_fitted(c);
  if (TYPE == OXC_TONEMAP_AGX) return agx_ds(k, c);
  if (TYPE == OXC_TONEMAP_GT7) return gt7(k, c);
  return c;
}

// ---------------------------------------------------------------- items 4-6: lens.slang

OXC_DI void tonemap_vignette(const TonemapParams& p, int x, int y, Vec3& c) {
  constexpr float PI_OVER_4 = 0x1.921fb6p-1f; // fl(PI * 0.25), 0x3F490FDB
  const float fx = fd((float)(x > p.cx ? x - p.cx : p.cx - x), (float)p.cx), fy = fd((float)(y > p.cy ? y - p.cy : p.cy - y), (float)p.cy);
  float mx = canonical_cos(fm(fm(fx, p.vignette_amount), PI_OVER_4)), my = canonical_cos(fm(fm(fy, p.vignette_amount), PI_OVER_4));
  mx = fm(mx, mx);
  my = fm(my, my);
  mx = fm(mx, mx);
  my = fm(my, my);
  c = vscale(c, clamp01(fm(mx, my)));
}

OXC_DI void tonemap_film_grain(const TonemapParams& p, int x, int y, Vec3& c) {
  const int d = p.grain_divisor;
  uint32_t v0 = d == 0 ? 0xFFFFFFFFu : (uint32_t)(x / d), v1 = d == 0 ? 0xFFFFFFFFu : (uint32_t)(y / d), v2 = p.grain_seed;
  v0 = v0 * 12829u + 47989u;
  v1 = v1 * 12829u + 47989u;
  v2 = v2 * 12829u + 47989u;
  for (int r = 0; r < 2; r++) {
    v0 += v1 * v2;
    v1 += v2 * v0;
    v2 += v0 * v1;
  }
  const float rx = fs(fm((float)(v0 >> 16), 0x1.0p-16f), 0.5f), ry = fs(fm((float)(v1 >> 16), 0x1.0p-16f), 0.5f);
  const float px = fa(fd((float)x, p.grain_scale), rx), py = fa(fd((float)y, p.grain_scale), ry);
  const float u = fm(fa(px, py), p.k.simplex_f2);
  const float ix = rintf(fa(px, u)), iy = rintf(fa(py, u));
  const float w = fm(fa(ix, iy), p.k.simplex_g2);
  const float fx = fs(px, fs(ix, w)), fy = fs(py, fs(iy, w));
  const float len = fsq(fa(fm(fx, fx), fm(fy, fy)));
  const float grain = fs(1.0f, fm(2.0f, canonical_pow(2.0f, fm(-len, 3.0f))));
  c = vec3(fa(c.x, fm(fm(grain, vmin(c.x, fs(1.0f, c.x))), p.grain_amount)), fa(c.y, fm(fm(grain, vmin(c.y, fs(1.0f, c.y))), p.grain_amount)),
           fa(c.z, fm(fm(grain, vmin(c.z, fs(1.0f, c.z))), p.grain_amount)));
}

// ---------------------------------------------------------------- the pixel

template <uint32_t TYPE>
OXC_DI float4 tonemap_pixel(const TonemapParams& p, int x, int y) {
  const float u = fd(fa((float)x, 0.5f), (float)p.width), v = fd(fa((float)y, 0.5f), (float)p.height);
  const float4 src = bilinear_tap<REPEAT>(p.frame, p.width, p.height, u, v);
  Vec3 c;
  if (p.flags & OXC_SCENE_HAS_CHROMATIC_ABERRATION) {
    // item 4: the colour is replaced, so exposure, bloom and curve are not computed
    const float dx = (float)(x - p.cx), dy = (float)(y - p.cy), cx = (float)p.cx, cy = (float)p.cy;
    c.x = bilinear_tap<REPEAT>(p.frame, p.width, p.height, fm(fa(fa(fm(dx, p.red_mag), cx), 0.5f), p.rcp_x), fm(fa(fa(fm(dy, p.red_mag), cy), 0.5f), p.rcp_y)).x;
    c.y = bilinear_tap<REPEAT>(p.frame, p.width, p.height, fm(fa(fa(fm(dx, p.green_mag), cx), 0.5f), p.rcp_x), fm(fa(fa(fm(dy, p.green_mag), cy), 0.5f), p.rcp_y)).y;
    c.z = bilinear_tap<REPEAT>(p.frame, p.width, p.height, fm((float)x, p.rcp_x), fm((float)y, p.rcp_y)).z;
  } else {
    c = vscale(vec3(src.x, src.y, src.z), p.record ? p.record->exposure : p.exposure);
    if (p.bloom) {
      const float4 b = bilinear_tap<REPEAT>(p.bloom, p.bloom_w, p.bloom_h, u, v);
      c = vadd(c, vscale(vec3(b.x, b.y, b.z), p.bloom_intensity));
    }
    c = tonemap_curve<TYPE>(p.k, c);
  }
  if (p.flags & OXC_SCENE_HAS_VIGNETTE) tonemap_vignette(p, x, y, c);
  if (p.flags & OXC_SCENE_HAS_FILM_GRAIN) tonemap_film_grain(p, x, y, c);
  return make_float4(nan_canonical(c.x), nan_canonical(c.y), nan_canonical(c.z),
                     nan_canonical((p.flags & OXC_SCENE_TRANSPARENT_BACKGROUND) ? src.w : 1.0f));
}

} // namespace oxc
