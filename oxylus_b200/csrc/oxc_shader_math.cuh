// oxc_shader_math.cuh — the HLSL-semantics primitives the screen-space passes' per-pixel headers share: max / min / saturate / sign /
// frac with the shaders' NaN rules, the saturating float -> integer conversions, the address modes and the bilinear taps (float4 and R16) of
// the software taps, the binary16 conversions of the planes the passes store, pi, and one 3-vector with the canonical operation order.  Each states its NaN and
// rounding rule once, so every pass that calls it gives the same bits.
// No warp intrinsics, no shared memory: tests compile this source for the host.
#pragma once
#include <climits>

#include "oxc_exact.cuh"

namespace oxc {

constexpr float PI = 0x1.921fb6p+1f; // 0x40490FDB, common/math.slang:4

// HLSL max / min with IEEE maxNum / minNum NaN handling (a NaN operand yields the other one); equal operands yield b
OXC_HD float vmax(float a, float b) { return (b != b || a > b) ? a : b; }
OXC_HD float vmin(float a, float b) { return (b != b || a < b) ? a : b; }
OXC_HD float saturate(float x) { return vmin(vmax(x, 0.0f), 1.0f); } // NaN -> 0
OXC_DI float sign(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); } // NaN -> 0
OXC_DI float frac(float x) { return fs(x, floorf(x)); } // x - floor(x)

// float -> i32, truncating, saturating, NaN -> 0 (cvt.rzi.s32.f32; the host build and the device agree for every input)
OXC_DI int sat_i32(float f) { return !(f == f) ? 0 : (f >= 2147483648.0f ? INT_MAX : (f <= -2147483648.0f ? INT_MIN : (int)f)); }
// float -> u32, truncating, saturating, NaN -> 0
OXC_DI uint32_t sat_u32(float f) { return !(f > 0.0f) ? 0u : (f >= 4294967296.0f ? 0xFFFFFFFFu : (uint32_t)f); }
// a texel index clamped to the edge of an extent n >= 1
OXC_DI int clamp_index(long long i, int n) { return (int)(i < 0 ? 0 : (i > n - 1 ? n - 1 : i)); }
// a texel index wrapped into an extent n >= 1 (the Repeat address mode); an index already inside skips the division
OXC_DI int wrap_index(long long i, int n) {
  if (i >= 0 && i < n) return (int)i;
  const long long r = i % n;
  return (int)(r < 0 ? r + n : r);
}

// the texel index rule of a sampler's address mode: ClampToEdge (clamp_index) or Repeat (wrap_index)
enum AddressMode { CLAMP_TO_EDGE, REPEAT };
template <AddressMode MODE>
OXC_DI int address_index(long long i, int n) { return MODE == REPEAT ? wrap_index(i, n) : clamp_index(i, n); }

// the bilinear blend a + w * (b - a) of one channel, and of four
OXC_DI float tap_lerp(float a, float b, float w) { return fa(a, fm(w, fs(b, a))); }
OXC_DI float4 tap_lerp(float4 a, float4 b, float w) {
  return make_float4(tap_lerp(a.x, b.x, w), tap_lerp(a.y, b.y, w), tap_lerp(a.z, b.z, w), tap_lerp(a.w, b.w, w));
}

// the bilinear tap of a W x H plane at the unnormalised, half-texel-shifted coordinate (x, y): oxc_bloom item 1's rule, x0 = floor(x),
// wx = x - x0, texels x0, x0 + 1 / y0, y0 + 1 through the address mode, top = a00 + wx * (a10 - a00), bottom likewise,
// top + wy * (bottom - top).  NaN-safe: the floor goes through sat_i32 and a NaN coordinate gives NaN weights.  fetch(i) returns
// texel i (row-major) as a float or a float4.
template <AddressMode MODE, class Fetch>
OXC_DI auto bilinear_fetch(Fetch fetch, int W, int H, float x, float y) -> decltype(fetch(size_t(0))) {
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = fs(x, x0), wy = fs(y, y0);
  const long long ix = sat_i32(x0), iy = sat_i32(y0);
  const int c0 = address_index<MODE>(ix, W), c1 = address_index<MODE>(ix + 1, W);
  const size_t r0 = (size_t)address_index<MODE>(iy, H) * W, r1 = (size_t)address_index<MODE>(iy + 1, H) * W;
  const auto a00 = fetch(r0 + c0), a10 = fetch(r0 + c1), a01 = fetch(r1 + c0), a11 = fetch(r1 + c1);
  return tap_lerp(tap_lerp(a00, a10, wx), tap_lerp(a01, a11, wx), wy);
}
// the four-channel tap of a float4 plane
template <AddressMode MODE>
OXC_DI float4 bilinear_at(const float4* src, int W, int H, float x, float y) {
  return bilinear_fetch<MODE>([src](size_t i) { return src[i]; }, W, H, x, y);
}
// Sample / SampleLevel(uv) at level 0: x = u * W - 0.5 (y likewise)
template <AddressMode MODE>
OXC_DI float4 bilinear_tap(const float4* src, int W, int H, float u, float v) {
  return bilinear_at<MODE>(src, W, H, fs(fm(u, (float)W), 0.5f), fs(fm(v, (float)H), 0.5f));
}
// Sample(uv, int2(dx, dy)): the constant texel offset joins the unnormalised coordinate before the half-texel shift (Vulkan's
// order), x = (u * W + dx) - 0.5
template <AddressMode MODE>
OXC_DI float4 bilinear_tap(const float4* src, int W, int H, float u, float v, int dx, int dy) {
  return bilinear_at<MODE>(src, W, H, fs(fa(fm(u, (float)W), (float)dx), 0.5f), fs(fa(fm(v, (float)H), (float)dy), 0.5f));
}
// the one-channel sibling of bilinear_tap for an R16Unorm plane: SampleLevel(uv, 0) with texel t read as t / 65535 in binary32
template <AddressMode MODE>
OXC_DI float bilinear_tap_r16(const uint16_t* src, int W, int H, float u, float v) {
  return bilinear_fetch<MODE>([src](size_t i) { return fd((float)src[i], 65535.0f); }, W, H, fs(fm(u, (float)W), 0.5f),
                              fs(fm(v, (float)H), 0.5f));
}

// the blend of two mip levels' values: (1 - f) * lo + f * hi
OXC_DI float lerp_levels(float f, float lo, float hi) { return fa(fm(fs(1.0f, f), lo), fm(f, hi)); }
OXC_DI float4 lerp_levels(float f, float4 lo, float4 hi) {
  return make_float4(lerp_levels(f, lo.x, hi.x), lerp_levels(f, lo.y, hi.y), lerp_levels(f, lo.z, hi.z), lerp_levels(f, lo.w, hi.w));
}

// binary32 -> binary16 with round-to-nearest-even -> binary32 (the R16G16B16A16Sfloat normal attachment); NaN stays NaN
OXC_DI float round_to_half(float f) {
#ifdef __CUDA_ARCH__
  return __half2float(__float2half_rn(f));
#else
  const uint32_t u = __float_as_uint(f), sign = u & 0x80000000u, a = u & 0x7FFFFFFFu;
  if (a >= 0x7F800000u) return f;                                        // inf, NaN
  if (a >= 0x38800000u) {                                                // half normal range: keep 10 fraction bits
    const uint32_t r = (a + 0xFFFu + ((a >> 13) & 1u)) & ~0x1FFFu;
    return __uint_as_float(sign | (r > 0x477FE000u ? 0x7F800000u : r)); // above 65504: inf
  }
  const float m = rintf(__uint_as_float(a) * 16777216.0f);             // half subnormals: multiples of 2^-24
  return __uint_as_float(sign | __float_as_uint(m * 5.9604644775390625e-08f));
#endif
}

// binary32 -> binary16 bits, round to nearest even
OXC_DI uint16_t half_bits(float f) {
#ifdef __CUDA_ARCH__
  return __half_as_ushort(__float2half_rn(f));
#else
  const float r = round_to_half(f);
  const uint32_t u = __float_as_uint(r), s = (u >> 16) & 0x8000u, a = u & 0x7FFFFFFFu;
  if (a > 0x7F800000u) return (uint16_t)(s | 0x7FFFu);
  if (a == 0x7F800000u) return (uint16_t)(s | 0x7C00u);
  if (a >= 0x38800000u) return (uint16_t)(s | (((a >> 23) - 112u) << 10) | ((a >> 13) & 0x3FFu));
  return (uint16_t)(s | (uint32_t)fm(__uint_as_float(a), 16777216.0f));
#endif
}
OXC_DI float half_float(uint16_t h) { return __half2float(__ushort_as_half(h)); }

// the value a binary32 plane is stored as: a NaN is written as 0x7FFFFFFF, the NaN the GPU's arithmetic produces (the host's differs)
OXC_DI float nan_canonical(float v) { return v != v ? __uint_as_float(0x7FFFFFFFu) : v; }

// a 3-vector; every operation rounds each component once, dot is (a.x * b.x + a.y * b.y) + a.z * b.z
struct Vec3 {
  float x, y, z;
};
OXC_DI Vec3 vec3(float x, float y, float z) { return Vec3{x, y, z}; }
OXC_DI float vdot(Vec3 a, Vec3 b) { return dot3(a.x, a.y, a.z, b.x, b.y, b.z); }
OXC_DI float vlength(Vec3 a) { return fsq(vdot(a, a)); }
OXC_DI Vec3 vadd(Vec3 a, Vec3 b) { return vec3(fa(a.x, b.x), fa(a.y, b.y), fa(a.z, b.z)); }
OXC_DI Vec3 vsub(Vec3 a, Vec3 b) { return vec3(fs(a.x, b.x), fs(a.y, b.y), fs(a.z, b.z)); }
OXC_DI Vec3 vmul(Vec3 a, Vec3 b) { return vec3(fm(a.x, b.x), fm(a.y, b.y), fm(a.z, b.z)); }
OXC_DI Vec3 vscale(Vec3 a, float s) { return vec3(fm(a.x, s), fm(a.y, s), fm(a.z, s)); } // a * s
OXC_DI Vec3 vdiv(Vec3 a, float s) { return vec3(fd(a.x, s), fd(a.y, s), fd(a.z, s)); }
OXC_DI Vec3 vnormalize(Vec3 a) { return vdiv(a, vlength(a)); }
OXC_DI Vec3 vcross(Vec3 a, Vec3 b) { return vec3(fs(fm(a.y, b.z), fm(a.z, b.y)), fs(fm(a.z, b.x), fm(a.x, b.z)), fs(fm(a.x, b.y), fm(a.y, b.x))); }

} // namespace oxc
