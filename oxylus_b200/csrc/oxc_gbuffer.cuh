// oxc_gbuffer.cuh — the material half of the vis-buffer decode (passes/visbuffer_decode.slang:117-183, scene.slang:110-159) as pure
// per-thread functions: the material's uv transform, SampleGrad of up to five RGBA images in software, the tangent frame of the
// screen-space derivatives and the normal map, and the four attachments albedo / normal / emissive / metallic-roughness-occlusion.
// No warp intrinsics, no shared memory, no atomics: tests compile this source, and the host code that builds the device table,
// for the host.
// Specification: include/oxcull.h (comment above OxcGBufferTargets) == oracle/oxc_oracle_gbuffer.c, operation for operation.
#pragma once
#include <cstdio>
#include <string>
#include <vector>

#include "oxc_alpha.cuh"

namespace oxc {

enum : uint32_t { GB_ALBEDO = 0, GB_NORMAL = 1, GB_EMISSIVE = 2, GB_METALLIC_ROUGHNESS = 3, GB_OCCLUSION = 4, GB_SLOTS = 5 };

// Device copy of one material, reduced to what the decode reads (scene.slang:51-159); the five image descriptors follow the
// material records in the same table (GBufImage[material_count][GB_SLOTS]).
struct __align__(16) GBufMaterial {
  float albedo[4];      // dequantize_half of the factors
  float emissive[3];
  float metallic, roughness;
  float uv_size[2], uv_offset[2];
  uint32_t flags;       // MaterialFlag; an image flag is set only when its descriptor is valid
  uint32_t sampler;     // mag_filter | min_filter << 2 | mipmap_mode << 4 | address_u << 6 | address_v << 8
  uint32_t pad;
};
static_assert(sizeof(GBufMaterial) == 64, "GBufMaterial");

struct __align__(16) GBufImage {
  const uint8_t* texels; // level 0, 4-byte aligned; the other levels follow, tightly packed
  uint32_t width, height;
  uint32_t format;       // OxcImageFormat
  uint32_t levels;       // >= 1
  uint32_t pad[2];
};
static_assert(sizeof(GBufImage) == 32, "GBufImage");

// sRGB EOTF of c / 255 for c = 0..255, each entry the binary32 nearest to the exact value (oracle: its own table, tests: decimal)
__device__ const float k_srgb_to_linear[256] = {
    0x0p+0f, 0x1.3e4568p-12f, 0x1.3e4568p-11f, 0x1.dd681cp-11f, 0x1.3e4568p-10f, 0x1.8dd6c2p-10f, 0x1.dd681cp-10f, 0x1.167cbap-9f,
    0x1.3e4568p-9f, 0x1.660e14p-9f, 0x1.8dd6c2p-9f, 0x1.b6a31cp-9f, 0x1.e1e31ep-9f, 0x1.07c38cp-8f, 0x1.1fcc2cp-8f, 0x1.390ffap-8f,
    0x1.53936cp-8f, 0x1.6f5adep-8f, 0x1.8c6a94p-8f, 0x1.aac6cp-8f, 0x1.ca7382p-8f, 0x1.eb74e2p-8f, 0x1.06e76cp-7f, 0x1.18c2a6p-7f,
    0x1.2b4e0ap-7f, 0x1.3e8b7cp-7f, 0x1.527cd6p-7f, 0x1.6723eep-7f, 0x1.7c8292p-7f, 0x1.929a88p-7f, 0x1.a96d92p-7f, 0x1.c0fd68p-7f,
    0x1.d94bbep-7f, 0x1.f25a44p-7f, 0x1.061552p-6f, 0x1.135f3ep-6f, 0x1.210bb8p-6f, 0x1.2f1b8cp-6f, 0x1.3d8f84p-6f, 0x1.4c6866p-6f,
    0x1.5ba6fap-6f, 0x1.6b4c04p-6f, 0x1.7b5842p-6f, 0x1.8bcc74p-6f, 0x1.9ca958p-6f, 0x1.adefaap-6f, 0x1.bfa02p-6f, 0x1.d1bb74p-6f,
    0x1.e4425ap-6f, 0x1.f73586p-6f, 0x1.054ad4p-5f, 0x1.0f31bap-5f, 0x1.194fccp-5f, 0x1.23a55ep-5f, 0x1.2e32c8p-5f, 0x1.38f86p-5f,
    0x1.43f678p-5f, 0x1.4f2d64p-5f, 0x1.5a9d76p-5f, 0x1.664702p-5f, 0x1.722a56p-5f, 0x1.7e47c8p-5f, 0x1.8a9fa4p-5f, 0x1.97323ap-5f,
    0x1.a3ffd8p-5f, 0x1.b108dp-5f, 0x1.be4d6cp-5f, 0x1.cbcdfap-5f, 0x1.d98ac6p-5f, 0x1.e7841cp-5f, 0x1.f5ba48p-5f, 0x1.0216cap-4f,
    0x1.096f26p-4f, 0x1.10e65cp-4f, 0x1.187c9p-4f, 0x1.2031e8p-4f, 0x1.280688p-4f, 0x1.2ffa92p-4f, 0x1.380e2ap-4f, 0x1.404174p-4f,
    0x1.489494p-4f, 0x1.5107acp-4f, 0x1.599adep-4f, 0x1.624e4ep-4f, 0x1.6b221ep-4f, 0x1.74167p-4f, 0x1.7d2b66p-4f, 0x1.86612p-4f,
    0x1.8fb7cp-4f, 0x1.992f68p-4f, 0x1.a2c83ap-4f, 0x1.ac8256p-4f, 0x1.b65ddcp-4f, 0x1.c05aecp-4f, 0x1.ca79a8p-4f, 0x1.d4ba3p-4f,
    0x1.df1ca2p-4f, 0x1.e9a12p-4f, 0x1.f447cap-4f, 0x1.ff10bcp-4f, 0x1.04fe0cp-3f, 0x1.0a84fep-3f, 0x1.101d44p-3f, 0x1.15c6eep-3f,
    0x1.1b8208p-3f, 0x1.214ea6p-3f, 0x1.272cd4p-3f, 0x1.2d1ca2p-3f, 0x1.331e1ep-3f, 0x1.393158p-3f, 0x1.3f566p-3f, 0x1.458d42p-3f,
    0x1.4bd60ep-3f, 0x1.5230d4p-3f, 0x1.589dap-3f, 0x1.5f1c84p-3f, 0x1.65ad8ap-3f, 0x1.6c50c4p-3f, 0x1.73063ep-3f, 0x1.79ce06p-3f,
    0x1.80a82ep-3f, 0x1.8794cp-3f, 0x1.8e93ccp-3f, 0x1.95a55ep-3f, 0x1.9cc986p-3f, 0x1.a40052p-3f, 0x1.ab49cep-3f, 0x1.b2a60ap-3f,
    0x1.ba1512p-3f, 0x1.c196f4p-3f, 0x1.c92bbep-3f, 0x1.d0d37cp-3f, 0x1.d88e3ep-3f, 0x1.e05c0ep-3f, 0x1.e83cfcp-3f, 0x1.f03116p-3f,
    0x1.f83866p-3f, 0x1.00297ep-2f, 0x1.044072p-2f, 0x1.086116p-2f, 0x1.0c8b7p-2f, 0x1.10bf86p-2f, 0x1.14fd6p-2f, 0x1.194502p-2f,
    0x1.1d9676p-2f, 0x1.21f1bep-2f, 0x1.2656e4p-2f, 0x1.2ac5ecp-2f, 0x1.2f3edep-2f, 0x1.33c1cp-2f, 0x1.384e98p-2f, 0x1.3ce56cp-2f,
    0x1.418642p-2f, 0x1.46312p-2f, 0x1.4ae60ep-2f, 0x1.4fa51p-2f, 0x1.546e2cp-2f, 0x1.59416cp-2f, 0x1.5e1edp-2f, 0x1.630664p-2f,
    0x1.67f82ap-2f, 0x1.6cf428p-2f, 0x1.71fa68p-2f, 0x1.770aecp-2f, 0x1.7c25bcp-2f, 0x1.814adcp-2f, 0x1.867a54p-2f, 0x1.8bb428p-2f,
    0x1.90f86p-2f, 0x1.9647p-2f, 0x1.9ba01p-2f, 0x1.a10394p-2f, 0x1.a67192p-2f, 0x1.abea1p-2f, 0x1.b16d14p-2f, 0x1.b6faa4p-2f,
    0x1.bc92c6p-2f, 0x1.c2357ep-2f, 0x1.c7e2d2p-2f, 0x1.cd9acap-2f, 0x1.d35d6ap-2f, 0x1.d92ab6p-2f, 0x1.df02b8p-2f, 0x1.e4e57p-2f,
    0x1.ead2e8p-2f, 0x1.f0cb26p-2f, 0x1.f6ce2cp-2f, 0x1.fcdcp-2f, 0x1.017a56p-1f, 0x1.048c18p-1f, 0x1.07a34ap-1f, 0x1.0abfeep-1f,
    0x1.0de208p-1f, 0x1.11099ap-1f, 0x1.1436a8p-1f, 0x1.176932p-1f, 0x1.1aa13ep-1f, 0x1.1ddecap-1f, 0x1.2121dep-1f, 0x1.246a7ap-1f,
    0x1.27b8ap-1f, 0x1.2b0c54p-1f, 0x1.2e6598p-1f, 0x1.31c46ep-1f, 0x1.3528dcp-1f, 0x1.3892ep-1f, 0x1.3c028p-1f, 0x1.3f77bcp-1f,
    0x1.42f29ap-1f, 0x1.467318p-1f, 0x1.49f93ep-1f, 0x1.4d850ap-1f, 0x1.511682p-1f, 0x1.54ada4p-1f, 0x1.584a78p-1f, 0x1.5becfep-1f,
    0x1.5f9538p-1f, 0x1.634328p-1f, 0x1.66f6d4p-1f, 0x1.6ab03ap-1f, 0x1.6e6f6p-1f, 0x1.723448p-1f, 0x1.75fef4p-1f, 0x1.79cf64p-1f,
    0x1.7da59ep-1f, 0x1.8181a4p-1f, 0x1.856378p-1f, 0x1.894b1cp-1f, 0x1.8d3892p-1f, 0x1.912bdep-1f, 0x1.9525p-1f, 0x1.9923fep-1f,
    0x1.9d28d8p-1f, 0x1.a13392p-1f, 0x1.a5442cp-1f, 0x1.a95aacp-1f, 0x1.ad771p-1f, 0x1.b1995ep-1f, 0x1.b5c198p-1f, 0x1.b9efbep-1f,
    0x1.be23d4p-1f, 0x1.c25ddep-1f, 0x1.c69ddcp-1f, 0x1.cae3d2p-1f, 0x1.cf2fcp-1f, 0x1.d381aap-1f, 0x1.d7d994p-1f, 0x1.dc377ep-1f,
    0x1.e09b6ap-1f, 0x1.e5055cp-1f, 0x1.e97556p-1f, 0x1.edeb5cp-1f, 0x1.f2676cp-1f, 0x1.f6e98cp-1f, 0x1.fb71bcp-1f, 0x1p+0f
};

template <typename T>
OXC_DI T ldg_struct(const T* p) {
  static_assert(sizeof(T) % 16 == 0, "16-byte records");
  T v;
  for (uint32_t i = 0; i < sizeof(T) / 16; i++) reinterpret_cast<uint4*>(&v)[i] = __ldg(reinterpret_cast<const uint4*>(p) + i);
  return v;
}

OXC_DI uint32_t gb_texel_bytes(uint32_t format) {
  return format == OXC_IMAGE_R8_UNORM ? 1u : (format == OXC_IMAGE_RG8_UNORM ? 2u : 4u);
}

// texel (x, y) of a level as RGBA, converted before filtering as Vulkan does: one aligned 32-bit load holds the whole texel
OXC_DI float4 gb_texel(uint32_t format, const uint8_t* base, uint32_t w, uint32_t x, uint32_t y) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(base) + ((size_t)y * w + x) * gb_texel_bytes(format);
  const uint32_t t = __ldg(reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3)) >> ((uint32_t)(a & 3u) * 8u);
  const float c0 = fd((float)(t & 255u), 255.0f);
  if (format == OXC_IMAGE_R8_UNORM) return make_float4(c0, 0.0f, 0.0f, 1.0f);
  const float c1 = fd((float)((t >> 8) & 255u), 255.0f);
  if (format == OXC_IMAGE_RG8_UNORM) return make_float4(c0, c1, 0.0f, 1.0f);
  const float c3 = fd((float)(t >> 24), 255.0f);
  if (format == OXC_IMAGE_RGBA8_SRGB)
    return make_float4(__ldg(&k_srgb_to_linear[t & 255u]), __ldg(&k_srgb_to_linear[(t >> 8) & 255u]), __ldg(&k_srgb_to_linear[(t >> 16) & 255u]), c3);
  return make_float4(c0, c1, fd((float)((t >> 16) & 255u), 255.0f), c3);
}

OXC_DI float gb_bilerp(float wx, float wy, float a00, float a10, float a01, float a11) { // alpha_sample_level's operation order
  const float top = fa(a00, fm(wx, fs(a10, a00))), bot = fa(a01, fm(wx, fs(a11, a01)));
  return fa(top, fm(wy, fs(bot, top)));
}

// one level of an image with one filter: alpha_sample_level on four channels
OXC_DI float4 gb_sample_level(const GBufImage& im, uint32_t address_u, uint32_t address_v, uint32_t level, uint32_t filter, float u, float v) {
  const uint32_t bpp = gb_texel_bytes(im.format);
  const uint8_t* base = im.texels;
  uint32_t w = im.width, h = im.height;
  for (uint32_t l = 0; l < level; l++) {
    base += (size_t)w * h * bpp;
    w = w > 1u ? w >> 1 : 1u;
    h = h > 1u ? h >> 1 : 1u;
  }
  const float fw = (float)w, fh = (float)h;
  if (filter == OXC_FILTER_NEAREST) {
    const int ix = sat_i32(floorf(fm(u, fw))), iy = sat_i32(floorf(fm(v, fh)));
    return gb_texel(im.format, base, w, alpha_wrap(ix, w, address_u), alpha_wrap(iy, h, address_v));
  }
  const float x = fs(fm(u, fw), 0.5f), y = fs(fm(v, fh), 0.5f);
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = fs(x, x0), wy = fs(y, y0);
  const int ix = sat_i32(x0), iy = sat_i32(y0);
  const uint32_t xa = alpha_wrap(ix, w, address_u), xb = alpha_wrap((long long)ix + 1, w, address_u);
  const uint32_t ya = alpha_wrap(iy, h, address_v), yb = alpha_wrap((long long)iy + 1, h, address_v);
  const float4 a00 = gb_texel(im.format, base, w, xa, ya), a10 = gb_texel(im.format, base, w, xb, ya), a01 = gb_texel(im.format, base, w, xa, yb),
               a11 = gb_texel(im.format, base, w, xb, yb);
  return make_float4(gb_bilerp(wx, wy, a00.x, a10.x, a01.x, a11.x), gb_bilerp(wx, wy, a00.y, a10.y, a01.y, a11.y),
                     gb_bilerp(wx, wy, a00.z, a10.z, a01.z, a11.z), gb_bilerp(wx, wy, a00.w, a10.w, a01.w, a11.w));
}

// SampleGrad(image, sampler, uv, ddx, ddy) (spec step 4)
OXC_DI float4 gb_sample_grad(const GBufImage& im, uint32_t sampler, float u, float v, float dxu, float dxv, float dyu, float dyv) {
  const uint32_t mag = sampler & 3u, min = (sampler >> 2) & 3u, mip = (sampler >> 4) & 3u, au = (sampler >> 6) & 3u, av = (sampler >> 8) & 3u;
  if (im.levels <= 1u && mag == min) return gb_sample_level(im, au, av, 0u, min, u, v); // nothing to select
  const float w0 = (float)im.width, h0 = (float)im.height;
  return sample_grad_levels(fm(dxu, w0), fm(dxv, h0), fm(dyu, w0), fm(dyv, h0), im.levels, mag, min, mip,
                            [&](uint32_t level, uint32_t filter) { return gb_sample_level(im, au, av, level, filter, u, v); });
}

// common/encoding.slang:17-21 vec3_to_oct
OXC_DI void vec3_to_oct(float vx, float vy, float vz, float& ex, float& ey) {
  const float inv = fd(1.0f, fa(fa(fabsf(vx), fabsf(vy)), fabsf(vz)));
  const float ox = fm(vx, inv), oy = fm(vy, inv);
  if (vz <= 0.0f) {
    ex = fm(fs(1.0f, fabsf(oy)), ox >= 0.0f ? 1.0f : -1.0f);
    ey = fm(fs(1.0f, fabsf(ox)), oy >= 0.0f ? 1.0f : -1.0f);
  } else {
    ex = ox; ey = oy;
  }
}

// What the decode's geometry half hands the material evaluation for one decoded pixel.
struct GBufferPixel {
  float ddx[3], ddy[3];        // d lambda / d pixel x | y
  float wp[3][3];              // world positions of the three vertices
  float uv[2];                 // interpolated texture coordinate, before the material's uv transform
  float uv_ddx[2], uv_ddy[2];
  float n[3];                  // normalize(mul(lambda, world normals))
};

// The four attachments of one decoded pixel (spec steps 3-9).  want: bit k = target k is written (albedo, normal, emissive, mro);
// images of the other targets are not sampled.
OXC_DI void gbuffer_shade(const GBufMaterial& m, const GBufImage* images /* this material's GB_SLOTS descriptors */, const GBufferPixel& px,
                          float cam_x, float cam_y, float cam_z, uint32_t want, float4& albedo, float4& normal, float4& emissive, float4& mro) {
  // :117-122
  const float u = fa(fm(px.uv[0], m.uv_size[0]), m.uv_offset[0]), v = fa(fm(px.uv[1], m.uv_size[1]), m.uv_offset[1]);
  const float dxu = fm(px.uv_ddx[0], m.uv_size[0]), dxv = fm(px.uv_ddx[1], m.uv_size[1]);
  const float dyu = fm(px.uv_ddy[0], m.uv_size[0]), dyv = fm(px.uv_ddy[1], m.uv_size[1]);
  const auto sample = [&](uint32_t slot) { return gb_sample_grad(ldg_struct(images + slot), m.sampler, u, v, dxu, dxv, dyu, dyv); };
  if (want & 1u) { // scene.slang:110-119
    albedo = make_float4(m.albedo[0], m.albedo[1], m.albedo[2], m.albedo[3]);
    if (m.flags & OXC_MATERIAL_HAS_ALBEDO_IMAGE) {
      const float4 s = sample(GB_ALBEDO);
      albedo = make_float4(fm(albedo.x, s.x), fm(albedo.y, s.y), fm(albedo.z, s.z), fm(albedo.w, s.w));
    }
  }
  if (want & 2u) { // :127-170
    const float nx = px.n[0], ny = px.n[1], nz = px.n[2];
    float p[3][3];
    for (int c = 0; c < 3; c++) { p[c][0] = fs(px.wp[c][0], cam_x); p[c][1] = fs(px.wp[c][1], cam_y); p[c][2] = fs(px.wp[c][2], cam_z); }
    float pdx[3], pdy[3];
    for (int k = 0; k < 3; k++) {
      pdx[k] = fa(fa(fm(px.ddx[0], p[0][k]), fm(px.ddx[1], p[1][k])), fm(px.ddx[2], p[2][k]));
      pdy[k] = fa(fa(fm(px.ddy[0], p[0][k]), fm(px.ddy[1], p[1][k])), fm(px.ddy[2], p[2][k]));
    }
    const float dx_n = dot3(pdx[0], pdx[1], pdx[2], nx, ny, nz), dy_n = dot3(pdy[0], pdy[1], pdy[2], nx, ny, nz);
    const float sx[3] = {fs(pdx[0], fm(dx_n, nx)), fs(pdx[1], fm(dx_n, ny)), fs(pdx[2], fm(dx_n, nz))};
    const float sy[3] = {fs(pdy[0], fm(dy_n, nx)), fs(pdy[1], fm(dy_n, ny)), fs(pdy[2], fm(dy_n, nz))};
    const float js = sign(fs(fm(dxu, dyv), fm(dxv, dyu)));
    float tx = fm(js, fs(fm(dyv, sx[0]), fm(dxv, sy[0]))), ty = fm(js, fs(fm(dyv, sx[1]), fm(dxv, sy[1]))),
          tz = fm(js, fs(fm(dyv, sx[2]), fm(dxv, sy[2])));
    if (js != 0.0f) {
      const float len = length3(tx, ty, tz);
      tx = fd(tx, len); ty = fd(ty, len); tz = fd(tz, len);
    }
    // cross(n, pos_ddx), then w = js * sign(dot(pos_ddy, .))
    const float cx = fs(fm(ny, pdx[2]), fm(nz, pdx[1])), cy = fs(fm(nz, pdx[0]), fm(nx, pdx[2])), cz = fs(fm(nx, pdx[1]), fm(ny, pdx[0]));
    const float nw = -fm(js, sign(dot3(pdy[0], pdy[1], pdy[2], cx, cy, cz)));
    const float bx = fm(nw, fs(fm(ny, tz), fm(nz, ty))), by = fm(nw, fs(fm(nz, tx), fm(nx, tz))), bz = fm(nw, fs(fm(nx, ty), fm(ny, tx)));
    float ox = nx, oy = ny, oz = nz;
    if (m.flags & OXC_MATERIAL_HAS_NORMAL_IMAGE) {
      const float4 s = sample(GB_NORMAL);
      const float s0 = fs(fm(s.x, 2.0f), 1.0f);
      float s1 = fs(fm(s.y, 2.0f), 1.0f), s2 = fs(fm(s.z, 2.0f), 1.0f);
      if (m.flags & OXC_MATERIAL_NORMAL_FLIP_Y) s1 = -s1;
      if (m.flags & OXC_MATERIAL_NORMAL_TWO_COMPONENT) {
        const float t = fs(1.0f, fa(fm(s0, s0), fm(s1, s1)));
        s2 = fsq(t > 0.0f ? (t < 1.0f ? t : 1.0f) : 0.0f); // saturate, NaN -> 0
      }
      const float mx = fa(fa(fm(s0, tx), fm(s1, bx)), fm(s2, nx)), my = fa(fa(fm(s0, ty), fm(s1, by)), fm(s2, ny)),
                  mz = fa(fa(fm(s0, tz), fm(s1, bz)), fm(s2, nz));
      const float len = length3(mx, my, mz);
      ox = fd(mx, len); oy = fd(my, len); oz = fd(mz, len);
    }
    vec3_to_oct(ox, oy, oz, normal.x, normal.y);
    vec3_to_oct(nx, ny, nz, normal.z, normal.w);
  }
  if (want & 4u) { // scene.slang:130-139
    emissive = make_float4(m.emissive[0], m.emissive[1], m.emissive[2], 0.0f);
    if (m.flags & OXC_MATERIAL_HAS_EMISSIVE_IMAGE) {
      const float4 s = sample(GB_EMISSIVE);
      emissive.x = fm(emissive.x, s.x); emissive.y = fm(emissive.y, s.y); emissive.z = fm(emissive.z, s.z);
    }
  }
  if (want & 8u) { // scene.slang:141-159
    mro = make_float4(m.metallic, m.roughness, 1.0f, 0.0f);
    if (m.flags & OXC_MATERIAL_HAS_METALLIC_ROUGHNESS_IMAGE) {
      const float4 s = sample(GB_METALLIC_ROUGHNESS);
      mro.x = fm(mro.x, s.z); mro.y = fm(mro.y, s.y);
    }
    if (m.flags & OXC_MATERIAL_HAS_OCCLUSION_IMAGE) mro.z = sample(GB_OCCLUSION).x;
  }
}

// ---- host side: the device table ----

// scene.slang:92-94 on the host (integer bit manipulation: identical to the device's dequantize_half)
inline float host_dequantize_half(uint16_t h) {
  const uint32_t sgn = ((uint32_t)h & 0x8000u) << 16, em = (uint32_t)h & 0x7fffu;
  uint32_t r = (em + (112u << 10)) << 13;
  r = (em < (1u << 10)) ? 0u : r;
  r += (em >= (31u << 10)) ? (112u << 23) : 0u;
  const uint32_t bits = sgn | r;
  float f;
  memcpy(&f, &bits, 4);
  return f;
}

// The G-buffer decode's copy of a material table, built on the host by oxc_set_materials (which has validated the pointers).  An image slot whose flag is set but
// whose image the decode cannot read keeps a null descriptor, and *error names the first such material and slot: oxc_decode_gbuffer
// refuses the table, while the encode's alpha test, which reads the albedo slot only, goes on with it.
inline std::vector<uint8_t> gbuffer_table(const OxcMaterialTable* t, std::string* error) {
  static const char* const slot_name[GB_SLOTS] = {"albedo", "normal", "emissive", "metallic_roughness", "occlusion"};
  static const uint32_t slot_flag[GB_SLOTS] = {OXC_MATERIAL_HAS_ALBEDO_IMAGE, OXC_MATERIAL_HAS_NORMAL_IMAGE, OXC_MATERIAL_HAS_EMISSIVE_IMAGE,
                                               OXC_MATERIAL_HAS_METALLIC_ROUGHNESS_IMAGE, OXC_MATERIAL_HAS_OCCLUSION_IMAGE};
  const uint32_t n = t->material_count;
  std::vector<uint8_t> out((size_t)n * (sizeof(GBufMaterial) + GB_SLOTS * sizeof(GBufImage)), 0);
  GBufMaterial* mats = reinterpret_cast<GBufMaterial*>(out.data());
  GBufImage* imgs = reinterpret_cast<GBufImage*>(out.data() + (size_t)n * sizeof(GBufMaterial));
  char msg[256];
  for (uint32_t i = 0; i < n; i++) {
    const OxcMaterial& m = t->materials[i];
    GBufMaterial& d = mats[i];
    for (int k = 0; k < 4; k++) d.albedo[k] = host_dequantize_half(m.albedo_color[k]);
    for (int k = 0; k < 3; k++) d.emissive[k] = host_dequantize_half(m.emissive_color[k]);
    d.metallic = host_dequantize_half(m.metallic_factor); d.roughness = host_dequantize_half(m.roughness_factor);
    for (int k = 0; k < 2; k++) { d.uv_size[k] = host_dequantize_half(m.uv_size[k]); d.uv_offset[k] = host_dequantize_half(m.uv_offset[k]); }
    d.flags = m.flags;
    OxcSamplerDesc sd = {OXC_FILTER_LINEAR, OXC_FILTER_LINEAR, OXC_MIPMAP_LINEAR, OXC_ADDRESS_REPEAT, OXC_ADDRESS_REPEAT}; // Texture.hpp:38-45
    if (t->samplers && m.sampler_index < t->sampler_count) sd = t->samplers[m.sampler_index];
    const uint32_t indices[GB_SLOTS] = {m.albedo_image_index, m.normal_image_index, m.emissive_image_index, m.metallic_roughness_image_index,
                                        m.occlusion_image_index};
    bool any_image = false;
    for (uint32_t k = 0; k < GB_SLOTS; k++) {
      if (!(m.flags & slot_flag[k])) continue;
      any_image = true;
      const char* why = nullptr;
      const OxcAlphaImage* im = indices[k] < t->image_count ? &t->images[indices[k]] : nullptr;
      uint32_t full_chain = 1;
      if (im)
        for (uint32_t e = im->width > im->height ? im->width : im->height; e > 1; e >>= 1) full_chain++;
      if (!im) why = "lies outside the image table";
      else if (!im->texels_dev || (reinterpret_cast<uintptr_t>(im->texels_dev) & 3u)) why = "has null or not 4-byte aligned texels";
      else if (im->width == 0 || im->height == 0 || im->width > (1u << 16) || im->height > (1u << 16)) why = "has an extent outside 1..65536";
      else if (im->format > OXC_IMAGE_RG8_UNORM) why = "has an unknown format";
      else if (im->level_count > full_chain) why = "has more levels than its extent allows";
      if (why) {
        d.flags &= ~slot_flag[k];
        if (error->empty()) {
          snprintf(msg, sizeof msg, "material %u: %s image %u %s", i, slot_name[k], indices[k], why);
          *error = msg;
        }
        continue;
      }
      GBufImage& g = imgs[(size_t)i * GB_SLOTS + k];
      g.texels = static_cast<const uint8_t*>(im->texels_dev); g.width = im->width; g.height = im->height; g.format = im->format;
      g.levels = im->level_count ? im->level_count : 1u;
    }
    if (any_image && (sd.mag_filter > OXC_FILTER_NEAREST || sd.min_filter > OXC_FILTER_NEAREST || sd.mipmap_mode > OXC_MIPMAP_NEAREST ||
                      sd.address_u > OXC_ADDRESS_MIRRORED_REPEAT || sd.address_v > OXC_ADDRESS_MIRRORED_REPEAT) && error->empty()) {
      snprintf(msg, sizeof msg, "material %u: sampler %u has an unknown filter / mipmap / address mode", i, m.sampler_index);
      *error = msg;
    }
    d.sampler = (sd.mag_filter & 3u) | (sd.min_filter & 3u) << 2 | (sd.mipmap_mode & 3u) << 4 | (sd.address_u & 3u) << 6 | (sd.address_v & 3u) << 8;
  }
  return out;
}

} // namespace oxc
