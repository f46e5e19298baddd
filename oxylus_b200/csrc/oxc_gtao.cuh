// oxc_gtao.cuh — the visibility-bitmask GTAO of one pixel (passes/gtao/vbgtao_prefilter.slang, vbgtao_main.slang,
// vbgtao_denoise.slang) as pure per-thread functions: the pyramid's linearize and weighted average, the edges, the sector pass with
// its trilinear depth taps, and the edge-aware 3 x 3 denoise.
// No warp intrinsics, no shared memory: tests compile this source for the host.
// Specification: include/oxcull.h (comment above oxc_generate_ambient_occlusion) == oracle/oxc_oracle_gtao.c, operation for operation.
#pragma once
#include "oxc_alpha.cuh"
#include "oxc_vsm_resolve.cuh"

namespace oxc {

constexpr int GTAO_LEVELS = 5;                 // vbgtao_main.slang:14
constexpr uint32_t GTAO_SECTORS = 32u;         // :12
constexpr float GTAO_HALF_PI = 1.57079632679f; // common/math.slang:3-4
constexpr float GTAO_PI = 3.1415926535897932384626433832795f;

struct GtaoParams {
  const float* depth;
  const float4* normals;      // oct(world normal) in .zw
  float* mips;                // levels 0..4 packed
  uint32_t* edges;
  uint16_t* noisy;            // binary16 bits
  float* ao;
  int width, height;
  int mip_w[GTAO_LEVELS], mip_h[GTAO_LEVELS];
  long long mip_off[GTAO_LEVELS];
  float m23, m22;             // projection[3][2], projection[2][2]
  float p00, p11;             // projection[0][0], projection[1][1]
  float4 view_row[3];         // rows 0..2 of Camera::view
  float far_clip;
  float thickness, effect_radius, final_power;
  uint32_t slice_count, samples_per_slice_side, noise_index;
};

// the packed pyramid (OxcGtaoTargets::depth_mips): level k is max(w >> k, 1) x max(h >> k, 1), the levels one after another.
// gtao_mip_texels(w, h, k) is level k's offset, and with the default argument the plane's size.
__host__ inline int gtao_mip_extent(uint32_t n, int k) { return (int)((n >> k) > 1u ? (n >> k) : 1u); }
__host__ inline long long gtao_mip_texels(uint32_t w, uint32_t h, int levels = GTAO_LEVELS) {
  long long n = 0;
  for (int k = 0; k < levels; k++) n += (long long)gtao_mip_extent(w, k) * gtao_mip_extent(h, k);
  return n;
}

// the kernels' parameters from the C ABI's arguments (oxc_generate_ambient_occlusion, and the host build of the tests)
__host__ inline GtaoParams gtao_make_params(const OxcGtaoCamera& cam, const OxcGtaoSettings& st, const float* depth, const float* normals,
                                            uint32_t w, uint32_t h, const OxcGtaoTargets& t) {
  GtaoParams p{};
  p.depth = depth; p.normals = reinterpret_cast<const float4*>(normals);
  p.mips = t.depth_mips; p.edges = t.edges; p.noisy = t.noisy_occlusion; p.ao = t.ambient_occlusion;
  p.width = (int)w; p.height = (int)h;
  for (int k = 0; k < GTAO_LEVELS; k++) {
    p.mip_w[k] = gtao_mip_extent(w, k); p.mip_h[k] = gtao_mip_extent(h, k); p.mip_off[k] = gtao_mip_texels(w, h, k);
  }
  p.m23 = cam.projection[14]; p.m22 = cam.projection[10]; p.p00 = cam.projection[0]; p.p11 = cam.projection[5];
  for (int i = 0; i < 3; i++) p.view_row[i] = make_float4(cam.view[i], cam.view[4 + i], cam.view[8 + i], cam.view[12 + i]);
  p.far_clip = cam.far_clip;
  p.thickness = st.thickness; p.effect_radius = st.effect_radius; p.final_power = st.final_power;
  p.slice_count = st.slice_count; p.samples_per_slice_side = st.samples_per_slice_side; p.noise_index = st.noise_index;
  return p;
}

OXC_DI float gtao_sat(float x) { return vmin(vmax(x, 0.0f), 1.0f); }
OXC_DI float gtao_sign(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }
OXC_DI uint32_t gtao_u32(float f) { return !(f > 0.0f) ? 0u : (f >= 4294967296.0f ? 0xFFFFFFFFu : (uint32_t)f); }
OXC_DI int gtao_clamp(long long i, int n) { return (int)(i < 0 ? 0 : (i > n - 1 ? n - 1 : i)); }
OXC_DI uint32_t gtao_popc(uint32_t v) {
#ifdef __CUDA_ARCH__
  return (uint32_t)__popc(v);
#else
  return (uint32_t)__builtin_popcount(v);
#endif
}

// binary32 -> binary16 bits, round to nearest even (the R16F noisy-occlusion store; the values stored are in [0, 1])
OXC_DI uint16_t gtao_half_bits(float f) {
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
OXC_DI float gtao_half_float(uint16_t h) { return __half2float(__ushort_as_half(h)); }

// RendererInstance.cpp:151-170, the Hilbert index of (x, y) in the 64 x 64 noise table
OXC_DI uint32_t gtao_hilbert_index(uint32_t px, uint32_t py) {
  uint32_t index = 0;
  for (uint32_t level = 32u; level > 0u; level >>= 1) {
    const uint32_t rx = (px & level) ? 1u : 0u, ry = (py & level) ? 1u : 0u;
    index += level * level * ((3u * rx) ^ ry);
    if (ry == 0u) {
      if (rx == 1u) { px = 63u - px; py = 63u - py; }
      const uint32_t t = px; px = py; py = t;
    }
  }
  return index;
}

// the value a mip texel is stored as: a NaN is written as 0x7FFFFFFF, the NaN the GPU's arithmetic produces (the host's differs)
OXC_DI float gtao_mip_store(float v) { return v != v ? __uint_as_float(0x7FFFFFFFu) : v; }

// vbgtao_prefilter.slang:19-21
OXC_DI float gtao_linearize(const GtaoParams& p, float d) { return fd(p.m23, fa(d, p.m22)); }

// vbgtao_prefilter.slang:23-39 (its falloff constants, binary32 in written order)
OXC_DI float gtao_weighted_average(float d0, float d1, float d2, float d3) {
  const float effect_radius = fm(fm(0.75f, 0.5f), 1.457f);
  const float falloff_range = fm(0.615f, effect_radius);
  const float falloff_from = fm(effect_radius, fs(1.0f, 0.615f));
  const float falloff_mul = fd(-1.0f, falloff_range);
  const float falloff_add = fa(fd(falloff_from, falloff_range), 1.0f);
  const float mn = vmin(vmin(d0, d1), vmin(d2, d3));
  const float w0 = gtao_sat(fa(fm(fs(d0, mn), falloff_mul), falloff_add)), w1 = gtao_sat(fa(fm(fs(d1, mn), falloff_mul), falloff_add));
  const float w2 = gtao_sat(fa(fm(fs(d2, mn), falloff_mul), falloff_add)), w3 = gtao_sat(fa(fm(fs(d3, mn), falloff_mul), falloff_add));
  const float total = fa(fa(fa(w0, w1), w2), w3);
  return fd(fa(fa(fa(fm(w0, d0), fm(w1, d1)), fm(w2, d2)), fm(w3, d3)), total);
}

// level 0 of the virtual pyramid at any (x, y) >= 0: the clamped depth texel, linearized
OXC_DI float gtao_level0(const GtaoParams& p, long long x, long long y) {
  const int cx = x < p.width - 1 ? (int)x : p.width - 1, cy = y < p.height - 1 ? (int)y : p.height - 1;
  return gtao_linearize(p, __ldg(&p.depth[(size_t)cy * p.width + cx]));
}

// level k of the virtual pyramid at (x, y) by recursion (host checks; the prefilter kernel builds the same values in shared memory)
template <int K>
OXC_DI float gtao_virtual_level(const GtaoParams& p, long long x, long long y) {
  if constexpr (K == 0) {
    return gtao_level0(p, x, y);
  } else {
    return gtao_weighted_average(gtao_virtual_level<K - 1>(p, 2 * x, 2 * y), gtao_virtual_level<K - 1>(p, 2 * x + 1, 2 * y),
                                 gtao_virtual_level<K - 1>(p, 2 * x, 2 * y + 1), gtao_virtual_level<K - 1>(p, 2 * x + 1, 2 * y + 1));
  }
}

// one level of SampleLevel(linear_clamp, ...): bilinear at uv * size - 0.5, clamp to edge
OXC_DI float gtao_bilinear(const GtaoParams& p, int k, float u, float v) {
  const float* lvl = p.mips + p.mip_off[k];
  const int w = p.mip_w[k], h = p.mip_h[k];
  const float x = fs(fm(u, (float)w), 0.5f), y = fs(fm(v, (float)h), 0.5f);
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = fs(x, x0), wy = fs(y, y0);
  const long long ix = alpha_f2i(x0), iy = alpha_f2i(y0);
  const int xa = gtao_clamp(ix, w), xb = gtao_clamp(ix + 1, w), ya = gtao_clamp(iy, h), yb = gtao_clamp(iy + 1, h);
  const float a00 = __ldg(&lvl[(size_t)ya * w + xa]), a10 = __ldg(&lvl[(size_t)ya * w + xb]);
  const float a01 = __ldg(&lvl[(size_t)yb * w + xa]), a11 = __ldg(&lvl[(size_t)yb * w + xb]);
  const float top = fa(a00, fm(wx, fs(a10, a00))), bot = fa(a01, fm(wx, fs(a11, a01)));
  return fa(top, fm(wy, fs(bot, top)));
}

// SampleLevel(linear_clamp, uv, lambda) for lambda in [0, 4]: both levels always read
OXC_DI float gtao_sample_level(const GtaoParams& p, float u, float v, float lambda) {
  const float fl = floorf(lambda);
  const int lo = (int)fl, hi = lo + 1 < GTAO_LEVELS - 1 ? lo + 1 : GTAO_LEVELS - 1;
  const float f = fs(lambda, fl);
  return lerp_levels(f, gtao_bilinear(p, lo, u, v), gtao_bilinear(p, hi, u, v));
}

// vbgtao_main.slang:32-37
OXC_DI float gtao_fast_acos(float in_x) {
  const float x = fabsf(in_x);
  float res = fa(fm(-0.156583f, x), GTAO_HALF_PI);
  res = fm(res, fsq(gtao_sat(fs(1.0f, x))));
  return in_x >= 0.0f ? res : fs(GTAO_PI, res);
}

// :102-119
OXC_DI uint32_t gtao_update_sectors(float min_h, float max_h, uint32_t bitmask) {
  const uint32_t angle = gtao_u32(ceilf(fm(gtao_sat(fs(max_h, min_h)), (float)GTAO_SECTORS)));
  if (angle == 0u) return bitmask;
  uint32_t start = gtao_u32(fm(gtao_sat(min_h), (float)GTAO_SECTORS));
  start = start < GTAO_SECTORS - 1u ? start : GTAO_SECTORS - 1u;
  return bitmask | ((0xFFFFFFFFu >> (GTAO_SECTORS - angle)) << start);
}

OXC_DI void gtao_normalize(float x, float y, float z, float& ox, float& oy, float& oz) {
  const float l = length3(x, y, z);
  ox = fd(x, l); oy = fd(y, l); oz = fd(z, l);
}

// :124-146
OXC_DI uint32_t gtao_sector_mask(float thickness, float dx, float dy, float dz, float vx, float vy, float vz, float sd, float n) {
  const float bx = fs(dx, fm(vx, thickness)), by = fs(dy, fm(vy, thickness)), bz = fs(dz, fm(vz, thickness));
  float ax, ay, az, cx, cy, cz;
  gtao_normalize(dx, dy, dz, ax, ay, az);
  gtao_normalize(bx, by, bz, cx, cy, cz);
  float h0 = gtao_fast_acos(dot3(ax, ay, az, vx, vy, vz)), h1 = gtao_fast_acos(dot3(cx, cy, cz, vx, vy, vz));
  h0 = gtao_sat(fd(fa(fa(fm(sd, -h0), n), GTAO_HALF_PI), GTAO_PI));
  h1 = gtao_sat(fd(fa(fa(fm(sd, -h1), n), GTAO_HALF_PI), GTAO_PI));
  return sd >= 0.0f ? gtao_update_sectors(h1, h0, 0u) : gtao_update_sectors(h0, h1, 0u);
}

// vbgtao_main.slang:39-45 load_noise
OXC_DI void gtao_noise(uint32_t x, uint32_t y, uint32_t noise_index, float& n0, float& n1) {
  const uint32_t index = gtao_hilbert_index(x & 63u, y & 63u) + 288u * (noise_index & 63u);
  const float fi = (float)index;
  n0 = vfract(fa(0.5f, fm(fi, 0.75487766624669276005f)));
  n1 = vfract(fa(0.5f, fm(fi, 0.5698402909980532659114f)));
}

// :69-100 calculate_edges: the packed edges of pixel (x, y); *centre receives its linear depth
OXC_DI uint32_t gtao_edges(const GtaoParams& p, int x, int y, float* centre) {
  const float* m0 = p.mips;
  const int W = p.width, H = p.height;
  const float c = __ldg(&m0[(size_t)y * W + x]);
  const float l = __ldg(&m0[(size_t)y * W + gtao_clamp((long long)x - 1, W)]), r = __ldg(&m0[(size_t)y * W + gtao_clamp((long long)x + 1, W)]);
  const float t = __ldg(&m0[(size_t)gtao_clamp((long long)y - 1, H) * W + x]), b = __ldg(&m0[(size_t)gtao_clamp((long long)y + 1, H) * W + x]);
  float e[4] = {fs(l, c), fs(r, c), fs(t, c), fs(b, c)};
  const float slr = fm(fs(e[1], e[0]), 0.5f), stb = fm(fs(e[3], e[2]), 0.5f);
  const float adj[4] = {fa(e[0], slr), fa(e[1], -slr), fa(e[2], stb), fa(e[3], -stb)};
  const float scale = fm(c, 0.011f);
  uint32_t packed = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const float v = gtao_sat(fs(1.25f, fd(vmin(fabsf(e[i]), fabsf(adj[i])), scale)));
    packed |= (uint32_t)rintf(fm(gtao_sat(v), 255.0f)) << (8 * i);
  }
  *centre = c;
  return packed;
}

// :59-67 view_position_from_linear_depth
OXC_DI void gtao_view_position(const GtaoParams& p, float u, float v, float ld, float& x, float& y, float& z) {
  x = fm(fd(fs(fm(u, 2.0f), 1.0f), p.p00), ld);
  y = fm(fd(fs(fm(v, 2.0f), 1.0f), p.p11), ld);
  z = fm(-1.0f, ld);
}

// :148-254 for pixel (x, y) after calculate_edges: the noisy occlusion before its binary16 store, from the centre's linear depth
OXC_DI float gtao_occlusion(const GtaoParams& p, int x, int y, float ld) {
  if (ld >= fm(p.far_clip, 0.999f)) return 1.0f;
  const float rx = (float)p.width, ry = (float)p.height;
  const float slice_count = (float)p.slice_count, sps = (float)p.samples_per_slice_side;
  const float effect_radius = fm(p.effect_radius, 1.457f);
  const float falloff_range = fm(0.615f, effect_radius);
  const float falloff_from = fm(effect_radius, fs(1.0f, 0.615f));
  const float falloff_mul = fd(-1.0f, falloff_range);
  const float falloff_add = fa(fd(falloff_from, falloff_range), 1.0f);
  const float u = fd(fa((float)x, 0.5f), rx), v = fd(fa((float)y, 0.5f), ry);
  ld = fm(ld, 0.99999f);
  float ox, oy, oz, vx, vy, vz;
  gtao_view_position(p, u, v, ld, ox, oy, oz);
  gtao_normalize(-ox, -oy, -oz, vx, vy, vz);
  // load_normal_view_space :47-57: oct_to_vec3 of the binary16 .zw, mul(view, (n, 0)).xyz, normalize
  const float4 nrm = __ldg(&p.normals[(size_t)y * p.width + x]);
  const float ex = round_to_half(nrm.z), ey = round_to_half(nrm.w);
  float wx = ex, wy = ey;
  const float wz = fs(fs(1.0f, fabsf(ex)), fabsf(ey));
  const float sx = wx >= 0.0f ? 1.0f : -1.0f, sy = wy >= 0.0f ? 1.0f : -1.0f;
  if (wz < 0.0f) { wx = fm(fs(1.0f, fabsf(ey)), sx); wy = fm(fs(1.0f, fabsf(ex)), sy); }
  float ux, uy, uz;
  gtao_normalize(wx, wy, wz, ux, uy, uz);
  float nx, ny, nz;
  gtao_normalize(row_dot4(p.view_row[0], ux, uy, uz, 0.0f), row_dot4(p.view_row[1], ux, uy, uz, 0.0f), row_dot4(p.view_row[2], ux, uy, uz, 0.0f),
                 nx, ny, nz);
  float n0, n1;
  gtao_noise((uint32_t)x, (uint32_t)y, p.noise_index, n0, n1);
  const float half_r = fm(0.5f, effect_radius);
  const float sr_u = fd(fm(half_r, fabsf(p.p00)), ld), sr_v = fd(fm(half_r, fabsf(p.p11)), ld);
  const float min_s = fd(1.3f, vmax(fm(sr_u, rx), 1.3f));
  float visibility = 0.0f;
  for (float slice_t = 0.0f; slice_t < slice_count; slice_t = fa(slice_t, 1.0f)) {
    const float phi = fm(fd(fa(slice_t, n0), slice_count), GTAO_PI);
    float sn, cs;
    canonical_sincos(phi, sn, cs);
    const float dd = dot3(cs, sn, 0.0f, vx, vy, vz);
    float odx, ody, odz, axx, axy, axz;
    gtao_normalize(fs(cs, fm(dd, vx)), fs(sn, fm(dd, vy)), fs(0.0f, fm(dd, vz)), odx, ody, odz);
    gtao_normalize(fs(fm(sn, vz), fm(0.0f, vy)), fs(fm(0.0f, vx), fm(cs, vz)), fs(fm(cs, vy), fm(sn, vx)), axx, axy, axz);
    const float na = dot3(nx, ny, nz, axx, axy, axz);
    const float pnx = fs(nx, fm(axx, na)), pny = fs(ny, fm(axy, na)), pnz = fs(nz, fm(axz, na));
    const float pnl = vmax(length3(pnx, pny, pnz), 1e-6f);
    const float sign_norm = gtao_sign(dot3(odx, ody, odz, pnx, pny, pnz));
    const float cos_norm = gtao_sat(fd(dot3(pnx, pny, pnz, vx, vy, vz), pnl));
    const float n = fm(sign_norm, gtao_fast_acos(cos_norm));
    const float mul_u = fm(cs, sr_u), mul_v = fm(-sn, sr_v);
    uint32_t bitmask = 0;
    float occlusion = 0.0f;
    for (float sample_t = 0.0f; sample_t < sps; sample_t = fa(sample_t, 1.0f)) {
      const float sample_noise = vfract(fa(n1, fm(fa(slice_t, fm(sample_t, sps)), 0.6180339887498948482f)));
      float s = fd(fa(sample_t, sample_noise), sps);
      s = fm(s, s);
      s = fa(s, min_s);
      const float off_u = fm(s, mul_u), off_v = fm(s, mul_v);
      const float p1u = fa(u, off_u), p1v = fa(v, off_v), p2u = fs(u, off_u), p2v = fs(v, off_v);
      const float lu = fm(off_u, rx), lv = fm(off_v, ry);
      const float lam = vmin(vmax(fs(canonical_log2(fsq(fa(fm(lu, lu), fm(lv, lv)))), 3.30f), 0.0f), (float)(GTAO_LEVELS - 1));
      const float d1 = gtao_sample_level(p, p1u, p1v, lam), d2 = gtao_sample_level(p, p2u, p2v, lam);
      float s1x, s1y, s1z, s2x, s2y, s2z;
      gtao_view_position(p, p1u, p1v, d1, s1x, s1y, s1z);
      gtao_view_position(p, p2u, p2v, d2, s2x, s2y, s2z);
      const float e1x = fs(s1x, ox), e1y = fs(s1y, oy), e1z = fs(s1z, oz);
      const float e2x = fs(s2x, ox), e2y = fs(s2y, oy), e2z = fs(s2z, oz);
      const uint32_t m1 = gtao_sector_mask(p.thickness, e1x, e1y, e1z, vx, vy, vz, 1.0f, n);
      const uint32_t m2 = gtao_sector_mask(p.thickness, e2x, e2y, e2z, vx, vy, vz, -1.0f, n);
      const float f1 = gtao_sat(fa(fm(length3(e1x, e1y, e1z), falloff_mul), falloff_add));
      const float f2 = gtao_sat(fa(fm(length3(e2x, e2y, e2z), falloff_mul), falloff_add));
      occlusion = fa(occlusion, fd(fm(f1, (float)gtao_popc(m1 & ~bitmask)), (float)GTAO_SECTORS));
      bitmask |= m1;
      occlusion = fa(occlusion, fd(fm(f2, (float)gtao_popc(m2 & ~bitmask)), (float)GTAO_SECTORS));
      bitmask |= m2;
    }
    visibility = fa(visibility, gtao_sat(fs(1.0f, occlusion)));
  }
  return gtao_sat(fd(visibility, slice_count));
}

OXC_DI float gtao_unorm8(uint32_t v, int i) { return fd((float)((v >> (8 * i)) & 0xFFu), 255.0f); }

// vbgtao_denoise.slang:14-82 for pixel (x, y)
OXC_DI float gtao_denoise(const GtaoParams& p, int x, int y) {
  const int W = p.width, H = p.height;
  const int xl = gtao_clamp((long long)x - 1, W), xr = gtao_clamp((long long)x + 1, W);
  const size_t rt = (size_t)gtao_clamp((long long)y - 1, H) * W, rc = (size_t)y * W, rb = (size_t)gtao_clamp((long long)y + 1, H) * W;
  const uint32_t ec = __ldg(&p.edges[rc + x]), el = __ldg(&p.edges[rc + xl]), er = __ldg(&p.edges[rc + xr]);
  const uint32_t et = __ldg(&p.edges[rt + x]), eb = __ldg(&p.edges[rb + x]);
  const float center_w = 1.2f;
  const float left_w = fm(gtao_unorm8(ec, 0), gtao_unorm8(el, 1));
  const float right_w = fm(gtao_unorm8(ec, 1), gtao_unorm8(er, 0));
  const float top_w = fm(gtao_unorm8(ec, 2), gtao_unorm8(et, 3));
  const float bottom_w = fm(gtao_unorm8(ec, 3), gtao_unorm8(eb, 2));
  const float tl_w = fm(0.425f, fa(fm(top_w, gtao_unorm8(et, 0)), fm(left_w, gtao_unorm8(el, 2))));
  const float tr_w = fm(0.425f, fa(fm(top_w, gtao_unorm8(et, 1)), fm(right_w, gtao_unorm8(er, 2))));
  const float bl_w = fm(0.425f, fa(fm(bottom_w, gtao_unorm8(eb, 0)), fm(left_w, gtao_unorm8(el, 3))));
  const float br_w = fm(0.425f, fa(fm(bottom_w, gtao_unorm8(eb, 1)), fm(right_w, gtao_unorm8(er, 3))));
  const uint16_t* q = p.noisy;
  float sum = fm(gtao_half_float(__ldg(&q[rc + x])), center_w);
  sum = fa(sum, fm(gtao_half_float(__ldg(&q[rc + xl])), left_w));
  sum = fa(sum, fm(gtao_half_float(__ldg(&q[rc + xr])), right_w));
  sum = fa(sum, fm(gtao_half_float(__ldg(&q[rt + x])), top_w));
  sum = fa(sum, fm(gtao_half_float(__ldg(&q[rb + x])), bottom_w));
  sum = fa(sum, fm(gtao_half_float(__ldg(&q[rt + xl])), tl_w));
  sum = fa(sum, fm(gtao_half_float(__ldg(&q[rt + xr])), tr_w));
  sum = fa(sum, fm(gtao_half_float(__ldg(&q[rb + xl])), bl_w));
  sum = fa(sum, fm(gtao_half_float(__ldg(&q[rb + xr])), br_w));
  float sw = center_w;
  sw = fa(sw, left_w);
  sw = fa(sw, right_w);
  sw = fa(sw, top_w);
  sw = fa(sw, bottom_w);
  sw = fa(sw, tl_w);
  sw = fa(sw, tr_w);
  sw = fa(sw, bl_w);
  sw = fa(sw, br_w);
  return canonical_pow(vmax(fd(sum, sw), 0.0f), p.final_power);
}

} // namespace oxc
