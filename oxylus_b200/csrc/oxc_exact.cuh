// oxc_exact.cuh — the canonical binary32 arithmetic of the pipeline on the device.
//
// Every function here reproduces, operation for operation, the evaluation order the CPU oracle commits
// to (oracle/oxc_oracle.h header): IEEE RN, no fma contraction, denormals kept, IEEE divide / sqrt.
// The __f*_rn intrinsics are never contracted by nvcc, whatever -fmad says.
// Reference lines: Oxylus/src/Render/Shaders/cull.slang, scene.slang, common/math.slang.
#pragma once
#include <cuda_fp16.h>
#include <string.h>

#include "oxc_types.cuh"

namespace oxc {

#define OXC_DI __device__ __forceinline__

OXC_DI float fm(float a, float b) { return __fmul_rn(a, b); }
OXC_DI float fa(float a, float b) { return __fadd_rn(a, b); }
OXC_DI float fs(float a, float b) { return __fsub_rn(a, b); }
OXC_DI float fd(float a, float b) { return __fdiv_rn(a, b); }
OXC_DI float fsq(float a) { return __fsqrt_rn(a); }
OXC_DI float omin(float a, float b) { return a < b ? a : b; }
OXC_DI float omax(float a, float b) { return a > b ? a : b; }

// dot(a,b) = (a.x*b.x + a.y*b.y) + a.z*b.z
OXC_DI float dot3(float ax, float ay, float az, float bx, float by, float bz) {
  return fa(fa(fm(ax, bx), fm(ay, by)), fm(az, bz));
}
OXC_DI float length3(float x, float y, float z) { return fsq(dot3(x, y, z, x, y, z)); }

// common/math.slang:193-201 dequantize_half.  Identical for every one of the 65536 inputs to
// "hardware half->float, except denormals flush to (signed) zero" (tests/test_gpu_units.py checks all).
OXC_DI float dequantize_half(uint32_t h) {
  uint32_t s = (h & 0x8000u) << 16;
  uint32_t em = h & 0x7fffu;
  uint32_t r = (em + (112u << 10)) << 13;
  r = (em < (1u << 10)) ? 0u : r;
  r += (em >= (31u << 10)) ? (112u << 23) : 0u;
  return __uint_as_float(s | r);
}

// Same function through the hardware half->float conversion: identical for all 65536 inputs up to NaN
// payloads (hardware quiets signalling NaNs; every consumer only compares).  ~4 instructions instead of ~10.
OXC_DI float dequantize_half_hw(uint32_t h) {
  const float f = __half2float(__ushort_as_half((unsigned short)h));
  return (h & 0x7C00u) == 0u ? __uint_as_float((h & 0x8000u) << 16) : f; // denormals flush to signed zero
}

// scene.slang:408-418: i8 / 127.0
OXC_DI float s8_over_127(int v) { return fd((float)v, 127.0f); }

// row . (x,y,z,w): ((r.x*x + r.y*y) + r.z*z) + r.w*w
OXC_DI float row_dot4(float4 r, float x, float y, float z, float w) {
  return fa(fa(fa(fm(r.x, x), fm(r.y, y)), fm(r.z, z)), fm(r.w, w));
}
// w == 1.0f: r.w * 1.0f == r.w exactly
OXC_DI float row_dot_p1(float4 r, float x, float y, float z) { return fa(fa(fa(fm(r.x, x), fm(r.y, y)), fm(r.z, z)), r.w); }

struct ScreenAabb {
  float minx, miny, minz, maxx, maxy, maxz;
};

// cull.slang:12-47.  mvp rows r0..r3.  e = FULL extent.  Returns false for `none`.
// SX/SY/SZ: mul(mvp, (e.x,0,0,0))[i] = ((M[i][0]*e.x + M[i][1]*0) + M[i][2]*0) + M[i][3]*0 == M[i][0]*e.x
// up to the sign of a zero, which no consumer below can observe.
OXC_DI bool project_aabb(const float4 r0, const float4 r1, const float4 r2, const float4 r3, float near_clip, float cx,
                         float cy, float cz, float ex, float ey, float ez, ScreenAabb& out) {
  const float SXx = fm(r0.x, ex), SXy = fm(r1.x, ex), SXz = fm(r2.x, ex), SXw = fm(r3.x, ex);
  const float SYx = fm(r0.y, ey), SYy = fm(r1.y, ey), SYz = fm(r2.y, ey), SYw = fm(r3.y, ey);
  const float SZx = fm(r0.z, ez), SZy = fm(r1.z, ez), SZz = fm(r2.z, ez), SZw = fm(r3.z, ez);
  const float px = fs(cx, fm(ex, 0.5f)), py = fs(cy, fm(ey, 0.5f)), pz = fs(cz, fm(ez, 0.5f));
  float X[8], Y[8], Z[8], W[8];
  X[0] = row_dot_p1(r0, px, py, pz); Y[0] = row_dot_p1(r1, px, py, pz);
  Z[0] = row_dot_p1(r2, px, py, pz); W[0] = row_dot_p1(r3, px, py, pz);
#define OXC_ADDV(d, s, V) X[d] = fa(X[s], V##x); Y[d] = fa(Y[s], V##y); Z[d] = fa(Z[s], V##z); W[d] = fa(W[s], V##w);
  OXC_ADDV(1, 0, SZ) OXC_ADDV(2, 0, SY) OXC_ADDV(3, 2, SZ) OXC_ADDV(4, 0, SX)
  OXC_ADDV(5, 4, SZ) OXC_ADDV(6, 4, SY) OXC_ADDV(7, 6, SZ)
#undef OXC_ADDV
  float depth = W[7];
#pragma unroll
  for (int i = 6; i >= 0; i--) depth = omin(W[i], depth);
  if (depth < near_clip) return false;
  float mnx, mny, mnz, mxx, mxy, mxz;
#pragma unroll
  for (int i = 7; i >= 0; i--) {
    const float dx = fd(X[i], W[i]), dy = fd(Y[i], W[i]), dz = fd(Z[i], W[i]);
    if (i == 7) { mnx = mxx = dx; mny = mxy = dy; mnz = mxz = dz; }
    else {
      mnx = omin(dx, mnx); mny = omin(dy, mny); mnz = omin(dz, mnz);
      mxx = omax(dx, mxx); mxy = omax(dy, mxy); mxz = omax(dz, mxz);
    }
  }
  out.minx = fa(fm(mnx, 0.5f), 0.5f); out.miny = fa(fm(mny, 0.5f), 0.5f); out.minz = mnz;
  out.maxx = fa(fm(mxx, 0.5f), 0.5f); out.maxy = fa(fm(mxy, 0.5f), 0.5f); out.maxz = mxz;
  return true;
}

// cull.slang:73-81 with the six normalised planes hoisted per instance (InstCull::plane)
OXC_DI bool test_frustum_planes(const float4* __restrict__ planes, float cx, float cy, float cz, float ex, float ey,
                                float ez) {
  const float hx = fm(ex, 0.5f), hy = fm(ey, 0.5f), hz = fm(ez, 0.5f);
  float4 pl[6];
#pragma unroll
  for (int i = 0; i < 6; i++) pl[i] = __ldg(&planes[i]); // all six loads in flight before the first test
  bool inside = true;
#pragma unroll
  for (int i = 0; i < 6; i++) {
    const float4 p = pl[i];
    const float sx = __uint_as_float(__float_as_uint(hx) ^ (__float_as_uint(p.x) & 0x80000000u));
    const float sy = __uint_as_float(__float_as_uint(hy) ^ (__float_as_uint(p.y) & 0x80000000u));
    const float sz = __uint_as_float(__float_as_uint(hz) ^ (__float_as_uint(p.z) & 0x80000000u));
    inside = inside && !(dot3(fa(cx, sx), fa(cy, sy), fa(cz, sz), p.x, p.y, p.z) <= -p.w);
  }
  return inside;
}

// ceil(log2(float(n))) in integers (oracle: orc_ceil_log2_u32)
OXC_DI uint32_t ceil_log2_u32(uint32_t n) { return n <= 1u ? 0u : 32u - (uint32_t)__clz((int)(n - 1u)); }

// cull.slang:86-135.  hiz_off = per-level float offsets (shared memory copy).
OXC_DI bool test_occlusion(const ScreenAabb& a, const float* __restrict__ hiz, uint32_t hw_u, uint32_t hh_u,
                           uint32_t levels, const uint32_t* hiz_off) {
  const float hw = (float)hw_u, hh = (float)hh_u;
  const uint32_t min_tx = __float2uint_rz(omax(fm(a.minx, hw), 0.0f));
  const uint32_t min_ty = __float2uint_rz(omax(fm(a.miny, hh), 0.0f));
  const uint32_t max_tx = __float2uint_rz(omin(fm(a.maxx, hw), fs(hw, 1.0f)));
  const uint32_t max_ty = __float2uint_rz(omin(fm(a.maxy, hh), fs(hh, 1.0f)));
  const uint32_t sx = max_tx - min_tx, sy = max_ty - min_ty;
  const uint32_t max_size = sx > sy ? sx : sy;
  uint32_t mip = ceil_log2_u32(max_size);
  mip = mip > levels - 1 ? levels - 1 : mip;
  const float u = fd(fm(fa((float)min_tx, (float)max_tx), 0.5f), hw);
  const float v = fd(fm(fa((float)min_ty, (float)max_ty), 0.5f), hh);
  uint32_t mw = hw_u >> mip, mh = hh_u >> mip;
  mw = mw < 1 ? 1 : mw;
  mh = mh < 1 ? 1 : mh;
  const int bx = __float2int_rz(floorf(fs(fm(u, (float)mw), 0.5f)));
  const int by = __float2int_rz(floorf(fs(fm(v, (float)mh), 0.5f)));
  const int mx = (int)mw - 1, my = (int)mh - 1;
  const int x0 = min(max(bx, 0), mx), x1 = min(max(bx + 1, 0), mx);
  const int y0 = min(max(by, 0), my), y1 = min(max(by + 1, 0), my);
  const float* lvl = hiz + hiz_off[mip];
  const float p00 = __ldg(lvl + (size_t)y0 * mw + x0), p10 = __ldg(lvl + (size_t)y0 * mw + x1);
  const float p01 = __ldg(lvl + (size_t)y1 * mw + x0), p11 = __ldg(lvl + (size_t)y1 * mw + x1);
  const float d = omin(omin(p00, p10), omin(p01, p11));
  return a.maxz <= fs(d, 1e-7f);
}

// cull_meshlets_hiz.slang:53-58 cone part with the per-instance terms hoisted.  Returns cone_visible.
OXC_DI bool cone_visible_positional(const InstCull* __restrict__ ic, float cx, float cy, float cz, float ex, float ey,
                                    float ez, float ax, float ay, float az, float cutoff, float camx, float camy,
                                    float camz) {
  if (cutoff >= 1.0f) return true;
  const float4 n0 = __ldg(&ic->nrm[0]), n1 = __ldg(&ic->nrm[1]), n2 = __ldg(&ic->nrm[2]);
  // mul(N, axis)[i] = (r0[i]*a.x + r1[i]*a.y) + r2[i]*a.z
  const float nx = fa(fa(fm(n0.x, ax), fm(n1.x, ay)), fm(n2.x, az));
  const float ny = fa(fa(fm(n0.y, ax), fm(n1.y, ay)), fm(n2.y, az));
  const float nz = fa(fa(fm(n0.z, ax), fm(n1.z, ay)), fm(n2.z, az));
  const float len = length3(nx, ny, nz);
  const float wax = fd(nx, len), way = fd(ny, len), waz = fd(nz, len);
  const float4 w0 = __ldg(&ic->world_row[0]), w1 = __ldg(&ic->world_row[1]), w2 = __ldg(&ic->world_row[2]);
  const float wcx = row_dot_p1(w0, cx, cy, cz), wcy = row_dot_p1(w1, cx, cy, cz), wcz = row_dot_p1(w2, cx, cy, cz);
  const float hx = fm(ex, 0.5f), hy = fm(ey, 0.5f), hz = fm(ez, 0.5f);
  const float wr = fm(length3(hx, hy, hz), n0.w); // to_world_radius: radius * max row length
  const float dx = fs(wcx, camx), dy = fs(wcy, camy), dz = fs(wcz, camz);
  // test_cone: dot(d, axis) >= cutoff * length(d) + radius
  const bool culled = dot3(dx, dy, dz, wax, way, waz) >= fa(fm(cutoff, length3(dx, dy, dz)), wr);
  return !culled;
}

// world-space cone axis only (directional cone test, cull_meshlets_hpb.slang:53-54)
OXC_DI void world_cone_axis(const InstCull* __restrict__ ic, float ax, float ay, float az, float& wax, float& way,
                            float& waz) {
  const float4 n0 = __ldg(&ic->nrm[0]), n1 = __ldg(&ic->nrm[1]), n2 = __ldg(&ic->nrm[2]);
  const float nx = fa(fa(fm(n0.x, ax), fm(n1.x, ay)), fm(n2.x, az));
  const float ny = fa(fa(fm(n0.y, ax), fm(n1.y, ay)), fm(n2.y, az));
  const float nz = fa(fa(fm(n0.z, ax), fm(n1.z, ay)), fm(n2.z, az));
  const float len = length3(nx, ny, nz);
  wax = fd(nx, len); way = fd(ny, len); waz = fd(nz, len);
}

// mul(A, B) with column-major storage (m[col*4+row]); out row-major rows as float4
OXC_DI void mul_mm_rows(const float* __restrict__ a, const float* __restrict__ b, float4 rows[4]) {
#define A(i, j) a[(j) * 4 + (i)]
#define B(i, j) b[(j) * 4 + (i)]
#pragma unroll
  for (int i = 0; i < 4; i++) {
    float r[4];
#pragma unroll
    for (int j = 0; j < 4; j++)
      r[j] = fa(fa(fa(fm(A(i, 0), B(0, j)), fm(A(i, 1), B(1, j))), fm(A(i, 2), B(2, j))), fm(A(i, 3), B(3, j)));
    rows[i] = make_float4(r[0], r[1], r[2], r[3]);
  }
#undef A
#undef B
}

// cull.slang:58-71 + normalize_plane :49-51
OXC_DI void frustum_planes(const float4 rows[4], float4 planes[6]) {
  float4 p[6];
  p[0] = make_float4(fa(rows[3].x, rows[0].x), fa(rows[3].y, rows[0].y), fa(rows[3].z, rows[0].z), fa(rows[3].w, rows[0].w));
  p[1] = make_float4(fs(rows[3].x, rows[0].x), fs(rows[3].y, rows[0].y), fs(rows[3].z, rows[0].z), fs(rows[3].w, rows[0].w));
  p[2] = make_float4(fa(rows[3].x, rows[1].x), fa(rows[3].y, rows[1].y), fa(rows[3].z, rows[1].z), fa(rows[3].w, rows[1].w));
  p[3] = make_float4(fs(rows[3].x, rows[1].x), fs(rows[3].y, rows[1].y), fs(rows[3].z, rows[1].z), fs(rows[3].w, rows[1].w));
  p[4] = rows[2];
  p[5] = make_float4(fs(rows[3].x, rows[2].x), fs(rows[3].y, rows[2].y), fs(rows[3].z, rows[2].z), fs(rows[3].w, rows[2].w));
#pragma unroll
  for (int i = 0; i < 6; i++) {
    const float len = length3(p[i].x, p[i].y, p[i].z);
    planes[i] = make_float4(fd(p[i].x, len), fd(p[i].y, len), fd(p[i].z, len), fd(p[i].w, len));
  }
}

// full test_frustum from rows (mesh-level test in cull_meshes.slang:34)
OXC_DI bool test_frustum_rows(const float4 planes[6], float cx, float cy, float cz, float ex, float ey, float ez) {
  const float hx = fm(ex, 0.5f), hy = fm(ey, 0.5f), hz = fm(ez, 0.5f);
#pragma unroll
  for (int i = 0; i < 6; i++) {
    const float4 p = planes[i];
    const float sx = __uint_as_float(__float_as_uint(hx) ^ (__float_as_uint(p.x) & 0x80000000u));
    const float sy = __uint_as_float(__float_as_uint(hy) ^ (__float_as_uint(p.y) & 0x80000000u));
    const float sz = __uint_as_float(__float_as_uint(hz) ^ (__float_as_uint(p.z) & 0x80000000u));
    if (dot3(fa(cx, sx), fa(cy, sy), fa(cz, sz), p.x, p.y, p.z) <= -p.w) return false;
  }
  return true;
}

// log2 for decision paths (VSM clipmap selection): the same operation sequence as oracle/oxc_oracle.c orc_log2_canonical, so the
// result is bit-identical on both sides.  |error| < 1e-7 absolute on [2^-126, 2^127].
OXC_DI float canonical_log2(float x) {
  if (!(x > 0.0f)) return -3.0e38f;
  if (!(x <= 3.0e38f)) return 3.0e38f;
  int e = 0;
  if (x < 1.17549435e-38f) { x = fm(x, 16777216.0f); e = -24; }
  const uint32_t bits = __float_as_uint(x);
  e += (int)(bits >> 23) - 127;
  float m = __uint_as_float((bits & 0x007FFFFFu) | 0x3F800000u);
  if (m > 1.41421354f) { m = fm(m, 0.5f); e += 1; }
  const float t = fd(fs(m, 1.0f), fa(m, 1.0f));
  const float t2 = fm(t, t);
  float p = 0.412198562f;
  p = fa(0.577078044f, fm(t2, p));
  p = fa(0.961796701f, fm(t2, p));
  p = fa(2.88539004f, fm(t2, p));
  return fa((float)e, fm(t, p));
}

// functions the parameter builders also call on the host
#define OXC_HD __host__ __device__ __forceinline__

// binary64 operations of canonical_sincos, canonical_acos and canonical_atan2: the device intrinsics are never contracted; the host
// build runs -ffp-contract=off
OXC_HD double dmul64(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
OXC_HD double dadd64(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
OXC_HD float d2f_rn(double a) {
#ifdef __CUDA_ARCH__
  return __double2float_rn(a);
#else
  return (float)a;
#endif
}

// sin and cos for decision paths (VSM shadow resolve), bit-identical to oracle/oxc_oracle_vsm_resolve.c orc_sincos_canonical.  Binary64 throughout: k = rint(x * 2/pi),
// r = (x - k * PIO2_HI) - k * PIO2_LO (PIO2_HI has 33 significant bits, so k * PIO2_HI is exact for |k| < 2^20), Taylor
// polynomials of sin (to r^15) and cos (to r^16) on |r| <= pi/4, the quadrant k mod 4, one rounding to binary32.
// Error against the exact sin / cos: <= 1 ulp of the binary32 result on [0, 2 pi]; <= 2^-24 absolute for |x| <= 2^21 (the hash's
// arguments reach 1.43e6 at 3840 x 2160).  Non-finite x gives NaN.  The host runs it for per-call constants (draw_sun's cosine).
OXC_HD void canonical_sincos(float xf, float& s_out, float& c_out) {
  const double x = (double)xf;
  if (!(x - x == 0.0)) { s_out = c_out = xf - xf; return; } // inf / NaN -> NaN
  const double k = rint(dmul64(x, 0.63661977236758134308));
  const double r = dadd64(dadd64(x, -dmul64(k, 1.57079632673412561417e+00)), -dmul64(k, 6.07710050650619224932e-11));
  const double z = dmul64(r, r);
  double ps = -7.6471637318198164759e-13;                    // -1/15!
  ps = dadd64(1.6059043836821614599e-10, dmul64(z, ps));     // 1/13!
  ps = dadd64(-2.5052108385441718775e-08, dmul64(z, ps));    // -1/11!
  ps = dadd64(2.7557319223985890653e-06, dmul64(z, ps));     // 1/9!
  ps = dadd64(-1.9841269841269841270e-04, dmul64(z, ps));    // -1/7!
  ps = dadd64(8.3333333333333333333e-03, dmul64(z, ps));     // 1/5!
  ps = dadd64(-1.6666666666666666667e-01, dmul64(z, ps));    // -1/3!
  const double sn = dadd64(r, dmul64(dmul64(r, z), ps));
  double pc = 4.7794773323873852974e-14;                     // 1/16!
  pc = dadd64(-1.1470745597729724714e-11, dmul64(z, pc));    // -1/14!
  pc = dadd64(2.0876756987868098979e-09, dmul64(z, pc));     // 1/12!
  pc = dadd64(-2.7557319223985890653e-07, dmul64(z, pc));    // -1/10!
  pc = dadd64(2.4801587301587301587e-05, dmul64(z, pc));     // 1/8!
  pc = dadd64(-1.3888888888888888889e-03, dmul64(z, pc));    // -1/6!
  pc = dadd64(4.1666666666666666667e-02, dmul64(z, pc));     // 1/4!
  pc = dadd64(-0.5, dmul64(z, pc));                          // -1/2!
  const double cs = dadd64(1.0, dmul64(z, pc));
  const int q = (int)dadd64(k, -dmul64(4.0, floor(dmul64(k, 0.25)))); // k mod 4, exact for every finite k
  const double sv = q == 0 ? sn : (q == 1 ? cs : (q == 2 ? -sn : -cs));
  const double cv = q == 0 ? cs : (q == 1 ? -sn : (q == 2 ? -cs : sn));
  s_out = d2f_rn(sv);
  c_out = d2f_rn(cv);
}
OXC_DI float canonical_sin(float x) { float s, c; canonical_sincos(x, s, c); return s; }
OXC_HD float canonical_cos(float x) { float s, c; canonical_sincos(x, s, c); return c; }

OXC_HD double ddiv64(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}

// pow for the GTAO denoise, bit-identical to oracle/oxc_oracle_gtao.c orc_pow_canonical.  Binary64 throughout, one rounding to
// binary32: x = m * 2^e with m in [sqrt(1/2), sqrt(2)] (taken from the binary32 bits), log m = 2 atanh(t), t = (m - 1) / (m + 1), by
// its series to t^23; L = e * LN2_HI + (e * LN2_LO + log m); z = y * L clamped to +-1100; exp(z) = 2^k exp(r), k = rint(z / ln 2),
// r = (z - k * LN2_HI) - k * LN2_LO (LN2_HI has 32 significant bits, so k * LN2_HI is exact), exp(r) by Taylor to r^13, ldexp.
// Before the rounding the relative error is a few units of 2^-50, so the result is within 1 ulp of the correctly rounded binary32
// power (it can differ from it only next to a rounding tie).  pow(1, y) = 1 and pow(x, 0) = 1 (NaN included); NaN or x < 0 gives
// NaN; pow(+-0, y) = 0 for y > 0, +inf for y < 0; pow(inf, y) = inf for y > 0, else 0; y = +-inf by |x| against 1.
OXC_DI float canonical_pow(float xf, float yf) {
  if (xf == 1.0f || yf == 0.0f) return 1.0f;
  if (xf != xf || yf != yf || xf < 0.0f) return __uint_as_float(0x7FC00000u);
  if (xf == 0.0f) return yf > 0.0f ? 0.0f : __uint_as_float(0x7F800000u);
  if (xf == __uint_as_float(0x7F800000u)) return yf > 0.0f ? xf : 0.0f;
  if (fabsf(yf) == __uint_as_float(0x7F800000u)) return (xf < 1.0f) == (yf > 0.0f) ? 0.0f : __uint_as_float(0x7F800000u);
  int e = 0;
  float xm = xf;
  if (xm < 1.17549435e-38f) { xm = fm(xm, 16777216.0f); e = -24; }
  const uint32_t bits = __float_as_uint(xm);
  e += (int)(bits >> 23) - 127;
  float m = __uint_as_float((bits & 0x007FFFFFu) | 0x3F800000u);
  if (m > 1.41421354f) { m = fm(m, 0.5f); e += 1; }
  const double md = (double)m;
  const double t = ddiv64(dadd64(md, -1.0), dadd64(md, 1.0));
  const double s = dmul64(t, t);
  double p = 1.0 / 23.0;
  p = dadd64(1.0 / 21.0, dmul64(s, p));
  p = dadd64(1.0 / 19.0, dmul64(s, p));
  p = dadd64(1.0 / 17.0, dmul64(s, p));
  p = dadd64(1.0 / 15.0, dmul64(s, p));
  p = dadd64(1.0 / 13.0, dmul64(s, p));
  p = dadd64(1.0 / 11.0, dmul64(s, p));
  p = dadd64(1.0 / 9.0, dmul64(s, p));
  p = dadd64(1.0 / 7.0, dmul64(s, p));
  p = dadd64(1.0 / 5.0, dmul64(s, p));
  p = dadd64(1.0 / 3.0, dmul64(s, p));
  const double u = dmul64(t, 2.0);
  const double lm = dadd64(u, dmul64(dmul64(u, s), p));
  const double ed = (double)e;
  const double L = dadd64(dmul64(ed, 6.93147180369123816490e-01), dadd64(dmul64(ed, 1.90821492927058770002e-10), lm));
  double z = dmul64((double)yf, L);
  z = z > 1100.0 ? 1100.0 : (z < -1100.0 ? -1100.0 : z);
  const double k = rint(dmul64(z, 1.44269504088896338700e+00));
  const double r = dadd64(dadd64(z, -dmul64(k, 6.93147180369123816490e-01)), -dmul64(k, 1.90821492927058770002e-10));
  double q = 1.0 / 6227020800.0; // 1/13!
  q = dadd64(1.0 / 479001600.0, dmul64(r, q));
  q = dadd64(1.0 / 39916800.0, dmul64(r, q));
  q = dadd64(1.0 / 3628800.0, dmul64(r, q));
  q = dadd64(1.0 / 362880.0, dmul64(r, q));
  q = dadd64(1.0 / 40320.0, dmul64(r, q));
  q = dadd64(1.0 / 5040.0, dmul64(r, q));
  q = dadd64(1.0 / 720.0, dmul64(r, q));
  q = dadd64(1.0 / 120.0, dmul64(r, q));
  q = dadd64(1.0 / 24.0, dmul64(r, q));
  q = dadd64(1.0 / 6.0, dmul64(r, q));
  q = dadd64(0.5, dmul64(r, q));
  q = dadd64(1.0, dmul64(r, q));
  const double er = dadd64(1.0, dmul64(r, q));
  return d2f_rn(ldexp(er, (int)k));
}

// pow(x, 5.0) for F_Schlick (PBR apply), bit-identical to oracle/oxc_oracle_pbr.c orc_pow5_canonical: x2 = x * x in binary64, then
// (x2 * x2) * x in binary64, one rounding to binary32.  Within 1 ulp of the correctly rounded binary32 power: x has 24 significant
// bits, so x2 (48 bits) is exact; x2 * x2 and the product with x each round once with relative error <= 2^-53, so the binary64 value
// is x^5 (1 + d) with |d| < 2^-51.  No binary64 overflow or underflow can occur for finite binary32 x (|x^5| lies in [2^-745,
// 2^640] or is 0), so the bound holds everywhere.  Half a binary32 ulp is at least 2^-25 relative (less only among binary32
// subnormals, where the absolute spacing 2^-149 only widens it), so rounding x^5 (1 + d) gives RN(x^5) or, when x^5 lies within
// 2^-51 relative of a rounding tie, its neighbour across that tie: in both cases |result - x^5| < 1 ulp.  NaN stays NaN, +-inf and
// +-0 follow the sign of x.
OXC_DI float canonical_pow5(float xf) {
  const double x = (double)xf;
  const double x2 = dmul64(x, x);
  return d2f_rn(dmul64(dmul64(x2, x2), x));
}

// binary32 operations for functions the parameter builders also call on the host: the device intrinsics, or one IEEE operation in the
// host code (compiled with -ffp-contract=off, as the library's host code is)
OXC_HD float hd_mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
OXC_HD float hd_add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
OXC_HD float hd_sub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
OXC_HD float hd_pow2(int k) { // 2^k for k in -126..127, from its bits
  const uint32_t u = (uint32_t)(k + 127) << 23;
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}

// exp in binary32 for the atmosphere's media (sky.slang:134-135, :231), bit-identical to oracle/oxc_oracle_atmosphere.c
// orc_exp_canonical.  Cody-Waite: k = rint(x * fl(log2 e)), r = (x - k * LN2_HI) - k * LN2_LO with LN2_HI = 0.693359375 (9 significant
// bits, so k * LN2_HI is exact for every k reached, and x - k * LN2_HI is exact by Sterbenz), exp(r) = 1 + (r + r^2 * q(r)) with q the
// Taylor polynomial to r^8 / 8! by Horner, then the bits of 2^k: one multiplication for k in -126..127, two for k = 128 (the first
// exact) and for k < -126 (the first exact, the second rounds once into the subnormals).  Error: at most 1 ulp against the exact
// exp over all binary32 inputs (tests/test_oracle_atmosphere.py checks 10^7 inputs against binary64); exp(+-0) = 1 exactly, x > 89
// and +inf give +inf, x < -104 and -inf give +0, NaN stays NaN (the input's bits).
OXC_HD float canonical_exp(float x) {
  if (x != x) return x;
  if (x > 89.0f) return hd_mul(hd_pow2(127), hd_pow2(127)); // +inf
  if (x < -104.0f) return 0.0f;
  const float k = rintf(hd_mul(x, 1.44269502f));
  const float r = hd_sub(hd_sub(x, hd_mul(k, 0.693359375f)), hd_mul(k, -2.12194440e-4f));
  float q = 2.48015873e-05f;               // 1/8!
  q = hd_add(1.98412701e-04f, hd_mul(r, q)); // 1/7!
  q = hd_add(1.38888892e-03f, hd_mul(r, q)); // 1/6!
  q = hd_add(8.33333377e-03f, hd_mul(r, q)); // 1/5!
  q = hd_add(4.16666679e-02f, hd_mul(r, q)); // 1/4!
  q = hd_add(1.66666672e-01f, hd_mul(r, q)); // 1/3!
  q = hd_add(0.5f, hd_mul(r, q));
  const float p = hd_add(1.0f, hd_add(r, hd_mul(hd_mul(r, r), q)));
  const int ki = (int)k;
  if (ki > 127) return hd_mul(hd_mul(p, hd_pow2(127)), hd_pow2(ki - 127));
  if (ki < -126) return hd_mul(hd_mul(p, hd_pow2(ki + 100)), hd_pow2(-100));
  return hd_mul(p, hd_pow2(ki));
}

// acos, bit-identical to oracle/oxc_oracle_atmosphere.c orc_acos_canonical: the parameter builders' beta (sky.slang:76, once per
// call on the host) and the sky IBL's per-sample view-zenith angle (sky.slang:49, on the device).  Binary64 throughout, one rounding
// to binary32: for |x| <= 1/2, pi/2 - asin(x); above, 2 asin(sqrt((1 - |x|) / 2)) (x > 0) or pi - that (x < 0); asin(s) = s + s z P(z),
// z = s^2 <= 1/4, by its series to s^57.  The coefficients c[n] = central(n) / (2n + 1), central(n) = central(n - 1) * (2n - 1) / (2n),
// are the binary64 values of that recurrence as the oracle evaluates it (tests/test_oracle_sky_ibl.py recomputes them), written out so
// that the device does not rerun it per call.  Before the rounding the error is a few units of 2^-53 relative, so the result is within
// 1 ulp of the exact acos.  |x| > 1 and NaN give NaN (0x7FC00000).
OXC_HD float canonical_acos(float xf) {
  const double x = (double)xf;
  if (!(x >= -1.0 && x <= 1.0)) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(0x7FC00000u);
#else
    return __builtin_nanf("");
#endif
  }
  const double a = x < 0.0 ? -x : x;
#ifdef __CUDA_ARCH__
  const double s = a <= 0.5 ? x : __dsqrt_rn(dmul64(dadd64(1.0, -a), 0.5));
#else
  const double s = a <= 0.5 ? x : sqrt((1.0 - a) * 0.5);
#endif
  const double z = dmul64(s, s);
  double p = 0x1.e82be60d9127ep-10;
  p = dadd64(0x1.018f963c229bfp-9, dmul64(z, p));
  p = dadd64(0x1.1052bc5fa960ap-9, dmul64(z, p));
  p = dadd64(0x1.208d3570ae5a6p-9, dmul64(z, p));
  p = dadd64(0x1.3275586c5f2f0p-9, dmul64(z, p));
  p = dadd64(0x1.464c0950f7d47p-9, dmul64(z, p));
  p = dadd64(0x1.5c5f56efaaaabp-9, dmul64(z, p));
  p = dadd64(0x1.750de64d7d05fp-9, dmul64(z, p));
  p = dadd64(0x1.90cb77f60c7cep-9, dmul64(z, p));
  p = dadd64(0x1.b026f57b13b14p-9, dmul64(z, p));
  p = dadd64(0x1.d3d2a8e0dd67dp-9, dmul64(z, p));
  p = dadd64(0x1.fcaf8fb6db6dbp-9, dmul64(z, p));
  p = dadd64(0x1.15ee9d45d1746p-8, dmul64(z, p));
  p = dadd64(0x1.31683bdef7bdfp-8, dmul64(z, p));
  p = dadd64(0x1.51ba308d3dcb1p-8, dmul64(z, p));
  p = dadd64(0x1.782dda12f684cp-8, dmul64(z, p));
  p = dadd64(0x1.a6863d70a3d71p-8, dmul64(z, p));
  p = dadd64(0x1.df3bd37a6f4dfp-8, dmul64(z, p));
  p = dadd64(0x1.12ef3cf3cf3cfp-7, dmul64(z, p));
  p = dadd64(0x1.3fde50d79435ep-7, dmul64(z, p));
  p = dadd64(0x1.7a87878787878p-7, dmul64(z, p));
  p = dadd64(0x1.c99999999999ap-7, dmul64(z, p));
  p = dadd64(0x1.1c4ec4ec4ec4fp-6, dmul64(z, p));
  p = dadd64(0x1.6e8ba2e8ba2e9p-6, dmul64(z, p));
  p = dadd64(0x1.f1c71c71c71c7p-6, dmul64(z, p));
  p = dadd64(0x1.6db6db6db6db7p-5, dmul64(z, p));
  p = dadd64(0x1.3333333333333p-4, dmul64(z, p));
  p = dadd64(0x1.5555555555555p-3, dmul64(z, p));
  const double as = dadd64(s, dmul64(dmul64(s, z), p));
  const double PI_D = 3.141592653589793116;
  if (a <= 0.5) return d2f_rn(dadd64(dmul64(PI_D, 0.5), -as));
  return d2f_rn(x > 0.0 ? dmul64(2.0, as) : dadd64(PI_D, -dmul64(2.0, as)));
}

// atan2 for the sky IBL's per-sample longitude (sky.slang:64), bit-identical to oracle/oxc_oracle_sky_ibl.c orc_atan2_canonical.
// Binary64 throughout, one rounding to binary32.  Special cases as C99 Annex F: a NaN operand gives NaN (0x7FC00000); y = +-0 gives
// +-0 for x > 0 or x = +0 and +-pi for x < 0 or x = -0; x = +-0 (y != 0) gives +-pi/2; y = +-inf gives +-pi/4 (x = +inf), +-3 pi/4
// (x = -inf), else +-pi/2; x = +inf (y finite) gives +-0 and x = -inf +-pi; the sign is y's.  Otherwise t = min(|y|, |x|) / max(|y|, |x|)
// in [0, 1]; above tan(pi/8), atan(t) = pi/4 + atan((t - 1) / (t + 1)), so the series argument u has |u| <= tan(pi/8) and
// atan(u) = u + u z P(z), z = u^2 <= 0.1716, by its series to u^45 (truncation below 2^-60 relative); then pi/2 - a when |y| > |x|,
// pi - a when x < 0.  Before the rounding the error is a few units of 2^-53 relative, so the result is within 1 ulp of the exact
// atan2 (tests/test_oracle_sky_ibl.py checks 10^7 inputs against binary64).
OXC_HD float canonical_atan2(float yf, float xf) {
  const double y = (double)yf, x = (double)xf;
  const double PI_D = 3.141592653589793116, PIO2 = dmul64(PI_D, 0.5), PIO4 = dmul64(PI_D, 0.25);
  if (y != y || x != x) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(0x7FC00000u);
#else
    return __builtin_nanf("");
#endif
  }
  const double ay = y < 0.0 ? -y : y, ax = x < 0.0 ? -x : x;
  const double INF = dmul64(1e300, 1e300);
  const bool x_neg = signbit(x);
  double r;
  if (ay == 0.0) r = x_neg ? PI_D : 0.0;
  else if (ay == INF && ax == INF) r = x_neg ? dadd64(PI_D, -PIO4) : PIO4;
  else if (ay == INF || ax == 0.0) r = PIO2;
  else if (ax == INF) r = x_neg ? PI_D : 0.0;
  else {
    const bool swap = ay > ax;
    const double t = swap ? ddiv64(ax, ay) : ddiv64(ay, ax);
    const bool reduce = t > 0.41421356237309503;
    const double u = reduce ? ddiv64(dadd64(t, -1.0), dadd64(t, 1.0)) : t;
    const double z = dmul64(u, u);
    double p = -1.0 / 45.0;
    p = dadd64(1.0 / 43.0, dmul64(z, p));
    p = dadd64(-1.0 / 41.0, dmul64(z, p));
    p = dadd64(1.0 / 39.0, dmul64(z, p));
    p = dadd64(-1.0 / 37.0, dmul64(z, p));
    p = dadd64(1.0 / 35.0, dmul64(z, p));
    p = dadd64(-1.0 / 33.0, dmul64(z, p));
    p = dadd64(1.0 / 31.0, dmul64(z, p));
    p = dadd64(-1.0 / 29.0, dmul64(z, p));
    p = dadd64(1.0 / 27.0, dmul64(z, p));
    p = dadd64(-1.0 / 25.0, dmul64(z, p));
    p = dadd64(1.0 / 23.0, dmul64(z, p));
    p = dadd64(-1.0 / 21.0, dmul64(z, p));
    p = dadd64(1.0 / 19.0, dmul64(z, p));
    p = dadd64(-1.0 / 17.0, dmul64(z, p));
    p = dadd64(1.0 / 15.0, dmul64(z, p));
    p = dadd64(-1.0 / 13.0, dmul64(z, p));
    p = dadd64(1.0 / 11.0, dmul64(z, p));
    p = dadd64(-1.0 / 9.0, dmul64(z, p));
    p = dadd64(1.0 / 7.0, dmul64(z, p));
    p = dadd64(-1.0 / 5.0, dmul64(z, p));
    p = dadd64(1.0 / 3.0, dmul64(z, p)); // P(z) = 1/3 - z/5 + ...; atan(u) = u - u z P(z)
    double a = dadd64(u, -dmul64(dmul64(u, z), p));
    if (reduce) a = dadd64(PIO4, a);
    r = swap ? dadd64(PIO2, -a) : a;
    if (x_neg) r = dadd64(PI_D, -r);
  }
  return d2f_rn(signbit(y) ? -r : r);
}

// cull.slang:169-171: determinant(f32x3x3(c0.xyw, c1.xyw, c2.xyw)) >= 0.0001
OXC_DI bool triangle_backface(float4 c0, float4 c1, float4 c2) {
  const float m00 = c0.x, m01 = c0.y, m02 = c0.w;
  const float m10 = c1.x, m11 = c1.y, m12 = c1.w;
  const float m20 = c2.x, m21 = c2.y, m22 = c2.w;
  const float t0 = fm(m00, fs(fm(m11, m22), fm(m12, m21)));
  const float t1 = fm(m01, fs(fm(m10, m22), fm(m12, m20)));
  const float t2 = fm(m02, fs(fm(m10, m21), fm(m11, m20)));
  return fa(fs(t0, t1), t2) >= 0.0001f;
}

} // namespace oxc
