// filter_soundness.cpp — HOST test of the cull kernel's filtered predicates (oxylus_b200/csrc/oxc_filtered.cuh).
//
// The kernel takes a decision with cheap arithmetic (fma chains, MUFU rcp / rsqrt) whenever an error bound proves that the
// canonical evaluation — the one the CPU oracle restates and every GPU parity test compares against — must agree, and falls
// back to the canonical path otherwise.  "Bit-identical for EVERY input" therefore rests on those bounds.  The GPU tests only
// ever see what one GPU's MUFU returns; this program compiles the very same device headers for the host (tests/host_shim/:
// each __f*_rn intrinsic is one IEEE binary32 operation under -ffp-contract=off, fmaf is exact) and replaces the two
// approximate units by an ADVERSARY that returns any float the PTX ISA's accuracy statement allows (rcp.approx: 2^-23
// relative, rsqrt.approx: 2^-22.4 relative, subnormal results flushed): always the lowest, always the highest, the nearest,
// or a random admissible neighbour per call.  Inputs are random scenes plus points bisected onto each predicate's decision
// boundary and stepped across it ulp by ulp.  Any decided (non-ambiguous) answer that differs from the canonical one is a
// failure.  Test infrastructure only; built and run by tests/test_filter_soundness_cpu.py.
//
//   g++ -O2 -std=c++17 -ffp-contract=off -I tests/host_shim -I oxylus_b200/csrc tests/filter_soundness.cpp -o filter_soundness
//   ./filter_soundness [cases per predicate, default 400000] [seed]
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define OXC_HOST_SOUNDNESS_HARNESS
#include "oxc_filtered.cuh"

namespace {

// SplitMix64
struct Rng {
  uint64_t s;
  explicit Rng(uint64_t seed) : s(seed) {}
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double uniform() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
  double range(double a, double b) { return a + (b - a) * uniform(); }
  uint32_t below(uint32_t n) { return (uint32_t)(next() % n); }
};

enum Mode { NEAREST = 0, LOWEST = 1, HIGHEST = 2, RANDOM = 3, ALTERNATE = 4, N_MODES = 5 };
int g_mode = NEAREST;
Rng g_adversary(7);
uint32_t g_calls = 0;

float step_ulps(float f, int k) {
  uint32_t u = __float_as_uint(f);
  // positive finite floats are ordered like their bit patterns (the units are only called with positive arguments)
  return __uint_as_float((uint32_t)((int64_t)u + k));
}

// any float within `rel` of the true value; subnormal results are flushed (".ftz")
float admissible(double truth, double rel) {
  const float nearest = (float)truth;
  float cand[9];
  int n = 0;
  for (int k = -4; k <= 4; k++) {
    const float c = step_ulps(nearest, k);
    if (!(c > 0.0f) || c != c || c > 3.4e38f) continue;
    const double err = (double)c - truth;
    if ((err < 0 ? -err : err) <= rel * truth) cand[n++] = c;
  }
  float r = nearest;
  if (n) {
    int pick = 0;
    switch (g_mode) {
      case LOWEST: pick = 0; break;
      case HIGHEST: pick = n - 1; break;
      case RANDOM: pick = (int)g_adversary.below((uint32_t)n); break;
      case ALTERNATE: pick = (g_calls++ & 1) ? n - 1 : 0; break;
      default: { // nearest among the admissible ones
        double best = 1e300;
        for (int i = 0; i < n; i++) { const double e = (double)cand[i] - truth; if ((e < 0 ? -e : e) < best) { best = e < 0 ? -e : e; pick = i; } }
      }
    }
    r = cand[pick];
  }
  if (r < 1.17549435e-38f) r = 0.0f;
  return r;
}

} // namespace

namespace oxc {
float rcp_approx(float x) {
  if (!(x > 0.0f) || x > 3.4e38f) return 1.0f / x; // never reached through the filters' preconditions; keep IEEE semantics
  if (x < 1.17549435e-38f) return __uint_as_float(0x7F800000u);
  return admissible(1.0 / (double)x, 1.1920928955078125e-07); // 2^-23
}
float rsqrt_approx(float x) {
  if (!(x > 0.0f) || x > 3.4e38f) return 1.0f / sqrtf(x);
  if (x < 1.17549435e-38f) return __uint_as_float(0x7F800000u);
  return admissible(1.0 / sqrt((double)x), 1.8064e-07); // 2^-22.4
}
} // namespace oxc

namespace {
using namespace oxc;

struct Counters {
  uint64_t cases = 0, decided = 0, ambiguous = 0, wrong = 0;
};

float random_half_value(Rng& r, double lo, double hi) { // a value a MeshletBounds field can hold: dequantised half
  const float f = (float)r.range(lo, hi);
  // round through half precision by bit tricks (truncate the mantissa to 10 bits: exact halves in the normal range)
  uint32_t u = __float_as_uint(f) & 0xFFFFE000u;
  const float h = __uint_as_float(u);
  return fabsf(h) < 6.2e-5f ? 0.0f : h;
}

// column-major 4x4 helpers (CullCamera / TransformWorld storage)
void perspective_reverse_z(float* m, double fovy, double aspect, double zn, double zf) { // Camera.cpp:36-54 shape: reverse-Z, y flipped
  for (int i = 0; i < 16; i++) m[i] = 0.0f;
  const double f = 1.0 / tan(fovy * 0.5);
  m[0] = (float)(f / aspect);
  m[5] = (float)(-f);
  m[10] = (float)(zn / (zf - zn));
  m[11] = -1.0f;
  m[14] = (float)(zf * zn / (zf - zn));
}
void random_world(Rng& r, float* m, double spread) {
  // random rotation (from a random unit quaternion) x uniform scale x translation in front of the camera
  double q[4], n = 0;
  for (double& c : q) { c = r.range(-1, 1); n += c * c; }
  n = sqrt(n);
  for (double& c : q) c /= n;
  const double s = r.range(0.5, 2.0);
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w), 2 * (x * y + z * w), 1 - 2 * (x * x + z * z),
                       2 * (y * z - x * w), 2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
  for (int c = 0; c < 3; c++)
    for (int rr = 0; rr < 3; rr++) m[c * 4 + rr] = (float)(R[rr * 3 + c] * s);
  m[3] = m[7] = m[11] = 0.0f;
  m[12] = (float)r.range(-spread, spread);
  m[13] = (float)r.range(-spread * 0.3, spread * 0.3);
  m[14] = (float)r.range(-2.0 * spread, 2.0);
  m[15] = 1.0f;
}

struct Instance {
  float world[16];
  InstCull ic;
};

void make_instance(Rng& r, const float* pv, Instance& in, double spread) {
  random_world(r, in.world, spread);
  float4 rows[4];
  mul_mm_rows(pv, in.world, rows);
  for (int i = 0; i < 4; i++) in.ic.mvp_row[i] = rows[i];
  frustum_planes(rows, in.ic.plane);
  const float* w = in.world;
  for (int i = 0; i < 3; i++) in.ic.world_row[i] = make_float4(w[0 * 4 + i], w[1 * 4 + i], w[2 * 4 + i], w[3 * 4 + i]);
  // normal matrix rows = cross products of the world's columns (scene.slang:291-298), max row length in nrm[0].w
  const float c0[3] = {w[0], w[1], w[2]}, c1[3] = {w[4], w[5], w[6]}, c2[3] = {w[8], w[9], w[10]};
  auto crossf = [](const float* a, const float* b, float* o) {
    o[0] = fs(fm(a[1], b[2]), fm(a[2], b[1])); o[1] = fs(fm(a[2], b[0]), fm(a[0], b[2])); o[2] = fs(fm(a[0], b[1]), fm(a[1], b[0]));
  };
  float n0[3], n1[3], n2[3];
  crossf(c1, c2, n0); crossf(c2, c0, n1); crossf(c0, c1, n2);
  const float l0 = length3(c0[0], c0[1], c0[2]), l1 = length3(c1[0], c1[1], c1[2]), l2 = length3(c2[0], c2[1], c2[2]);
  in.ic.nrm[0] = make_float4(n0[0], n0[1], n0[2], omax(omax(l0, l1), l2));
  in.ic.nrm[1] = make_float4(n1[0], n1[1], n1[2], 1.0f);
  in.ic.nrm[2] = make_float4(n2[0], n2[1], n2[2], 0.0f);
}

struct Pyramid {
  uint32_t w, h, levels;
  uint32_t off[OXC_HIZ_MAX_LEVELS];
  std::vector<float> data;
  void build(uint32_t w_, uint32_t h_) {
    w = w_; h = h_;
    levels = 0;
    uint32_t total = 0;
    for (uint32_t mw = w, mh = h;; mw = mw > 1 ? mw / 2 : 1, mh = mh > 1 ? mh / 2 : 1) {
      off[levels++] = total;
      total += mw * mh;
      if (mw == 1 && mh == 1) break;
    }
    data.assign(total, 0.0f);
  }
  void fill_random(Rng& r, float lo, float hi) { for (float& d : data) d = (float)r.range(lo, hi); }
  // every texel either occludes everything (1) or nothing (0): the answer is "does the 4-tap footprint hold a 0", so a footprint
  // that moves by one texel, or to another mip, flips it with high probability
  void fill_binary(Rng& r, double p_zero) { for (float& d : data) d = r.uniform() < p_zero ? 0.0f : 1.0f; }
  void fill_constant(float v) { for (float& d : data) d = v; }
};

bool exact_visible(const InstCull& ic, float near_clip, const float* b, const Pyramid& p) {
  ScreenAabb a;
  if (!project_aabb(ic.mvp_row[0], ic.mvp_row[1], ic.mvp_row[2], ic.mvp_row[3], near_clip, b[0], b[1], b[2], b[3], b[4], b[5], a)) return true;
  return !test_occlusion(a, p.data.data(), p.w, p.h, p.levels, p.off);
}

void check(Counters& c, Tri fast, bool exact, const char* what) {
  c.cases++;
  if (fast == TRI_AMBIGUOUS) { c.ambiguous++; return; }
  c.decided++;
  if ((fast == TRI_TRUE) != exact) {
    if (c.wrong < 5) std::fprintf(stderr, "WRONG %s: fast says %s, canonical says %s (mode %d)\n", what, fast == TRI_TRUE ? "true" : "false", exact ? "true" : "false", g_mode);
    c.wrong++;
  }
}

void random_bounds(Rng& r, float* b, double centre_range, double emin, double emax) {
  for (int a = 0; a < 3; a++) b[a] = random_half_value(r, -centre_range, centre_range);
  for (int a = 0; a < 3; a++) {
    const double e = emin * pow(emax / emin, r.uniform());
    b[3 + a] = random_half_value(r, e, e * 1.0001 + 1e-9);
  }
  // one box in 16 carries a value no mesh builder produces but a MeshletBounds record can hold: the canonical evaluation is
  // defined for it, so the fast paths must either agree or step aside (negative / NaN / infinite / denormal-flushed fields)
  if (r.below(16) == 0) {
    static const uint32_t specials[] = {0x0000, 0x8000, 0x7BFF, 0xFBFF, 0x7C00, 0xFC00, 0x7E00, 0xBC00, 0xB800, 0x0400, 0x8400};
    const int n = 1 + (int)r.below(2);
    for (int k = 0; k < n; k++) b[r.below(6)] = dequantize_half(specials[r.below(11)]);
  }
}

// ------------------------------------------------------------------------------------------------ occlusion
void run_occlusion(Rng& r, uint64_t n, Counters& c) {
  Pyramid pyr;
  float pv[16];
  Instance in;
  for (uint64_t i = 0; i < n; i++) {
    if (i % 4096 == 0) {
      static const uint32_t sizes[][2] = {{1024, 1024}, {2048, 2048}, {256, 128}, {64, 64}, {4096, 2048}};
      const uint32_t* s = sizes[r.below(5)];
      pyr.build(s[0], s[1]);
      if (r.below(2)) pyr.fill_random(r, 0.0f, 0.2f);
      else pyr.fill_binary(r, 0.16);
      perspective_reverse_z(pv, r.range(0.6, 1.5), r.range(1.0, 2.4), 0.1, r.range(100.0, 2000.0));
    }
    if (i % 64 == 0) make_instance(r, pv, in, i % 128 ? 40.0 : 4.0);
    float b[6];
    random_bounds(r, b, 4.0, 0.02, 2.0);
    const float near_clip = 0.1f;
    // (a) random pyramid
    const bool mvp_ok = true;
    for (g_mode = 0; g_mode < N_MODES; g_mode++) {
      const Tri t = occlusion_visible_fast(in.ic.mvp_row[0], in.ic.mvp_row[1], in.ic.mvp_row[2], in.ic.mvp_row[3], near_clip, b[0], b[1], b[2], b[3], b[4],
                                           b[5], pyr.data.data(), pyr.w, pyr.h, pyr.levels, pyr.off, mvp_ok);
      check(c, t, exact_visible(in.ic, near_clip, b, pyr), "occlusion (random pyramid)");
    }
    // (a') texel boundaries: slide the box along x until the canonical min / max texel column changes, bisect the change down to
    // adjacent floats of the centre, step across it (the fast divide may land on the other side of the integer)
    if (i % 4 == 2) {
      auto texels = [&](float cx, uint32_t& lo_t, uint32_t& hi_t) {
        ScreenAabb sa;
        if (!project_aabb(in.ic.mvp_row[0], in.ic.mvp_row[1], in.ic.mvp_row[2], in.ic.mvp_row[3], near_clip, cx, b[1], b[2], b[3], b[4], b[5], sa)) return false;
        const float hw = (float)pyr.w;
        lo_t = __float2uint_rz(omax(fm(sa.minx, hw), 0.0f));
        hi_t = __float2uint_rz(omin(fm(sa.maxx, hw), fs(hw, 1.0f)));
        return true;
      };
      uint32_t l0, h0, l1, h1;
      if (texels(b[0], l0, h0)) {
        float lo = b[0], hi = b[0];
        bool found = false;
        for (float d = 1e-4f; d < 8.0f; d *= 2.0f) {
          if (!texels(b[0] + d, l1, h1)) break;
          if (l1 != l0 || h1 != h0) { hi = b[0] + d; found = true; break; }
          lo = b[0] + d;
        }
        if (found) {
          for (int it = 0; it < 48; it++) {
            const float mid = 0.5f * (lo + hi);
            if (mid == lo || mid == hi) break;
            if (!texels(mid, l1, h1)) break;
            if (l1 != l0 || h1 != h0) hi = mid; else lo = mid;
          }
          for (int e = -12; e <= 12; e++) {
            const int k = e == 0 ? 0 : (e < 0 ? -(1 << (-e - 1)) : (1 << (e - 1)));
            const uint32_t u = __float_as_uint(lo);
            const float x = __uint_as_float((uint32_t)((int64_t)u + ((u & 0x80000000u) ? -k : k)));
            const float bb[6] = {x, b[1], b[2], b[3], b[4], b[5]};
            for (g_mode = 0; g_mode < N_MODES; g_mode++) {
              const Tri t = occlusion_visible_fast(in.ic.mvp_row[0], in.ic.mvp_row[1], in.ic.mvp_row[2], in.ic.mvp_row[3], near_clip, bb[0], bb[1], bb[2], bb[3],
                                                   bb[4], bb[5], pyr.data.data(), pyr.w, pyr.h, pyr.levels, pyr.off, mvp_ok);
              check(c, t, exact_visible(in.ic, near_clip, bb, pyr), "occlusion (texel boundary)");
            }
          }
        }
      }
    }
    // (b) the final depth compare on its boundary: every texel = max.z of this box, stepped a few ulps either way
    ScreenAabb a;
    if (i % 8 == 0 && project_aabb(in.ic.mvp_row[0], in.ic.mvp_row[1], in.ic.mvp_row[2], in.ic.mvp_row[3], near_clip, b[0], b[1], b[2], b[3], b[4], b[5], a) &&
        a.maxz > 1e-6f && a.maxz < 1.0f) {
      Pyramid flat;
      flat.build(64, 64);
      static const int steps[] = {0, 1, 2, 3, 4, 5, 6, 8, 12, 16, 24, 32, 64};
      for (int ks = -12; ks <= 12; ks++) {
        const int k = ks < 0 ? -steps[-ks] : steps[ks];
        flat.fill_constant(step_ulps(a.maxz + 1e-7f, k));
        for (g_mode = 0; g_mode < N_MODES; g_mode++) {
          const Tri t = occlusion_visible_fast(in.ic.mvp_row[0], in.ic.mvp_row[1], in.ic.mvp_row[2], in.ic.mvp_row[3], near_clip, b[0], b[1], b[2], b[3],
                                               b[4], b[5], flat.data.data(), flat.w, flat.h, flat.levels, flat.off, mvp_ok);
          check(c, t, exact_visible(in.ic, near_clip, b, flat), "occlusion (depth boundary)");
        }
      }
    }
    // (c) the cleared-pyramid shortcut: "surely visible" must imply the canonical answer against an all-zero pyramid
    if (i % 8 == 1) {
      Pyramid zero;
      zero.build(64, 64);
      c.cases++;
      if (cleared_hiz_surely_visible(in.ic.mvp_row[2], in.ic.mvp_row[3], b[0], b[1], b[2], b[3], b[4], b[5])) {
        c.decided++;
        if (!exact_visible(in.ic, near_clip, b, zero)) { c.wrong++; std::fprintf(stderr, "WRONG cleared-Hi-Z shortcut\n"); }
      } else c.ambiguous++;
    }
  }
}

// ------------------------------------------------------------------------------------------------ cone
void run_cone(Rng& r, uint64_t n, Counters& c) {
  float pv[16];
  perspective_reverse_z(pv, 1.0, 1.7, 0.1, 1000.0);
  Instance in;
  float lut[256];
  for (int v = -128; v < 128; v++) lut[v + 128] = s8_over_127(v);
  for (uint64_t i = 0; i < n; i++) {
    if (i % 32 == 0) make_instance(r, pv, in, 40.0);
    float b[6];
    random_bounds(r, b, 4.0, 0.02, 2.0);
    // s8 cone axis of roughly unit length, s8 cutoff below 127 (127 = test disabled)
    double ax[3], l = 0;
    for (double& a : ax) { a = r.range(-1, 1); l += a * a; }
    l = sqrt(l);
    const float axis[3] = {lut[(int)lrint(ax[0] / l * 127) + 128], lut[(int)lrint(ax[1] / l * 127) + 128], lut[(int)lrint(ax[2] / l * 127) + 128]};
    const float cutoff = lut[(int)r.below(254) - 127 + 128];
    float cam[3] = {(float)r.range(-30, 30), (float)r.range(-10, 10), (float)r.range(-30, 30)};
    auto eval = [&](const float* campos) {
      const ConeInputs ci = cone_inputs(&in.ic, b[0], b[1], b[2], b[3], b[4], b[5], axis[0], axis[1], axis[2], campos[0], campos[1], campos[2]);
      const bool exact = cone_visible_exact(ci, cutoff);
      for (g_mode = 0; g_mode < N_MODES; g_mode++) check(c, cone_visible_fast(ci, cutoff), exact, "cone");
      return exact;
    };
    const bool v0 = eval(cam);
    // walk the camera along a random line until the canonical answer flips, bisect the flip down to adjacent floats of the line
    // parameter, then step across it
    double dir[3] = {r.range(-1, 1), r.range(-1, 1), r.range(-1, 1)};
    float lo = 0.0f, hi = 0.0f;
    bool found = false;
    for (float t = 0.5f; t < 400.0f; t *= 1.7f) {
      const float p[3] = {(float)(cam[0] + dir[0] * t), (float)(cam[1] + dir[1] * t), (float)(cam[2] + dir[2] * t)};
      const ConeInputs ci = cone_inputs(&in.ic, b[0], b[1], b[2], b[3], b[4], b[5], axis[0], axis[1], axis[2], p[0], p[1], p[2]);
      if (cone_visible_exact(ci, cutoff) != v0) { hi = t; found = true; break; }
      lo = t;
    }
    if (!found) continue;
    for (int it = 0; it < 40; it++) {
      const float mid = 0.5f * (lo + hi);
      if (mid == lo || mid == hi) break;
      const float p[3] = {(float)(cam[0] + dir[0] * mid), (float)(cam[1] + dir[1] * mid), (float)(cam[2] + dir[2] * mid)};
      const ConeInputs ci = cone_inputs(&in.ic, b[0], b[1], b[2], b[3], b[4], b[5], axis[0], axis[1], axis[2], p[0], p[1], p[2]);
      if (cone_visible_exact(ci, cutoff) != v0) hi = mid; else lo = mid;
    }
    for (int e = -16; e <= 16; e++) { // 0, +-1, +-2, +-4 ... +-2^15 ulps of the line parameter: inside and just outside the margin
      const int k = e == 0 ? 0 : (e < 0 ? -(1 << (-e - 1)) : (1 << (e - 1)));
      const float t = step_ulps(lo, k);
      if (!(t > 0.0f)) continue;
      const float p[3] = {(float)(cam[0] + dir[0] * t), (float)(cam[1] + dir[1] * t), (float)(cam[2] + dir[2] * t)};
      eval(p);
    }
  }
}

// ------------------------------------------------------------------------------------------------ frustum (centre-inside filter)
void run_frustum(Rng& r, uint64_t n, Counters& c) {
  float pv[16];
  Instance in;
  for (uint64_t i = 0; i < n; i++) {
    if (i % 1024 == 0) perspective_reverse_z(pv, r.range(0.6, 1.5), r.range(1.0, 2.4), 0.1, r.range(100.0, 2000.0));
    if (i % 16 == 0) make_instance(r, pv, in, i % 32 ? 60.0 : 6.0);
    float b[6];
    random_bounds(r, b, 4.0, 0.02, 2.0);
    // flat and point-like boxes (extent 0 is a legitimate MeshletBounds value): there the box's p-vertex IS its centre and the
    // filter's margin is all that separates "inside" from the canonical reject
    if (i % 4 == 0) b[3] = b[4] = b[5] = 0.0f;
    else if (i % 4 == 1) b[3 + r.below(3)] = 0.0f;
    else if (i % 4 == 2) { b[3] = 6.1035e-05f; b[4] = b[5] = 0.0f; }
    auto eval = [&](const float* bb) {
      const bool exact = test_frustum_planes(in.ic.plane, bb[0], bb[1], bb[2], bb[3], bb[4], bb[5]);
      c.cases++;
      if (frustum_centre_inside(in.ic.plane, bb[0], bb[1], bb[2], bb[3], bb[4], bb[5])) {
        c.decided++;
        if (!exact) { c.wrong++; if (c.wrong < 5) std::fprintf(stderr, "WRONG frustum centre-inside filter\n"); }
      } else c.ambiguous++;
      return exact;
    };
    const bool v0 = eval(b);
    // slide the box centre along x until the canonical answer flips; bisect; step across (centres here need not be halves: the
    // filter's bound does not depend on it)
    float lo = b[0], hi = b[0];
    bool found = false;
    for (float d = 0.25f; d < 4096.0f; d *= 2.0f) {
      float bb[6] = {b[0] + d, b[1], b[2], b[3], b[4], b[5]};
      if (test_frustum_planes(in.ic.plane, bb[0], bb[1], bb[2], bb[3], bb[4], bb[5]) != v0) { hi = bb[0]; found = true; break; }
      lo = bb[0];
    }
    if (!found) continue;
    for (int it = 0; it < 48; it++) {
      const float mid = 0.5f * (lo + hi);
      if (mid == lo || mid == hi) break;
      if (test_frustum_planes(in.ic.plane, mid, b[1], b[2], b[3], b[4], b[5]) != v0) hi = mid; else lo = mid;
    }
    for (int e = -14; e <= 14; e++) {
      const int k = e == 0 ? 0 : (e < 0 ? -(1 << (-e - 1)) : (1 << (e - 1)));
      uint32_t u = __float_as_uint(lo);
      const float x = __uint_as_float((uint32_t)((int64_t)u + ((u & 0x80000000u) ? -k : k)));
      const float bb[6] = {x, b[1], b[2], b[3], b[4], b[5]};
      eval(bb);
    }
  }
}

// ------------------------------------------------------------------------------------------------ whole-instance shortcut
// union_box_inside_frustum(U) == true must imply that EVERY box inside U passes the canonical per-meshlet frustum test.  The
// worst boxes are the zero-extent ones at U's corners (the n-vertex corner in particular) and U itself.
void run_instance_inside(Rng& r, uint64_t n, Counters& c) {
  float pv[16];
  Instance in;
  for (uint64_t i = 0; i < n; i++) {
    if (i % 1024 == 0) perspective_reverse_z(pv, r.range(0.6, 1.5), r.range(1.0, 2.4), 0.1, r.range(100.0, 2000.0));
    if (i % 8 == 0) make_instance(r, pv, in, i % 16 ? 30.0 : 4.0);
    float u[6];
    for (int a = 0; a < 3; a++) {
      const float x0 = random_half_value(r, -4, 4), x1 = random_half_value(r, -4, 4);
      u[a] = omin(x0, x1); u[3 + a] = omax(x0, x1);
      if (i % 5 == 0) u[3 + a] = u[a]; // degenerate union box
    }
    auto probe = [&](const float* ua) {
      c.cases++;
      if (!union_box_inside_frustum(in.ic.plane, ua, true)) { c.ambiguous++; return false; }
      c.decided++;
      bool ok = true;
      for (int k = 0; k < 8 && ok; k++) { // corners, zero extent
        const float cx = (k & 1) ? ua[3] : ua[0], cy = (k & 2) ? ua[4] : ua[1], cz = (k & 4) ? ua[5] : ua[2];
        ok = test_frustum_planes(in.ic.plane, cx, cy, cz, 0.0f, 0.0f, 0.0f);
      }
      // U itself and random boxes inside it (centre / extent rounded like MeshletBounds fields, kept inside U after decoding)
      for (int k = 0; k < 6 && ok; k++) {
        float bb[6];
        for (int a = 0; a < 3; a++) {
          float lo_ = ua[a], hi_ = ua[3 + a];
          if (k) { const float x0 = (float)r.range(lo_, hi_), x1 = (float)r.range(lo_, hi_); lo_ = omin(x0, x1); hi_ = omax(x0, x1); }
          float cc = fm(fa(lo_, hi_), 0.5f), ee = fs(hi_, lo_);
          while (ee > 0.0f && (fs(cc, fm(ee, 0.5f)) < ua[a] || fa(cc, fm(ee, 0.5f)) > ua[3 + a])) ee = fm(ee, 0.99f);
          if (fs(cc, fm(ee, 0.5f)) < ua[a] || fa(cc, fm(ee, 0.5f)) > ua[3 + a]) ee = 0.0f;
          bb[a] = cc; bb[3 + a] = ee;
        }
        ok = test_frustum_planes(in.ic.plane, bb[0], bb[1], bb[2], bb[3], bb[4], bb[5]);
      }
      if (!ok) { c.wrong++; if (c.wrong < 5) std::fprintf(stderr, "WRONG whole-instance frustum shortcut\n"); }
      return true;
    };
    const bool v0 = probe(u);
    // slide U along x until the shortcut's answer flips, bisect, step across
    float lo = 0.0f, hi = 0.0f;
    bool found = false;
    for (float d = 0.25f; d < 4096.0f; d *= 2.0f) {
      const float uu[6] = {u[0] + d, u[1], u[2], u[3] + d, u[4], u[5]};
      if (union_box_inside_frustum(in.ic.plane, uu, true) != v0) { hi = d; found = true; break; }
      lo = d;
    }
    if (!found) continue;
    for (int it = 0; it < 48; it++) {
      const float mid = 0.5f * (lo + hi);
      if (mid == lo || mid == hi) break;
      const float uu[6] = {u[0] + mid, u[1], u[2], u[3] + mid, u[4], u[5]};
      if (union_box_inside_frustum(in.ic.plane, uu, true) != v0) hi = mid; else lo = mid;
    }
    for (int e = -10; e <= 10; e++) {
      const int k = e == 0 ? 0 : (e < 0 ? -(1 << (-e - 1)) : (1 << (e - 1)));
      const float d = step_ulps(lo > 0.0f ? lo : 1e-6f, k);
      const float uu[6] = {u[0] + d, u[1], u[2], u[3] + d, u[4], u[5]};
      probe(uu);
    }
  }
}

} // namespace

int main(int argc, char** argv) {
  const uint64_t n = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 400000ull;
  const uint64_t seed = argc > 2 ? std::strtoull(argv[2], nullptr, 10) : 0x0C115EEDull;
  Rng r(seed);
  Counters occ, cone, fr, inst;
  run_occlusion(r, n, occ);
  run_cone(r, n, cone);
  run_frustum(r, n, fr);
  run_instance_inside(r, n / 4, inst);
  auto line = [](const char* name, const Counters& c) {
    std::printf("%-10s evaluations %10llu  decided %10llu (%.1f %%)  ambiguous %10llu  wrong %llu\n", name, (unsigned long long)c.cases,
                (unsigned long long)c.decided, 100.0 * (double)c.decided / (double)(c.cases ? c.cases : 1), (unsigned long long)c.ambiguous,
                (unsigned long long)c.wrong);
  };
  line("occlusion", occ);
  line("cone", cone);
  line("frustum", fr);
  line("instance", inst);
  const uint64_t wrong = occ.wrong + cone.wrong + fr.wrong + inst.wrong;
  std::printf("%s\n", wrong ? "FAILED" : "ok");
  return wrong ? 1 : 0;
}
