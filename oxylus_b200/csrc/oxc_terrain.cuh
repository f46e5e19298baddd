// oxc_terrain.cuh — the terrain's vis-buffer draw (passes/terrain_visbuffer.slang via Passes/Terrain.cpp:218-277): per patch the
// corners, the tessellation factors and their fractional_odd rounding, per triangle its domain points, heights and clip positions, as
// include/oxcull.h oxc_draw_terrain specifies (items 1-7) and oracle/oxc_oracle_terrain_draw.c computes.  kernels_terrain.cuh
// schedules these functions over CTAs.
// No warp intrinsics, no shared memory: tests compile this source for the host.
#pragma once
#include "oxc_raster_core.cuh"
#include "oxc_shader_math.cuh"

namespace oxc {

constexpr float TERRAIN_MAX_FACTOR = 63.0f;         // item 2: maxTessellationGenerationLevel 64, minus one for odd spacing
constexpr float TERRAIN_ONE_PLUS_EPS = 0x1.000002p0f; // item 2: an inner factor of 1 beside a subdivided edge
constexpr float TERRAIN_DEG_TO_RAD = 0x1.1df46ap-6f;   // item 1: radians(x) = x * (pi / 180), 0x3C8EFA35

struct TerrainDrawParams {
  const uint16_t* heightmap;
  int res_x, res_y;
  float world_min[2], world_size[2], inv_world_size[2];
  uint32_t patch_count[2], patch_total;
  float base_height, height_scale, target_edge_pixels, max_tessellation;
  float4 pv_row[4];            // rows of projection_view
  float cam_pos[3], near_clip;
  float projection_scale;      // item 1: camera.resolution.y * 0.5 / tan(radians(fov) * 0.5), formed once per call
  const uint32_t* visible_patches;
  const OxcDrawIndirectCommand* draw_cmd;
  unsigned long long* vis;
  uint32_t width, height;
  float fW, fH;
  uint32_t data;               // item 5: TERRAIN_INSTANCE_ID << prim_bits
};

// item 1: tan through the canonical sin / cos, on the host once per call
inline float terrain_projection_scale(float fov_degrees, float resolution_y) {
  const float half = (fov_degrees * TERRAIN_DEG_TO_RAD) * 0.5f;
  float s, c;
  canonical_sincos(half, s, c);
  return (resolution_y * 0.5f) / (s / c);
}

// the kernel's parameters from the arguments of oxc_draw_terrain (checked by the caller); prim_bits 8 or 6
inline TerrainDrawParams terrain_make_params(const uint16_t* heightmap, uint32_t res_x, uint32_t res_y, const OxcTerrainDrawSettings& s,
                                             const uint32_t* visible_patches, const OxcDrawIndirectCommand* draw_cmd,
                                             const OxcCullCamera& cam, uint32_t w, uint32_t h, uint64_t* vis, uint32_t prim_bits) {
  TerrainDrawParams p{};
  p.heightmap = heightmap;
  p.res_x = (int)res_x;
  p.res_y = (int)res_y;
  for (int k = 0; k < 2; k++) {
    p.world_min[k] = s.terrain.world_min[k];
    p.world_size[k] = s.terrain.world_size[k];
    p.inv_world_size[k] = s.inv_world_size[k];
    p.patch_count[k] = s.terrain.patch_count[k];
  }
  p.patch_total = s.terrain.patch_count[0] * s.terrain.patch_count[1];
  p.base_height = s.terrain.base_height;
  p.height_scale = s.terrain.height_scale;
  p.target_edge_pixels = s.target_edge_pixels;
  p.max_tessellation = s.max_tessellation;
  const float* m = cam.projection_view; // column-major: row i = (m[i], m[4+i], m[8+i], m[12+i])
  for (int i = 0; i < 4; i++) p.pv_row[i] = make_float4(m[i], m[4 + i], m[8 + i], m[12 + i]);
  for (int k = 0; k < 3; k++) p.cam_pos[k] = cam.position[k];
  p.near_clip = cam.near_clip;
  p.projection_scale = terrain_projection_scale(s.fov, cam.resolution[1]);
  p.visible_patches = visible_patches;
  p.draw_cmd = draw_cmd;
  p.vis = reinterpret_cast<unsigned long long*>(vis);
  p.width = w;
  p.height = h;
  p.fW = (float)w;
  p.fH = (float)h;
  p.data = ((0xFFFFFFFFu >> prim_bits) - 1u) << prim_bits;
  return p;
}

// item 4: lerp(a, b, t) = a * (1 - t) + b * t; t = 1 gives b and t = 0 gives a exactly, so patches agree on their shared edges
OXC_DI float terrain_lerp(float a, float b, float t) { return fa(fm(a, fs(1.0f, t)), fm(b, t)); }

// item 4: sample_height(world_xz) = base_height + SampleLevel(world_to_uv(xz), 0) * height_scale
OXC_DI float terrain_height(const TerrainDrawParams& p, float x, float z) {
  const float u = fm(fs(x, p.world_min[0]), p.inv_world_size[0]), v = fm(fs(z, p.world_min[1]), p.inv_world_size[1]);
  return fa(p.base_height, fm(bilinear_tap_r16<CLAMP_TO_EDGE>(p.heightmap, p.res_x, p.res_y, u, v), p.height_scale));
}

// item 1: edge_tessellation(a, b), clamped to [1, max_tessellation] (a NaN quotient gives 1)
OXC_DI float terrain_edge_factor(const TerrainDrawParams& p, Vec3 a, Vec3 b) {
  const Vec3 center = vscale(vadd(a, b), 0.5f);
  const float radius = fm(vlength(vsub(a, b)), 0.5f);
  const float view_distance = vmax(fs(vlength(vsub(center, vec3(p.cam_pos[0], p.cam_pos[1], p.cam_pos[2]))), radius), p.near_clip);
  const float projected = fd(fm(fm(2.0f, radius), p.projection_scale), view_distance);
  return vmin(vmax(fd(projected, p.target_edge_pixels), 1.0f), p.max_tessellation);
}

// item 2: a factor pinned to [1, 63] (NaN -> 1) and its odd rounding 2 * ceil((f - 1) / 2) + 1 (f - 1 and the halving are exact)
OXC_DI float terrain_factor_clamp(float f) { return !(f >= 1.0f) ? 1.0f : (f > TERRAIN_MAX_FACTOR ? TERRAIN_MAX_FACTOR : f); }
OXC_DI int terrain_round_odd(float f) { return 2 * (int)ceilf(fm(fs(terrain_factor_clamp(f), 1.0f), 0.5f)) + 1; }

// item 3: domain point k in [0, n] of an edge of clamped factor f rounded to n: 0, then s + (k - 1) * L up to the middle, the mirror
// image 1 - t(n - k) past it, and 1; L = 1 / f, s = (f - (n - 2)) / (2 f) > 0 (f > n - 2)
OXC_DI float terrain_edge_point(float f, int n, int k) {
  if (k <= 0) return 0.0f;
  if (k >= n) return 1.0f;
  const bool mirror = 2 * k > n;
  const int kk = mirror ? n - k : k;
  const float L = fd(1.0f, f), s = fd(fs(f, (float)(n - 2)), fm(2.0f, f));
  const float t = fa(s, fm((float)(kk - 1), L));
  return mirror ? fs(1.0f, t) : t;
}

// item 1 and 2 for one patch: corners (x, z), clamped factors and their odd roundings, the triangle count of item 3's order
struct TerrainPatch {
  float px[4], pz[4];        // p0 = (0, 0), p1 = (1, 0), p2 = (1, 1), p3 = (0, 1)
  float f_edge[4], f_in[2];  // edges u0 = (p0, p3), v0 = (p0, p1), u1 = (p1, p2), v1 = (p3, p2); inner along u, along v
  int n_edge[4], n_in[2];
  uint32_t tri_count;
};

OXC_DI void terrain_patch_setup(const TerrainDrawParams& p, uint32_t patch_index, TerrainPatch& t) {
  const uint32_t ix = patch_index % p.patch_count[0], iz = patch_index / p.patch_count[0];
  const float cx = (float)p.patch_count[0], cz = (float)p.patch_count[1];
  Vec3 c[4];
  for (int k = 0; k < 4; k++) {
    const uint32_t dx = (k == 1 || k == 2) ? 1u : 0u, dz = k >= 2 ? 1u : 0u;
    t.px[k] = fa(p.world_min[0], fm(fd((float)(ix + dx), cx), p.world_size[0]));
    t.pz[k] = fa(p.world_min[1], fm(fd((float)(iz + dz), cz), p.world_size[1]));
    c[k] = vec3(t.px[k], terrain_height(p, t.px[k], t.pz[k]), t.pz[k]);
  }
  const float e[4] = {terrain_edge_factor(p, c[0], c[3]), terrain_edge_factor(p, c[0], c[1]), terrain_edge_factor(p, c[1], c[2]),
                      terrain_edge_factor(p, c[3], c[2])};
  const float in[2] = {vmax(e[1], e[3]), vmax(e[0], e[2])};
  bool all_one = true;
  for (int k = 0; k < 4; k++) {
    t.f_edge[k] = terrain_factor_clamp(e[k]);
    t.n_edge[k] = terrain_round_odd(t.f_edge[k]);
    all_one = all_one && t.n_edge[k] == 1;
  }
  for (int k = 0; k < 2; k++) {
    t.f_in[k] = terrain_factor_clamp(in[k]);
    t.n_in[k] = terrain_round_odd(t.f_in[k]);
    all_one = all_one && t.n_in[k] == 1;
  }
  if (all_one) {
    t.tri_count = 2;
    return;
  }
  for (int k = 0; k < 2; k++)
    if (t.n_in[k] == 1) { t.f_in[k] = TERRAIN_ONE_PLUS_EPS; t.n_in[k] = 3; }
  const uint32_t iu = (uint32_t)t.n_in[0] - 2u, iv = (uint32_t)t.n_in[1] - 2u;
  t.tri_count = (uint32_t)(t.n_edge[0] + t.n_edge[1] + t.n_edge[2] + t.n_edge[3]) + 2u * (iu + iv) + 2u * iu * iv;
}

// item 3: the stitch strip of edge e as a merge walk.  Outer points O_i (i = 0..n) have coordinate t(f_edge, n, i) along the edge,
// inner points I_j (j = 0..m, m = N - 2) coordinate t(f_in, N, j + 1); each step advances the outer row when the inner row is exhausted
// or the next outer coordinate is <= the next inner one (ties go to the outer row).  Step k's state (i, j = k - i) is found here by
// bisection on the merge path: i is the largest value in [max(0, k - m), min(k, n)] with i == 0 or O(i) <= I(k - i + 1) (I(m + 1) = inf).
OXC_DI void terrain_strip_step(float fo, int n, float fi, int N, int k, int& i, int& j, bool& outer) {
  const int m = N - 2;
  int lo = k - m > 0 ? k - m : 0, hi = k < n ? k : n;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    const int jj = k - mid + 1;
    if (jj > m || terrain_edge_point(fo, n, mid) <= terrain_edge_point(fi, N, jj + 1)) lo = mid;
    else hi = mid - 1;
  }
  i = lo;
  j = k - i;
  outer = j == m || (i < n && terrain_edge_point(fo, n, i + 1) <= terrain_edge_point(fi, N, j + 2));
}

// item 3: domain points (u, v) of triangle k < tri_count, in the order the raster receives them (item 6)
OXC_DI void terrain_triangle_domain(const TerrainPatch& t, uint32_t k, float2 d[3]) {
  if (t.tri_count == 2) {  // the two-triangle quad: (p0, p2, p1), (p0, p3, p2)
    d[0] = make_float2(0.0f, 0.0f);
    d[1] = k == 0 ? make_float2(1.0f, 1.0f) : make_float2(0.0f, 1.0f);
    d[2] = k == 0 ? make_float2(1.0f, 0.0f) : make_float2(1.0f, 1.0f);
    return;
  }
  const int Nu = t.n_in[0], Nv = t.n_in[1];
  const float fu = t.f_in[0], fv = t.f_in[1];
  // strips: bottom (edge v0, v = 0), top (v1, v = 1), left (u0, u = 0), right (u1, u = 1)
  const int edge_of[4] = {1, 3, 0, 2};
  for (int r = 0; r < 4; r++) {
    const int e = edge_of[r];
    const bool along_u = r < 2;
    const int N = along_u ? Nu : Nv;
    const uint32_t count = (uint32_t)(t.n_edge[e] + N - 2);
    if (k >= count) { k -= count; continue; }
    const float fi = along_u ? fu : fv;
    int i, j;
    bool outer;
    terrain_strip_step(t.f_edge[e], t.n_edge[e], fi, N, (int)k, i, j, outer);
    const float o0 = terrain_edge_point(t.f_edge[e], t.n_edge[e], i), i0 = terrain_edge_point(fi, N, j + 1);
    const float o1 = outer ? terrain_edge_point(t.f_edge[e], t.n_edge[e], i + 1) : o0;
    const float i1 = outer ? i0 : terrain_edge_point(fi, N, j + 2);
    // the fixed coordinate of the outer row and of the inner row
    const float oc = (r == 0 || r == 2) ? 0.0f : 1.0f;
    const float ic = along_u ? terrain_edge_point(fv, Nv, r == 0 ? 1 : Nv - 1) : terrain_edge_point(fu, Nu, r == 2 ? 1 : Nu - 1);
    float2 A, B, C; // counter-clockwise in (u, v): bottom and right (O_i, O_i+1, I_j) / (O_i, I_j+1, I_j), top and left mirrored
    const bool ccw_as_bottom = r == 0 || r == 3;
    float2 O0 = along_u ? make_float2(o0, oc) : make_float2(oc, o0), O1 = along_u ? make_float2(o1, oc) : make_float2(oc, o1);
    float2 I0 = along_u ? make_float2(i0, ic) : make_float2(ic, i0), I1 = along_u ? make_float2(i1, ic) : make_float2(ic, i1);
    if (outer) { A = O0; B = ccw_as_bottom ? O1 : I0; C = ccw_as_bottom ? I0 : O1; }
    else { A = O0; B = ccw_as_bottom ? I1 : I0; C = ccw_as_bottom ? I0 : I1; }
    d[0] = A; d[1] = C; d[2] = B; // item 6: the raster draws the clockwise order
    return;
  }
  // interior cells, row-major, each (P, Q, R), (P, R, S) counter-clockwise
  const uint32_t cu = (uint32_t)Nu - 2u, cell = k >> 1, ci = cell % cu, cj = cell / cu;
  const float a0 = terrain_edge_point(fu, Nu, (int)ci + 1), a1 = terrain_edge_point(fu, Nu, (int)ci + 2);
  const float b0 = terrain_edge_point(fv, Nv, (int)cj + 1), b1 = terrain_edge_point(fv, Nv, (int)cj + 2);
  const float2 P = make_float2(a0, b0), Q = make_float2(a1, b0), R = make_float2(a1, b1), S = make_float2(a0, b1);
  d[0] = P;
  d[1] = (k & 1) ? S : R;
  d[2] = (k & 1) ? R : Q;
}

// items 4-5: the clip position of domain point (u, v): ds_main's two lerps across the patch, the height at the lerped (x, z), then
// projection_view x (x, h, z, 1) with the meshlet raster's row order
OXC_DI float4 terrain_clip(const TerrainDrawParams& p, const TerrainPatch& t, float2 d) {
  const float x0 = terrain_lerp(t.px[0], t.px[1], d.x), z0 = terrain_lerp(t.pz[0], t.pz[1], d.x);
  const float x1 = terrain_lerp(t.px[3], t.px[2], d.x), z1 = terrain_lerp(t.pz[3], t.pz[2], d.x);
  const float x = terrain_lerp(x0, x1, d.y), z = terrain_lerp(z0, z1, d.y);
  const float h = terrain_height(p, x, z);
  return make_float4(row_dot_p1(p.pv_row[0], x, h, z), row_dot_p1(p.pv_row[1], x, h, z), row_dot_p1(p.pv_row[2], x, h, z),
                     row_dot_p1(p.pv_row[3], x, h, z));
}

// item 7: the patch slot `slot` of visible_patches draws, or patch_total (nothing) when the slot is past the clamped instance count or
// holds an index outside the grid
OXC_DI uint32_t terrain_slot_patch(const TerrainDrawParams& p, uint32_t slot, uint32_t count) {
  if (slot >= count) return p.patch_total;
  const uint32_t idx = p.visible_patches[slot];
  return idx < p.patch_total ? idx : p.patch_total;
}

} // namespace oxc
