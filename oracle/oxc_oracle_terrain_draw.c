/*
 * oxc_oracle_terrain_draw.c — CPU ORACLE (test infrastructure) of the terrain's vis-buffer draw: RendererInstance::
 * draw_terrain_for_visbuffer (Passes/Terrain.cpp:218-277) running passes/terrain_visbuffer.slang (vs_main, hs_constants, ds_main,
 * fs_main).  Same rules as oxc_oracle.c: plain C11, IEEE binary32 with round to nearest, no contraction, IEEE divide / sqrt.  It is
 * one translation unit with oxc_oracle_vsm_resolve.c (and so oxc_oracle.c), included below, so that it runs the raster
 * specification's own orc_raster_triangle and the library's canonical sin / cos rather than copies.  Built into
 * liboxc_oracle_terrain_draw.so by oracle/pyoracle_terrain_draw.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_terrain_draw.c
 *
 * SPECIFICATION: include/oxcull.h, the comment above oxc_draw_terrain (items 1-7).  The triangulation of item 3 is written here as
 * the sequential walk the item describes; the device finds each step of the same walk by bisection (oxc_terrain.cuh).
 */
#include "oxc_oracle_vsm_resolve.c"

#include "oxc_oracle_terrain_draw.h"

/* HLSL max / min: a NaN operand yields the other one */
static float td_max(float a, float b) { return (b != b || a > b) ? a : b; }
static float td_min(float a, float b) { return (b != b || a < b) ? a : b; }

float orc_terrain_projection_scale(float fov_degrees, float resolution_y) {
  const float half = (fov_degrees * 0x1.1df46ap-6f) * 0.5f; /* radians(fov) * 0.5, pi / 180 = 0x3C8EFA35 */
  float s, c;
  orc_sincos_canonical(half, &s, &c);
  return (resolution_y * 0.5f) / (s / c);
}

float orc_terrain_factor_clamp(float f) { return !(f >= 1.0f) ? 1.0f : (f > 63.0f ? 63.0f : f); }

int32_t orc_terrain_round_odd(float f) {
  const float c = orc_terrain_factor_clamp(f);
  return 2 * (int32_t)ceilf((c - 1.0f) * 0.5f) + 1;
}

void orc_terrain_edge_points(float f, int32_t n, float* out) {
  out[0] = 0.0f;
  out[n] = 1.0f;
  const float L = 1.0f / f, s = (f - (float)(n - 2)) / (2.0f * f);
  for (int32_t k = 1; 2 * k < n; k++) out[k] = s + (float)(k - 1) * L;
  for (int32_t k = n - 1; 2 * k > n; k--) out[k] = 1.0f - out[n - k];
}

/* item 4: the bilinear R16Unorm tap, ClampToEdge, level 0 */
static float td_texel(const uint16_t* hm, uint32_t rx, uint32_t ry, int64_t x, int64_t y) {
  x = x < 0 ? 0 : (x > (int64_t)rx - 1 ? (int64_t)rx - 1 : x);
  y = y < 0 ? 0 : (y > (int64_t)ry - 1 ? (int64_t)ry - 1 : y);
  return (float)hm[(size_t)y * rx + (size_t)x] / 65535.0f;
}
static int64_t td_floor_index(float f) { /* float -> int32 truncating, saturating, NaN -> 0 */
  return !(f == f) ? 0 : (f >= 2147483648.0f ? 2147483647 : (f <= -2147483648.0f ? (-2147483647 - 1) : (int64_t)(int32_t)f));
}
static float td_height(const uint16_t* hm, uint32_t rx, uint32_t ry, const OxcTerrainDrawSettings* s, float wx, float wz) {
  const float u = (wx - s->terrain.world_min[0]) * s->inv_world_size[0], v = (wz - s->terrain.world_min[1]) * s->inv_world_size[1];
  const float x = u * (float)rx - 0.5f, y = v * (float)ry - 0.5f;
  const float x0 = floorf(x), y0 = floorf(y);
  const float fx = x - x0, fy = y - y0;
  const int64_t ix = td_floor_index(x0), iy = td_floor_index(y0);
  const float a00 = td_texel(hm, rx, ry, ix, iy), a10 = td_texel(hm, rx, ry, ix + 1, iy);
  const float a01 = td_texel(hm, rx, ry, ix, iy + 1), a11 = td_texel(hm, rx, ry, ix + 1, iy + 1);
  const float top = a00 + fx * (a10 - a00), bot = a01 + fx * (a11 - a01);
  return s->terrain.base_height + (top + fy * (bot - top)) * s->terrain.height_scale;
}

static float td_length(float x, float y, float z) { return sqrtf((x * x + y * y) + z * z); }

/* item 1: edge_tessellation */
static float td_edge(const OxcTerrainDrawSettings* s, const OxcCullCamera* cam, float scale, const float* a, const float* b) {
  const float c[3] = {(a[0] + b[0]) * 0.5f, (a[1] + b[1]) * 0.5f, (a[2] + b[2]) * 0.5f};
  const float radius = td_length(a[0] - b[0], a[1] - b[1], a[2] - b[2]) * 0.5f;
  const float vd = td_max(td_length(c[0] - cam->position[0], c[1] - cam->position[1], c[2] - cam->position[2]) - radius, cam->near_clip);
  const float projected = ((2.0f * radius) * scale) / vd;
  return td_min(td_max(projected / s->target_edge_pixels, 1.0f), s->max_tessellation);
}

void orc_terrain_patch(const uint16_t* hm, uint32_t rx, uint32_t ry, const OxcTerrainDrawSettings* s, const OxcCullCamera* cam,
                       uint32_t patch_index, OrcTerrainPatch* o) {
  const OxcTerrainData* t = &s->terrain;
  const uint32_t px = patch_index % t->patch_count[0], pz = patch_index / t->patch_count[0];
  static const uint32_t dx[4] = {0, 1, 1, 0}, dz[4] = {0, 0, 1, 1};
  for (int k = 0; k < 4; k++) { /* vs_main: patch_corner, sample_height */
    const float x = t->world_min[0] + ((float)(px + dx[k]) / (float)t->patch_count[0]) * t->world_size[0];
    const float z = t->world_min[1] + ((float)(pz + dz[k]) / (float)t->patch_count[1]) * t->world_size[1];
    o->corner[k][0] = x;
    o->corner[k][1] = td_height(hm, rx, ry, s, x, z);
    o->corner[k][2] = z;
  }
  const float scale = orc_terrain_projection_scale(s->fov, cam->resolution[1]);
  o->factor[0] = td_edge(s, cam, scale, o->corner[0], o->corner[3]); /* hs_constants: u0 */
  o->factor[1] = td_edge(s, cam, scale, o->corner[0], o->corner[1]); /* v0 */
  o->factor[2] = td_edge(s, cam, scale, o->corner[1], o->corner[2]); /* u1 */
  o->factor[3] = td_edge(s, cam, scale, o->corner[3], o->corner[2]); /* v1 */
  o->factor[4] = td_max(o->factor[1], o->factor[3]);
  o->factor[5] = td_max(o->factor[0], o->factor[2]);
  int all_one = 1;
  for (int k = 0; k < 6; k++) {
    o->pinned[k] = orc_terrain_factor_clamp(o->factor[k]);
    o->n[k] = orc_terrain_round_odd(o->factor[k]);
    all_one = all_one && o->n[k] == 1;
  }
  if (all_one) { o->triangles = 2; return; }
  for (int k = 4; k < 6; k++)
    if (o->n[k] == 1) { o->pinned[k] = 0x1.000002p0f; o->n[k] = 3; }
  const uint32_t iu = (uint32_t)o->n[4] - 2, iv = (uint32_t)o->n[5] - 2;
  o->triangles = (uint32_t)(o->n[0] + o->n[1] + o->n[2] + o->n[3]) + 2 * (iu + iv) + 2 * iu * iv;
}

/* appends (a, c, b): item 6 hands each counter-clockwise (a, b, c) to the raster clockwise */
static void td_emit(float* tris, uint32_t cap, uint32_t* n, const float a[2], const float b[2], const float c[2]) {
  if (*n < cap) {
    float* o = tris + (size_t)*n * 6;
    o[0] = a[0]; o[1] = a[1]; o[2] = c[0]; o[3] = c[1]; o[4] = b[0]; o[5] = b[1];
  }
  (*n)++;
}

uint32_t orc_terrain_patch_domain(const OrcTerrainPatch* p, float* tris, uint32_t cap) {
  uint32_t n = 0;
  if (p->triangles == 2) {
    const float q[4][2] = {{0, 0}, {1, 0}, {1, 1}, {0, 1}};
    td_emit(tris, cap, &n, q[0], q[1], q[2]);
    td_emit(tris, cap, &n, q[0], q[2], q[3]);
    return n;
  }
  const int32_t Nu = p->n[4], Nv = p->n[5];
  float a[64], b[64];
  orc_terrain_edge_points(p->pinned[4], Nu, a);
  orc_terrain_edge_points(p->pinned[5], Nv, b);
  /* strips: bottom (edge v0 = 1, v = 0), top (v1 = 3, v = 1), left (u0 = 0, u = 0), right (u1 = 2, u = 1) */
  static const int edge_of[4] = {1, 3, 0, 2};
  for (int r = 0; r < 4; r++) {
    const int e = edge_of[r], along_u = r < 2, bottom_like = r == 0 || r == 3;
    float o[64], in[64];
    const int32_t no = p->n[e];
    orc_terrain_edge_points(p->pinned[e], no, o);
    const int32_t N = along_u ? Nu : Nv, m = N - 2;
    for (int32_t j = 0; j <= m; j++) in[j] = along_u ? a[j + 1] : b[j + 1];
    const float oc = (r == 0 || r == 2) ? 0.0f : 1.0f;
    const float ic = along_u ? (r == 0 ? b[1] : b[Nv - 1]) : (r == 2 ? a[1] : a[Nu - 1]);
    int32_t i = 0, j = 0;
    while (i < no || j < m) {
      float O0[2], O1[2], I0[2], I1[2];
      const int outer = j == m || (i < no && o[i + 1] <= in[j + 1]); /* ties go to the outer row */
#define TD_PT(P, c, fixed) do { if (along_u) { P[0] = (c); P[1] = (fixed); } else { P[0] = (fixed); P[1] = (c); } } while (0)
      TD_PT(O0, o[i], oc);
      TD_PT(I0, in[j], ic);
      if (outer) {
        TD_PT(O1, o[i + 1], oc);
        if (bottom_like) td_emit(tris, cap, &n, O0, O1, I0); else td_emit(tris, cap, &n, O0, I0, O1);
        i++;
      } else {
        TD_PT(I1, in[j + 1], ic);
        if (bottom_like) td_emit(tris, cap, &n, O0, I1, I0); else td_emit(tris, cap, &n, O0, I0, I1);
        j++;
      }
#undef TD_PT
    }
  }
  for (int32_t j = 1; j + 1 < Nv; j++) /* the inner grid's cells, row-major */
    for (int32_t i = 1; i + 1 < Nu; i++) {
      const float P[2] = {a[i], b[j]}, Q[2] = {a[i + 1], b[j]}, R[2] = {a[i + 1], b[j + 1]}, S[2] = {a[i], b[j + 1]};
      td_emit(tris, cap, &n, P, Q, R);
      td_emit(tris, cap, &n, P, R, S);
    }
  return n;
}

static float td_lerp(float a, float b, float t) { return a * (1.0f - t) + b * t; }

uint64_t orc_draw_terrain(const uint16_t* hm, uint32_t rx, uint32_t ry, const OxcTerrainDrawSettings* s, const uint32_t* visible,
                          uint32_t instance_count, const OxcCullCamera* cam, uint32_t prim_bits, uint32_t W, uint32_t H, uint64_t* vis) {
  const uint32_t total = s->terrain.patch_count[0] * s->terrain.patch_count[1];
  const uint32_t count = instance_count < total ? instance_count : total; /* item 7 */
  const uint32_t data = ((0xFFFFFFFFu >> prim_bits) - 1u) << prim_bits;   /* item 5 */
  const float* m = cam->projection_view;
  float* tris = (float*)malloc(sizeof(float) * 6 * 8192);
  if (!tris) abort(); /* test infrastructure: no partial image */
  uint64_t emitted = 0;
  for (uint32_t slot = 0; slot < count; slot++) {
    const uint32_t idx = visible[slot];
    if (idx >= total) continue;
    OrcTerrainPatch p;
    orc_terrain_patch(hm, rx, ry, s, cam, idx, &p);
    const uint32_t nt = orc_terrain_patch_domain(&p, tris, 8192);
    for (uint32_t k = 0; k < nt; k++) {
      float clip[3][4];
      for (int v = 0; v < 3; v++) { /* ds_main */
        const float u = tris[k * 6 + v * 2], w = tris[k * 6 + v * 2 + 1];
        const float e0x = td_lerp(p.corner[0][0], p.corner[1][0], u), e0z = td_lerp(p.corner[0][2], p.corner[1][2], u);
        const float e1x = td_lerp(p.corner[3][0], p.corner[2][0], u), e1z = td_lerp(p.corner[3][2], p.corner[2][2], u);
        const float x = td_lerp(e0x, e1x, w), z = td_lerp(e0z, e1z, w);
        const float h = td_height(hm, rx, ry, s, x, z);
        for (int r = 0; r < 4; r++) clip[v][r] = ((m[r] * x + m[4 + r] * h) + m[8 + r] * z) + m[12 + r];
      }
      orc_raster_triangle(clip, data, W, H, vis);
    }
    emitted += nt;
  }
  free(tris);
  return emitted;
}
