// kernels_vsm_draw.cuh — the VSM shadow raster into the physical atlas (Passes/Shadowmaps.cpp:433-754, the last step of
// draw_virtual_shadowmap: rmvsm_build_draw_commands.slang + rmvsm_draw_physical_pages.slang), drawn in software:
//   k_vsm_draw_prepare   one CTA: the per-frame bitmap of virtual pages whose entry is Backed && Dirty (clipmaps with a zero dirty
//                        flag get none), and the first pixel of every virtual page row / column
//   k_vsm_draw_meshlets  one warp per survivor of the HPB cull: the coarse-camera triangle test once per triangle, then per dirty
//                        clipmap the vertices into shared memory, a meshlet-level reject on the page rectangle, and one work item per
//                        (kept triangle, dirty page it may touch)
//   k_vsm_draw_items     one warp per work item: the triangle (two-sided set-up, clip path, alpha test) rasterised over the pixels
//                        of that one page only, min sink into the atlas
// Work is proportional to the samples inside dirty pages: a ground triangle over hundreds of clean pages costs a few bitmap
// tests, and a (meshlet, clipmap) pair whose page rectangle holds no dirty page costs no triangle work.  A work item the queue
// has no room for is rasterised by the lane that found it, so nothing is ever dropped.
// Specification: oracle/oxc_oracle_vsm_draw.c orc_vsm_draw_pages (bit-exact).
#pragma once
#include "kernels_alpha.cuh"
#include "kernels_vsm.cuh"

namespace oxc {

struct VsmDrawParams {
  const OxcMeshletInstance* meshlet_instances;
  const InstCull* inst;                 // built for the coarse camera (its mvp rows: the triangle test)
  const InstGeom* geom;
  const OxcMeshInstance* mesh_instances;
  const OxcTransformWorld* transforms;
  const uint32_t* visible_indices;      // the HPB cull's survivors, count in tri_cmd->x
  const OxcDispatchIndirectCommand* tri_cmd;
  const uint32_t* id_base;
  const AlphaMaterial* materials;       // null: no material is alpha tested
  uint32_t material_count;
  float4 pv_row[VSM_MAX_CLIPMAPS][4];   // clipmap projection_view_mat, row i
  int page_offset[VSM_MAX_CLIPMAPS][2];
  const uint32_t* dirty_flags;          // device
  const uint32_t* page_tables;          // [clipmap][size][size]
  uint32_t* atlas;                      // R32UI view of the physical atlas, P x P
  uint32_t* bitmap;                     // [clipmap][size][words_per_row]: virtual page is Backed && Dirty, its clipmap flagged
  int* first_px;                        // [size + 1]: first pixel whose virtual page is >= v (P if none)
  uint4* queue;                         // work items {survivor, triangle | clipmap << 8, vx, vy}
  uint32_t* counters;                   // [0] items found, [1] (meshlet, clipmap) pairs that reached triangle work
  uint32_t queue_capacity;
  int size, page_size, P, phys_per_row, clipmap_count, words_per_row;
  float fP, fsize, fpage;
};

// rmvsm_draw_physical_pages.slang:60-61 for one pixel coordinate: i32(floor((px + 0.5) / physical_extent * page_table_size))
OXC_DI int vsm_page_of(int px, float fP, float fsize) { return __float2int_rz(floorf(fm(fd(fa((float)px, 0.5f), fP), fsize))); }

// :67-70 for one pixel coordinate: the in-page texel, i32(mod(f32(i32(floor(virtual_uv * physical_size))), page_size))
OXC_DI int vsm_in_page(int px, float fP, float fpage) {
  const float t = (float)__float2int_rz(floorf(fm(fd(fa((float)px, 0.5f), fP), fP)));
  return __float2int_rz(fs(t, fm(fpage, floorf(fd(t, fpage)))));
}

__global__ void __launch_bounds__(1024, 1) k_vsm_draw_prepare(const __grid_constant__ VsmDrawParams p) {
  const uint32_t t = threadIdx.x;
  const int size = p.size, wpr = p.words_per_row;
  const uint32_t words = (uint32_t)p.clipmap_count * size * wpr;
  for (uint32_t i = t; i < words; i += blockDim.x) {
    const int c = (int)(i / ((uint32_t)size * wpr)), r = (int)(i % ((uint32_t)size * wpr)), vy = r / wpr, k = r % wpr;
    uint32_t bits = 0;
    int wy;
    if (__ldg(&p.dirty_flags[c]) != 0u && vsm_wrap(vy, p.page_offset[c][1], size, wy)) {
      const uint32_t* row = p.page_tables + ((size_t)c * size + wy) * size;
      for (int b = 0; b < 32; b++) {
        const int vx = k * 32 + b;
        int wx;
        if (vx >= size) break;
        if (!vsm_wrap(vx, p.page_offset[c][0], size, wx)) continue;
        const uint32_t e = __ldg(&row[wx]);
        if ((e & VSM_BACKED) && (e & VSM_DIRTY)) bits |= 1u << b;
      }
    }
    p.bitmap[i] = bits;
  }
  for (int v = (int)t; v <= size; v += (int)blockDim.x) { // vsm_page_of is monotone in px: binary search for the first pixel
    int lo = 0, hi = p.P;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (vsm_page_of(mid, p.fP, p.fsize) >= v) hi = mid; else lo = mid + 1;
    }
    p.first_px[v] = lo;
  }
  if (t < 2) p.counters[t] = 0u;
}

// screen x / y of a clip-space vertex exactly as to_screen computes them before snapping; false = no bound (w <= 0, NaN, inf)
OXC_DI bool vsm_screen_xy(const float4 c, float fP, float& sx, float& sy) {
  if (!(c.w > 0.0f)) return false;
  const float rw = fd(1.0f, c.w);
  sx = fm(fa(fm(fm(c.x, rw), 0.5f), 0.5f), fP);
  sy = fm(fa(fm(fm(c.y, rw), 0.5f), 0.5f), fP);
  return fabsf(sx) < 3.0e38f && fabsf(sy) < 3.0e38f;
}

// conservative page rectangle of screen extent [x0, x1] x [y0, y1]: samples of a triangle lie within one pixel of the extent of
// its vertices (snapping moves a vertex by 1/512 pixel, clipping cuts stay inside it up to rounding); false = empty
OXC_DI bool vsm_page_rect(const VsmDrawParams& p, float x0, float x1, float y0, float y1, bool bounded, int& vx0, int& vx1, int& vy0, int& vy1) {
  int px0 = 0, px1 = p.P - 1, py0 = 0, py1 = p.P - 1;
  if (bounded) {
    px0 = (int)fmaxf(floorf(x0) - 1.0f, 0.0f); px1 = (int)fminf(ceilf(x1) + 1.0f, (float)(p.P - 1));
    py0 = (int)fmaxf(floorf(y0) - 1.0f, 0.0f); py1 = (int)fminf(ceilf(y1) + 1.0f, (float)(p.P - 1));
    if (!(x1 >= -2.0f && y1 >= -2.0f && x0 <= (float)p.P + 1.0f && y0 <= (float)p.P + 1.0f) || px0 > px1 || py0 > py1) return false;
  }
  vx0 = max(vsm_page_of(px0, p.fP, p.fsize), 0); vx1 = min(vsm_page_of(px1, p.fP, p.fsize), p.size - 1);
  vy0 = max(vsm_page_of(py0, p.fP, p.fsize), 0); vy1 = min(vsm_page_of(py1, p.fP, p.fsize), p.size - 1);
  return vx0 <= vx1 && vy0 <= vy1;
}

OXC_DI bool vsm_page_dirty(const VsmDrawParams& p, int c, int vx, int vy) {
  return (p.bitmap[((size_t)c * p.size + vy) * p.words_per_row + (vx >> 5)] >> (vx & 31)) & 1u;
}

// one vertex of survivor meshlet: object position, world position (Transform::to_world_position) and clip position in clipmap c
OXC_DI float4 vsm_world(const float4 w0, const float4 w1, const float4 w2, uint2 q) {
  const float x = dequantize_half(q.x & 0xFFFFu), y = dequantize_half(q.x >> 16), z = dequantize_half(q.y & 0xFFFFu);
  return make_float4(row_dot_p1(w0, x, y, z), row_dot_p1(w1, x, y, z), row_dot_p1(w2, x, y, z), 1.0f);
}
OXC_DI float4 vsm_clip(const VsmDrawParams& p, int c, const float4 w) {
  return make_float4(row_dot_p1(p.pv_row[c][0], w.x, w.y, w.z), row_dot_p1(p.pv_row[c][1], w.x, w.y, w.z),
                     row_dot_p1(p.pv_row[c][2], w.x, w.y, w.z), row_dot_p1(p.pv_row[c][3], w.x, w.y, w.z));
}
OXC_DI void world_rows(const OxcTransformWorld* t, float4& w0, float4& w1, float4& w2) {
  const float* m = t->world; // column-major: row i = (m[i], m[4 + i], m[8 + i], m[12 + i])
  w0 = make_float4(__ldg(&m[0]), __ldg(&m[4]), __ldg(&m[8]), __ldg(&m[12]));
  w1 = make_float4(__ldg(&m[1]), __ldg(&m[5]), __ldg(&m[9]), __ldg(&m[13]));
  w2 = make_float4(__ldg(&m[2]), __ldg(&m[6]), __ldg(&m[10]), __ldg(&m[14]));
}

// the material the survivor's fragments are alpha tested with (texels null: opaque), as k_raster_alpha<true> resolves it
OXC_DI AlphaMaterial vsm_material(const VsmDrawParams& p, uint32_t mesh_instance) {
  AlphaMaterial m;
  m.texels = nullptr;
  if (p.materials) {
    const uint32_t mat = __ldg(&p.mesh_instances[mesh_instance].material_index);
    if (mat < p.material_count) m = p.materials[mat];
  }
  return m;
}

// one page of one drawable triangle: the pixels of virtual page (vx, vy) inside the set-up's box.  Every such pixel maps to the
// same page table entry (its page is (vx, vy) by construction of first_px), so the entry is read once; each sample still maps to
// its texel with the shader's own float arithmetic.  lanes / lane: the warp shares the box in 8 x 4 tiles, or one lane walks it.
struct VsmPage {
  int x0, x1, y0, y1;     // pixel box of the page
  int base_x, base_y;     // physical page origin in texels
  bool backed_dirty;
};

OXC_DI VsmPage vsm_page(const VsmDrawParams& p, int c, int vx, int vy) {
  VsmPage g;
  g.x0 = p.first_px[vx]; g.x1 = p.first_px[vx + 1] - 1; g.y0 = p.first_px[vy]; g.y1 = p.first_px[vy + 1] - 1;
  int wx, wy;
  g.backed_dirty = false; g.base_x = g.base_y = 0;
  if (vsm_wrap(vx, p.page_offset[c][0], p.size, wx) && vsm_wrap(vy, p.page_offset[c][1], p.size, wy)) {
    const uint32_t e = __ldg(&p.page_tables[((size_t)c * p.size + wy) * p.size + wx]);
    g.backed_dirty = (e & VSM_BACKED) && (e & VSM_DIRTY);
    const uint32_t phys = e >> 16; // rmvsm.slang:99-106
    g.base_x = (int)(phys % (uint32_t)p.phys_per_row) * p.page_size;
    g.base_y = (int)(phys / (uint32_t)p.phys_per_row) * p.page_size;
  }
  return g;
}

// the VSM atlas sink (kept out of oxc_raster_core.cuh, whose host build models only the vis buffer's max) (rmvsm_draw_physical_pages.slang:86, atomic_min on the R32UI view): texel = min(texel, asuint(z)) as u32,
// -0.0 stored as +0.0, so u32 order == depth order for the z in [0, 1] that reach it
OXC_DI void sink_min_depth(uint32_t* texel, float z) {
  const uint32_t zb = __float_as_uint(z);
  atomicMin(texel, zb == 0x80000000u ? 0u : zb);
}

OXC_DI void vsm_raster_page(const VsmDrawParams& p, const TriSetup& s, const AlphaMaterial& m, const AlphaTri& at, const VsmPage& g,
                            int lanes, int lane) {
  const int x0 = max(s.px0, g.x0), x1 = min(s.px1, g.x1), y0 = max(s.py0, g.y0), y1 = min(s.py1, g.y1);
  if (x0 > x1 || y0 > y1 || !g.backed_dirty) return;
  const int tw = lanes == 32 ? 8 : 1, th = lanes == 32 ? 4 : 1;
  const int lx = lanes == 32 ? (lane & 7) : 0, ly = lanes == 32 ? (lane >> 3) : 0;
  for (int ty = y0; ty <= y1; ty += th)
    for (int tx = x0; tx <= x1; tx += tw) {
      const int px = tx + lx, py = ty + ly;
      if (px > x1 || py > y1) continue;
      const int sx = px * 256 + 128, sy = py * 256 + 128;
      const long long e0 = orient2d(s.bx, s.by, s.cx, s.cy, sx, sy), e1 = orient2d(s.cx, s.cy, s.ax, s.ay, sx, sy),
                      e2 = orient2d(s.ax, s.ay, s.bx, s.by, sx, sy);
      float z;
      if (!sample_depth(s, e0, e1, e2, z)) continue;
      if (m.texels) { // rmvsm_draw_physical_pages.slang:73-84, the test of visbuffer_encode.slang:54-66
        const long long ex[3] = {-(long long)(s.cy - s.by) * 256, -(long long)(s.ay - s.cy) * 256, -(long long)(s.by - s.ay) * 256};
        const long long ey[3] = {(long long)(s.cx - s.bx) * 256, (long long)(s.ax - s.cx) * 256, (long long)(s.bx - s.ax) * 256};
        if (!alpha_keep(m, at, px, py, e0, e1, e2, ex, ey)) continue;
      }
      const int X = g.base_x + vsm_in_page(px, p.fP, p.fpage), Y = g.base_y + vsm_in_page(py, p.fP, p.fpage);
      if (X >= p.P || Y >= p.P) continue; // an out-of-bounds image atomic is discarded
      sink_min_depth(p.atlas + (size_t)Y * p.P + X, z);
    }
}

// one (triangle, clipmap, page) work item: plain set-up, or the clip path's fan, each piece over the page's pixels
OXC_DNI void vsm_draw_item(const VsmDrawParams& p, uint4 item, int lanes, int lane) {
  const uint32_t gid = __ldg(&p.visible_indices[item.x]);
  const uint32_t tri = item.y & 0xFFu;
  const int c = (int)(item.y >> 8);
  const uint2 mi = __ldg(reinterpret_cast<const uint2*>(p.meshlet_instances) + (gid - (p.id_base ? __ldg(p.id_base) : 0u)));
  const InstGeom* gm = p.geom + mi.x;
  const uint4 ml = __ldg(reinterpret_cast<const uint4*>(gm->meshlets + mi.y));
  const uint32_t base = ml.y + tri * 3u;
  uint32_t vi[3];
  for (int k = 0; k < 3; k++) vi[k] = __ldg(&gm->indirect_vertex_indices[ml.x + micro_index(gm->local_triangle_indices, base + (uint32_t)k)]);
  float4 w0, w1, w2;
  world_rows(p.transforms + gm->transform_index, w0, w1, w2);
  float4 cv[3];
  float2 uv[3];
  const AlphaMaterial m = vsm_material(p, mi.x);
  for (int k = 0; k < 3; k++) {
    cv[k] = vsm_clip(p, c, vsm_world(w0, w1, w2, __ldg(&gm->vertex_positions[vi[k]])));
    uv[k] = make_float2(0.f, 0.f);
    if (m.texels && gm->texture_coords) {
      const uint32_t t = __ldg(&gm->texture_coords[vi[k]]);
      uv[k] = make_float2(dequantize_half(t & 0xFFFFu), dequantize_half(t >> 16));
    }
  }
  const VsmPage g = vsm_page(p, c, (int)item.z, (int)item.w);
  const uint32_t W = (uint32_t)p.P;
  TriSetup s;
  bool kept;
  AlphaTri at;
  const int why = tri_setup_two_sided(to_screen(cv[0], p.fP, p.fP), to_screen(cv[1], p.fP, p.fP), to_screen(cv[2], p.fP, p.fP), W, W, s, kept);
  if (why == TRI_DRAW) {
    if (kept) alpha_tri_setup(cv[0], cv[2], cv[1], uv[0].x, uv[0].y, uv[2].x, uv[2].y, uv[1].x, uv[1].y, at);
    else alpha_tri_setup(cv[0], cv[1], cv[2], uv[0].x, uv[0].y, uv[1].x, uv[1].y, uv[2].x, uv[2].y, at);
    vsm_raster_page(p, s, m, at, g, lanes, lane);
  } else if (why == TRI_INVALID_VERTEX) { // a vertex at w <= 0 or beyond the snap range: the vis raster's clipper, uv carried
    ClipVertUV poly[2][12];
    int cur;
    const ClipVertUV a0 = {cv[0], uv[0].x, uv[0].y}, a1 = {cv[1], uv[1].x, uv[1].y}, a2 = {cv[2], uv[2].x, uv[2].y};
    const int n = clip_polygon_uv(a0, a1, a2, poly, cur);
    for (int i = 1; i + 1 < n; i++) {
      const ClipVertUV q0 = poly[cur][0], q1 = poly[cur][i], q2 = poly[cur][i + 1];
      TriSetup ps;
      if (tri_setup_two_sided(to_screen(q0.c, p.fP, p.fP), to_screen(q1.c, p.fP, p.fP), to_screen(q2.c, p.fP, p.fP), W, W, ps, kept) != TRI_DRAW)
        continue;
      if (kept) alpha_tri_setup(q0.c, q2.c, q1.c, q0.u, q0.v, q2.u, q2.v, q1.u, q1.v, at);
      else alpha_tri_setup(q0.c, q1.c, q2.c, q0.u, q0.v, q1.u, q1.v, q2.u, q2.v, at);
      vsm_raster_page(p, ps, m, at, g, lanes, lane);
    }
  }
}

constexpr int VSM_DRAW_THREADS = 128, VSM_DRAW_WARPS = VSM_DRAW_THREADS / 32;
constexpr uint32_t VSM_DRAW_QUEUE = 1u << 20; // work items (16 B each); beyond it the lane that finds an item draws it
constexpr int VSM_DRAW_MAX_EXTENT = 16384;    // atlas side: pixel centres stay inside the 2^22 sub-pixel snap range

__global__ void __launch_bounds__(VSM_DRAW_THREADS) k_vsm_draw_meshlets(const __grid_constant__ VsmDrawParams p) {
  __shared__ float4 world_all[VSM_DRAW_WARPS][OXC_MESHLET_MAX_VERTICES];
  __shared__ float4 clip_all[VSM_DRAW_WARPS][OXC_MESHLET_MAX_VERTICES];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float4* world_s = world_all[warp];
  float4* clip_s = clip_all[warp];
  const uint32_t count = p.tri_cmd->x;
  const uint32_t id_base = p.id_base ? __ldg(p.id_base) : 0u;
  for (uint32_t g = blockIdx.x * VSM_DRAW_WARPS + warp; g < count; g += gridDim.x * VSM_DRAW_WARPS) {
    const uint32_t gid = __ldg(&p.visible_indices[g]);
    const uint2 mi = __ldg(reinterpret_cast<const uint2*>(p.meshlet_instances) + (gid - id_base));
    const InstGeom* gm = p.geom + mi.x;
    const InstCull* ic = p.inst + mi.x;
    const uint4 ml = __ldg(reinterpret_cast<const uint4*>(gm->meshlets + mi.y));
    const uint32_t vertex_count = min(ml.z, (uint32_t)OXC_MESHLET_MAX_VERTICES), tri_count = min(ml.w, (uint32_t)OXC_MESHLET_MAX_PRIMITIVES);
    // the coarse camera's clip positions (cull_triangles.slang:62-66 with PV . W) and the world positions, once per vertex
    const float4 r0 = __ldg(&ic->mvp_row[0]), r1 = __ldg(&ic->mvp_row[1]), r2 = __ldg(&ic->mvp_row[2]), r3 = __ldg(&ic->mvp_row[3]);
    float4 w0, w1, w2;
    world_rows(p.transforms + gm->transform_index, w0, w1, w2);
    for (uint32_t v = lane; v < vertex_count; v += 32) {
      const uint2 q = __ldg(&gm->vertex_positions[__ldg(&gm->indirect_vertex_indices[ml.x + v])]);
      const float x = dequantize_half(q.x & 0xFFFFu), y = dequantize_half(q.x >> 16), z = dequantize_half(q.y & 0xFFFFu);
      clip_s[v] = make_float4(row_dot_p1(r0, x, y, z), row_dot_p1(r1, x, y, z), row_dot_p1(r2, x, y, z), row_dot_p1(r3, x, y, z));
      world_s[v] = vsm_world(w0, w1, w2, q);
    }
    __syncwarp();
    // the coarse triangle test (cull_triangles.slang:59-69), once per triangle: bit t of keep
    uint32_t i0[2], i1[2], i2[2];
    bool kept_tri[2];
    for (int k = 0; k < 2; k++) {
      const uint32_t t = lane + 32u * k;
      kept_tri[k] = false;
      i0[k] = i1[k] = i2[k] = 0;
      if (t < tri_count) {
        const uint32_t base = ml.y + t * 3u;
        i0[k] = micro_index(gm->local_triangle_indices, base + 0u); i1[k] = micro_index(gm->local_triangle_indices, base + 1u);
        i2[k] = micro_index(gm->local_triangle_indices, base + 2u);
        if (max(i0[k], max(i1[k], i2[k])) < vertex_count) {
          const float4 c0 = clip_s[i0[k]], c1 = clip_s[i1[k]], c2 = clip_s[i2[k]];
          kept_tri[k] = c0.z >= 0.0f && c1.z >= 0.0f && c2.z >= 0.0f && !triangle_backface(c0, c1, c2);
        }
      }
    }
    if (!__any_sync(0xffffffffu, kept_tri[0] || kept_tri[1])) { __syncwarp(); continue; }
    for (int c = p.clipmap_count - 1; c >= 0; c--) { // rmvsm_build_draw_commands.slang:21-31: dirty clipmaps, highest first
      if (__ldg(&p.dirty_flags[c]) == 0u) continue;
      __syncwarp(); // clip_s of the previous clipmap is read no more
      float mnx = 3.0e38f, mxx = -3.0e38f, mny = 3.0e38f, mxy = -3.0e38f;
      bool bounded = true;
      for (uint32_t v = lane; v < vertex_count; v += 32) {
        const float4 cc = vsm_clip(p, c, world_s[v]);
        clip_s[v] = cc;
        float sx, sy;
        if (vsm_screen_xy(cc, p.fP, sx, sy)) { mnx = fminf(mnx, sx); mxx = fmaxf(mxx, sx); mny = fminf(mny, sy); mxy = fmaxf(mxy, sy); }
        else bounded = false;
      }
      __syncwarp();
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        mnx = fminf(mnx, __shfl_xor_sync(0xffffffffu, mnx, o)); mxx = fmaxf(mxx, __shfl_xor_sync(0xffffffffu, mxx, o));
        mny = fminf(mny, __shfl_xor_sync(0xffffffffu, mny, o)); mxy = fmaxf(mxy, __shfl_xor_sync(0xffffffffu, mxy, o));
      }
      bounded = __all_sync(0xffffffffu, bounded);
      // meshlet-level reject: no dirty page in the meshlet's page rectangle
      int vx0, vx1, vy0, vy1;
      if (!vsm_page_rect(p, mnx, mxx, mny, mxy, bounded, vx0, vx1, vy0, vy1)) continue;
      bool any = false;
      for (int vy = vy0 + (int)lane; vy <= vy1 && !any; vy += 32)
        for (int k = vx0 >> 5; k <= (vx1 >> 5); k++) {
          uint32_t wbits = p.bitmap[((size_t)c * p.size + vy) * p.words_per_row + k];
          if (k == (vx0 >> 5)) wbits &= ~0u << (vx0 & 31);
          if (k == (vx1 >> 5) && (vx1 & 31) != 31) wbits &= (1u << ((vx1 & 31) + 1)) - 1u;
          if (wbits) { any = true; break; }
        }
      if (!__any_sync(0xffffffffu, any)) continue;
      if (lane == 0) atomicAdd(&p.counters[1], 1u);
      // triangle level: one work item per dirty page of each kept triangle's page rectangle
      for (int k = 0; k < 2; k++) {
        if (!kept_tri[k]) continue;
        const float4 cv[3] = {clip_s[i0[k]], clip_s[i1[k]], clip_s[i2[k]]};
        float tx0 = 3.0e38f, tx1 = -3.0e38f, ty0 = 3.0e38f, ty1 = -3.0e38f;
        bool tb = true;
        for (int j = 0; j < 3; j++) {
          float sx, sy;
          if (vsm_screen_xy(cv[j], p.fP, sx, sy)) { tx0 = fminf(tx0, sx); tx1 = fmaxf(tx1, sx); ty0 = fminf(ty0, sy); ty1 = fmaxf(ty1, sy); }
          else tb = false;
        }
        int ax0, ax1, ay0, ay1;
        if (!vsm_page_rect(p, tx0, tx1, ty0, ty1, tb, ax0, ax1, ay0, ay1)) continue;
        for (int vy = ay0; vy <= ay1; vy++)
          for (int vx = ax0; vx <= ax1; vx++) {
            if (!vsm_page_dirty(p, c, vx, vy)) continue;
            const uint4 item = make_uint4(g, (lane + 32u * k) | ((uint32_t)c << 8), (uint32_t)vx, (uint32_t)vy);
            const uint32_t slot = atomicAdd(&p.counters[0], 1u);
            if (slot < p.queue_capacity) p.queue[slot] = item;
            else vsm_draw_item(p, item, 1, 0); // no room: this lane draws it
          }
      }
    }
    __syncwarp(); // world_s / clip_s reuse
  }
}

__global__ void __launch_bounds__(VSM_DRAW_THREADS) k_vsm_draw_items(const __grid_constant__ VsmDrawParams p) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t n = min(p.counters[0], p.queue_capacity);
  for (uint32_t i = blockIdx.x * VSM_DRAW_WARPS + warp; i < n; i += gridDim.x * VSM_DRAW_WARPS) vsm_draw_item(p, p.queue[i], 32, (int)lane);
}

} // namespace oxc
