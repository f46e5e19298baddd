// kernels_tri.cuh — per-triangle cull (+ index-buffer output) and the software visibility-buffer raster.
// Reference: passes/cull_triangles.slang:27-90, passes/visbuffer_encode_ms.slang:110-171 (per-vertex
// transform into shared memory, per-primitive cull), visbuffer.slang:49-79 (64-bit depth|data packing).
// The raster itself has no reference implementation (HW rasteriser, DrawGeometry.cpp:104-190); its
// specification is the comment block above raster_triangle() in oracle/oxc_oracle.c (DESIGN.md §raster).
#pragma once
#include <climits>

#include "oxc_exact.cuh"
#include "oxc_raster_core.cuh"

namespace oxc {

#ifndef OXC_TRI_THREADS
#define OXC_TRI_THREADS 256
#endif
constexpr int TRI_THREADS = OXC_TRI_THREADS;
constexpr int TRI_WARPS = TRI_THREADS / 32;

struct TriParams {
  const OxcMeshletInstance* meshlet_instances;
  const InstCull* inst;
  const InstGeom* geom;
  const OxcMeshletInstanceVisibility* vis;
  const OxcDispatchIndirectCommand* tri_cmd;
  const uint32_t* visible_indices;
  const uint32_t* id_base;   // may be null; visible_indices already carry it, meshlet_instances is local
  uint32_t late;             // 0: survivors [0,E); 1: [E,E+L)   (cull_triangles.slang:34-37)
  // cull_triangles output
  uint32_t* reordered_indices;
  OxcDrawIndexedIndirectCommand* draw_cmd;
  // raster output
  unsigned long long* visbuf;
  uint32_t width, height;
  float f_width, f_height;   // (float)width / height: kernel-parameter operands cost no registers
  unsigned long long* tri_counter;
  uint32_t* work_counter;    // zeroed before every raster launch
  // deferred large triangles (k_raster_big): [0] = entries pushed, [1] = entries taken; zeroed before every raster launch
  uint4* big_queue;          // BIG_WORDS/4 uint4 per entry
  uint32_t* big_counters;
  uint32_t big_capacity;
  uint32_t* deferred_queue;  // data words (id << prim_bits | triangle) of the triangles a lane does not draw itself: k_raster_deferred
  uint32_t* deferred_counter; // entries pushed (keeps counting past the capacity); zeroed before every raster launch
  uint32_t deferred_capacity;
  uint32_t prim_bits;        // triangle bits of the vis-buffer word: 8 (visbuffer.slang:9-14) or 6 (OxcCreateInfo::wide_ids)
  uint32_t small_primitive_cull; // 1: triangles whose snapped bounding box holds no sample centre are culled before they are counted
  uint32_t* status;          // sticky OXC_STATUS_* bits
};

struct MeshletWork {
  uint32_t data_id;    // global meshlet instance id (<< 8 | tri later)
  uint32_t tri_count;
  uint32_t tri_offset; // byte offset of the micro indices
  uint32_t vertex_count;
  const uint32_t* micro;
};

// Loads one surviving meshlet for a warp: resolves the pointer chase, transforms its <=64 vertices ONCE
// (clip = mvp * (pos,1), visbuffer_encode_ms.slang:135-137 — same values cull_triangles.slang:62-66
// recomputes per corner) into the warp's shared-memory slab.
OXC_DI MeshletWork load_meshlet(const TriParams& p, uint32_t slot, uint32_t id_base, float4* clip_s, uint32_t lane) {
  MeshletWork w;
  const uint32_t gid = __ldg(&p.visible_indices[slot]);      // :44 (global id)
  const uint32_t local = gid - id_base;
  const uint2 mi = __ldg(reinterpret_cast<const uint2*>(p.meshlet_instances) + local); // :45
  const InstGeom* g = p.geom + mi.x;
  const InstCull* ic = p.inst + mi.x;
  const uint4 m = __ldg(reinterpret_cast<const uint4*>(g->meshlets + mi.y)); // Meshlet, :49
  const uint32_t vertex_offset = m.x, vertex_count = min(m.z, (uint32_t)OXC_MESHLET_MAX_VERTICES);
  w.tri_offset = m.y;
  w.tri_count = min(m.w, (uint32_t)OXC_MESHLET_MAX_PRIMITIVES);
  w.vertex_count = vertex_count;
  w.micro = g->local_triangle_indices;
  w.data_id = gid;
  const float4 r0 = __ldg(&ic->mvp_row[0]), r1 = __ldg(&ic->mvp_row[1]), r2 = __ldg(&ic->mvp_row[2]), r3 = __ldg(&ic->mvp_row[3]);
  const uint32_t* vidx = g->indirect_vertex_indices + vertex_offset;
  const uint2* pos = g->vertex_positions;
  for (uint32_t v = lane; v < vertex_count; v += 32) {
    const uint32_t vi = __ldg(&vidx[v]);
    const uint2 q = __ldg(&pos[vi]); // u16x4
    const float x = dequantize_half(q.x & 0xFFFFu), y = dequantize_half(q.x >> 16), z = dequantize_half(q.y & 0xFFFFu);
    clip_s[v] = make_float4(row_dot_p1(r0, x, y, z), row_dot_p1(r1, x, y, z), row_dot_p1(r2, x, y, z), row_dot_p1(r3, x, y, z));
  }
  __syncwarp();
  return w;
}

// scene.slang:336-342 get_micro_index
OXC_DI uint32_t micro_index(const uint32_t* __restrict__ buf, uint32_t byte_offset) {
  return (__ldg(&buf[byte_offset >> 2]) >> ((byte_offset & 3u) * 8u)) & 0xFFu;
}

// cull_triangles.slang:59-69
OXC_DI bool triangle_passes(const MeshletWork& w, uint32_t t, const float4* clip_s, float4& c0, float4& c1, float4& c2) {
  const uint32_t base = w.tri_offset + t * 3u;
  const uint32_t i0 = micro_index(w.micro, base + 0u), i1 = micro_index(w.micro, base + 1u), i2 = micro_index(w.micro, base + 2u);
  if (max(i0, max(i1, i2)) >= w.vertex_count) return false; // malformed meshlet: never index past the transformed vertices
  c0 = clip_s[i0];
  c1 = clip_s[i1];
  c2 = clip_s[i2];
  const bool in_front = c0.z >= 0.0f && c1.z >= 0.0f && c2.z >= 0.0f;
  return in_front && !triangle_backface(c0, c1, c2);
}

// ---- cull_triangles: materialise the reference's reordered index buffer ----
__global__ void __launch_bounds__(TRI_THREADS) k_cull_triangles(const __grid_constant__ TriParams p) {
  __shared__ float4 clip_all[TRI_WARPS][OXC_MESHLET_MAX_VERTICES];
  __shared__ uint32_t warp_cnt[TRI_WARPS];
  __shared__ uint32_t base_s;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t first = p.late ? p.vis->early_visible_meshlet_instances : 0u; // cull_triangles.slang:34-37
  const uint32_t count = p.tri_cmd->x;                                         // dispatch_indirect(cull_triangles_cmd), CullGeometry.cpp:365
  const uint32_t id_base = p.id_base ? __ldg(p.id_base) : 0u;
  const uint32_t n_tiles = (count + TRI_WARPS - 1) / TRI_WARPS;
  float4* clip_s = clip_all[warp];
  for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const uint32_t g = tile * TRI_WARPS + warp;
    bool pass[2] = {false, false};
    uint32_t rank[2] = {0, 0}, wtotal = 0, data_id = 0;
    if (g < count) {
      const MeshletWork w = load_meshlet(p, first + g, id_base, clip_s, lane);
      data_id = w.data_id;
#pragma unroll
      for (int k = 0; k < 2; k++) {
        const uint32_t t = lane + 32u * k;
        float4 c0, c1, c2;
        pass[k] = t < w.tri_count && triangle_passes(w, t, clip_s, c0, c1, c2);
        // opt-in small-primitive cull (north_star; the reference has none): snapped bounding box without a sample centre
        if (pass[k] && p.small_primitive_cull && tri_covers_no_sample(c0, c1, c2, p.f_width, p.f_height, p.width, p.height)) pass[k] = false;
        const uint32_t bal = __ballot_sync(0xffffffffu, pass[k]);
        rank[k] = wtotal + __popc(bal & ((1u << lane) - 1u));
        wtotal += __popc(bal);
      }
      __syncwarp();
    }
    if (lane == 0) warp_cnt[warp] = wtotal;
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t s = 0;
#pragma unroll
      for (int k = 0; k < TRI_WARPS; k++) { const uint32_t c = warp_cnt[k]; warp_cnt[k] = s; s += c; }
      base_s = s ? atomicAdd(&p.draw_cmd->index_count, s * 3u) : 0u; // :78
    }
    __syncthreads();
    const uint32_t wbase = base_s + warp_cnt[warp] * 3u;
#pragma unroll
    for (int k = 0; k < 2; k++)
      if (pass[k]) {
        const uint32_t t = lane + 32u * k, off = wbase + rank[k] * 3u, masked = data_id << OXC_VIS_PRIMITIVE_BITS; // :84-88
        p.reordered_indices[off + 0] = masked | ((t * 3u + 0u) & OXC_VIS_PRIMITIVE_MASK);
        p.reordered_indices[off + 1] = masked | ((t * 3u + 1u) & OXC_VIS_PRIMITIVE_MASK);
        p.reordered_indices[off + 2] = masked | ((t * 3u + 2u) & OXC_VIS_PRIMITIVE_MASK);
      }
    __syncthreads();
  }
}

// 3 CTAs / SM: 76 registers without spills.  At 4 (64 registers) the early and late passes store 24 and 44 B of spills, and on an
// H100 80GB HBM3 (700 W) at 1 M meshlet instances / 1080p the early raster takes 316-319 instead of 312-314 us and the late one
// 74 instead of 68-70 us (BASELINE.md 5.16); at 5 (48 registers) they store 140 and 164 B of spills.
#ifndef OXC_RASTER_MIN_BLOCKS
#define OXC_RASTER_MIN_BLOCKS 3
#endif
// 32 meshlets per grab (one per lane) and up to 128 pixels per lane-drawn triangle rather than 8 and 32: on H100 SXM at 1 M
// meshlet instances / 1080p the early raster takes 352-357 instead of 392-399 us, with fewer grabs on the contended work counter
// and fewer triangles through the warp-wide hand-off and the chunk queue (BASELINE.md 5.3).
#ifndef OXC_RASTER_BIG_PIXELS
#define OXC_RASTER_BIG_PIXELS 128
#endif
#ifndef OXC_RASTER_BATCH
#define OXC_RASTER_BATCH 32
#endif
constexpr int RASTER_BATCH = OXC_RASTER_BATCH;       // meshlets per work grab
static_assert(RASTER_BATCH >= 1 && RASTER_BATCH <= 32, "one header per lane: a grab holds at most 32 meshlets");
constexpr int RASTER_BIG_PIXELS = OXC_RASTER_BIG_PIXELS; // bbox area above which the whole warp rasterises the triangle together

// Header of one surviving meshlet, fetched by ONE lane (32 headers in flight per warp): the 4-level pointer
// chase visible_indices -> meshlet_instances -> InstGeom -> Meshlet is paid once per 32 meshlets per warp.
struct MeshletHeader {
  uint32_t gid, inst, vertex_offset, vertex_count, tri_offset, tri_count;
  const uint32_t* micro;
  const uint32_t* vidx;
  const uint2* pos;
};

OXC_DI MeshletHeader fetch_header(const TriParams& p, uint32_t slot, uint32_t id_base) {
  MeshletHeader h;
  h.gid = __ldg(&p.visible_indices[slot]);                                                    // cull_triangles.slang:44
  const uint2 mi = __ldg(reinterpret_cast<const uint2*>(p.meshlet_instances) + (h.gid - id_base)); // :45
  const InstGeom* g = p.geom + mi.x;
  const uint4 g0 = __ldg(reinterpret_cast<const uint4*>(g));      // meshlets, local_triangle_indices
  const uint4 g1 = __ldg(reinterpret_cast<const uint4*>(g) + 1);  // indirect_vertex_indices, vertex_positions
  const OxcMeshlet* meshlets = reinterpret_cast<const OxcMeshlet*>(((uint64_t)g0.y << 32) | g0.x);
  const uint4 m = __ldg(reinterpret_cast<const uint4*>(meshlets + mi.y));                    // :49
  h.inst = mi.x;
  h.vertex_offset = m.x;
  h.tri_offset = m.y;
  h.vertex_count = min(m.z, (uint32_t)OXC_MESHLET_MAX_VERTICES);
  h.tri_count = min(m.w, (uint32_t)OXC_MESHLET_MAX_PRIMITIVES);
  h.micro = reinterpret_cast<const uint32_t*>(((uint64_t)g0.w << 32) | g0.z);
  h.vidx = reinterpret_cast<const uint32_t*>(((uint64_t)g1.y << 32) | g1.x) + m.x;
  h.pos = reinterpret_cast<const uint2*>(((uint64_t)g1.w << 32) | g1.z);
  return h;
}

OXC_DI MeshletHeader bcast_header(const MeshletHeader& h, int src) {
  MeshletHeader o;
  o.gid = __shfl_sync(0xffffffffu, h.gid, src); o.inst = __shfl_sync(0xffffffffu, h.inst, src);
  o.vertex_offset = 0;
  o.vertex_count = __shfl_sync(0xffffffffu, h.vertex_count, src);
  o.tri_offset = __shfl_sync(0xffffffffu, h.tri_offset, src); o.tri_count = __shfl_sync(0xffffffffu, h.tri_count, src);
  o.micro = reinterpret_cast<const uint32_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(h.micro), src));
  o.vidx = nullptr; // load_vertex_indices
  o.pos = reinterpret_cast<const uint2*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(h.pos), src));
  return o;
}

// the vertex indices of the meshlet whose header lane src holds: lane l loads indices l and l + 32
OXC_DI void load_vertex_indices(const MeshletHeader& h, int src, uint32_t lane, uint32_t& vi0, uint32_t& vi1) {
  const uint32_t n = __shfl_sync(0xffffffffu, h.vertex_count, src);
  const uint32_t* vidx = reinterpret_cast<const uint32_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(h.vidx), src));
  vi0 = lane < n ? __ldg(&vidx[lane]) : 0u;
  vi1 = lane + 32u < n ? __ldg(&vidx[lane + 32u]) : 0u;
}

// ---- deferred large triangles ----
// A triangle whose pixel bounding box exceeds RASTER_BIG_PIXELS is not rasterised by the warp that found it: a meshlet
// close to the camera has dozens of them (hundreds of thousands of instructions for ONE warp, the tail of the launch).
// They are pushed to a global queue, split into chunks of at most BIG_CHUNK_W x BIG_CHUNK_H pixels, and k_raster_big
// spreads the chunks over every warp of the GPU.  Entry = the TriSetup with the chunk's bounding box + the vis data word.
constexpr int BIG_CHUNK_W = 64, BIG_CHUNK_H = 32;

OXC_DI void big_entry_store(uint4* dst, const TriSetup& s, int px0, int px1, int py0, int py1, uint32_t data) {
  dst[0] = make_uint4((uint32_t)s.ax, (uint32_t)s.ay, (uint32_t)s.bx, (uint32_t)s.by);
  dst[1] = make_uint4((uint32_t)s.cx, (uint32_t)s.cy, __float_as_uint(s.za), __float_as_uint(s.dzb));
  dst[2] = make_uint4(__float_as_uint(s.dzc), (uint32_t)px0, (uint32_t)px1, (uint32_t)py0);
  dst[3] = make_uint4((uint32_t)py1, (uint32_t)s.bias, data, 0u);
}

OXC_DI void big_entry_load(const uint4* src, TriSetup& s, uint32_t& data) {
  const uint4 a = src[0], b = src[1], c = src[2], d = src[3];
  s.ax = (int)a.x; s.ay = (int)a.y; s.bx = (int)a.z; s.by = (int)a.w;
  s.cx = (int)b.x; s.cy = (int)b.y; s.za = __uint_as_float(b.z); s.dzb = __uint_as_float(b.w);
  s.dzc = __uint_as_float(c.x); s.px0 = (int)c.y; s.px1 = (int)c.z; s.py0 = (int)c.w;
  s.py1 = (int)d.x; s.bias = (int)d.y; s.narrow = false;
  data = d.z;
}

// Pushes the triangle as chunks; returns false when the queue cannot take all of them (the caller then rasterises the
// triangle inline).  Reservations are never undone — with concurrent pushers an undo would shift other warps' slots —,
// so a reservation that straddles the capacity fills its slots below the capacity with EMPTY entries (px1 < px0), and
// the consumer processes min(counter, capacity) entries.
OXC_DI bool big_push(const TriParams& p, const TriSetup& s, uint32_t data) {
  if (*reinterpret_cast<volatile uint32_t*>(&p.big_counters[0]) >= p.big_capacity) return false; // also bounds the counter's growth
  const uint32_t cw = (uint32_t)(s.px1 - s.px0) / BIG_CHUNK_W + 1u, ch = (uint32_t)(s.py1 - s.py0) / BIG_CHUNK_H + 1u;
  const uint32_t n = cw * ch;
  const uint32_t base = atomicAdd(&p.big_counters[0], n);
  if (base >= p.big_capacity) return false;
  if (base + n > p.big_capacity) {
    for (uint32_t k = base; k < p.big_capacity; k++) big_entry_store(p.big_queue + (size_t)k * 4, s, 1, 0, 1, 0, data);
    return false;
  }
  uint32_t k = base;
  for (uint32_t cy = 0; cy < ch; cy++)
    for (uint32_t cx = 0; cx < cw; cx++, k++) {
      const int x0 = s.px0 + (int)(cx * BIG_CHUNK_W), y0 = s.py0 + (int)(cy * BIG_CHUNK_H);
      big_entry_store(p.big_queue + (size_t)k * 4, s, x0, min(s.px1, x0 + BIG_CHUNK_W - 1), y0, min(s.py1, y0 + BIG_CHUNK_H - 1), data);
    }
  return true;
}

// The same push done by a whole warp for ONE triangle (every lane holds its setup): lane l writes chunks l, l + 32, ...
OXC_DI bool big_push_warp(const TriParams& p, const TriSetup& s, uint32_t data, uint32_t lane) {
  const uint32_t cw = (uint32_t)(s.px1 - s.px0) / BIG_CHUNK_W + 1u, ch = (uint32_t)(s.py1 - s.py0) / BIG_CHUNK_H + 1u;
  const uint32_t n = cw * ch;
  uint32_t base = 0xFFFFFFFFu;
  if (lane == 0 && *reinterpret_cast<volatile uint32_t*>(&p.big_counters[0]) < p.big_capacity) base = atomicAdd(&p.big_counters[0], n);
  base = __shfl_sync(0xffffffffu, base, 0);
  if (base >= p.big_capacity) return false;
  if (base + n > p.big_capacity) { // straddles the capacity: fill the reserved slots below it with EMPTY entries (see big_push)
    for (uint32_t k = base + lane; k < p.big_capacity; k += 32) big_entry_store(p.big_queue + (size_t)k * 4, s, 1, 0, 1, 0, data);
    return false;
  }
  for (uint32_t k = lane; k < n; k += 32) {
    const uint32_t cy = k / cw, cx = k - cy * cw;
    const int x0 = s.px0 + (int)(cx * BIG_CHUNK_W), y0 = s.py0 + (int)(cy * BIG_CHUNK_H);
    big_entry_store(p.big_queue + (size_t)(base + k) * 4, s, x0, min(s.px1, x0 + BIG_CHUNK_W - 1), y0, min(s.py1, y0 + BIG_CHUNK_H - 1), data);
  }
  return true;
}

// The whole warp covers the box of one set-up triangle in 8x4-pixel tiles (raster spec steps 5-6).
OXC_DI void raster_tiles(const TriParams& p, const TriSetup& b, uint32_t data, uint32_t lane) {
  const int lx = lane & 7, ly = lane >> 3;
  for (int ty = b.py0; ty <= b.py1; ty += 4)
    for (int tx = b.px0; tx <= b.px1; tx += 8) {
      const int px = tx + lx, py = ty + ly;
      if (px <= b.px1 && py <= b.py1) raster_pixel(b, px, py, data, p.visbuf, p.width);
    }
}

// One warp per queued chunk.  Chunks are dealt to the warps of the grid round-robin: taking them from a counter costs every
// warp one same-address atomic, even just to learn that the queue is empty.
__global__ void __launch_bounds__(256) k_raster_big(const __grid_constant__ TriParams p) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t total = min(p.big_counters[0], p.big_capacity);
  for (uint32_t i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < total; i += gridDim.x * (blockDim.x >> 5)) {
    TriSetup b;
    uint32_t data;
    big_entry_load(p.big_queue + (size_t)i * 4, b, data);
    raster_tiles(p, b, data, lane);
  }
}

// A lane draws a set-up triangle itself when its edge functions fit 32 bits and its box holds at most RASTER_BIG_PIXELS
// pixels; k_raster_deferred draws the others (and clips the triangles with an invalid vertex).
OXC_DI bool lane_draws(const TriSetup& s) { return s.narrow && (s.px1 - s.px0 + 1) * (s.py1 - s.py0 + 1) <= RASTER_BIG_PIXELS; }

#if defined(OXC_RASTER_STATS) && OXC_RASTER_STATS == 1
// Statistics build only. Warp-wide, over every lane's v0 (when has0) and v1 (when has1): true when the snapped pixel box of the
// vertices, clamped to the image as tri_setup clamps a triangle's, holds no sample centre and no vertex is invalid.  Every
// triangle's corners are meshlet vertices and snap and clamp are monotone, so every triangle of such a meshlet is TRI_NO_SAMPLE.
// The coordinates are reduced as unsigned with the sign bit flipped, which orders them as signed ints.
OXC_DI bool meshlet_covers_no_sample(const ScreenVert& v0, const ScreenVert& v1, bool has0, bool has1, uint32_t W, uint32_t H) {
  constexpr int FAR = 1 << 30; // identity: beyond the snap range (|fx|, |fy| <= 2^22), and the snap below cannot overflow on it
  constexpr uint32_t SIGN = 0x80000000u;
  const bool ok0 = has0 && v0.fx != INT_MIN, ok1 = has1 && v1.fx != INT_MIN;
  const int lx = min(ok0 ? v0.fx : FAR, ok1 ? v1.fx : FAR), hx = max(ok0 ? v0.fx : -FAR, ok1 ? v1.fx : -FAR);
  const int ly = min(ok0 ? v0.fy : FAR, ok1 ? v1.fy : FAR), hy = max(ok0 ? v0.fy : -FAR, ok1 ? v1.fy : -FAR);
  const int minx = (int)(__reduce_min_sync(0xffffffffu, (uint32_t)lx ^ SIGN) ^ SIGN);
  const int maxx = (int)(__reduce_max_sync(0xffffffffu, (uint32_t)hx ^ SIGN) ^ SIGN);
  const int miny = (int)(__reduce_min_sync(0xffffffffu, (uint32_t)ly ^ SIGN) ^ SIGN);
  const int maxy = (int)(__reduce_max_sync(0xffffffffu, (uint32_t)hy ^ SIGN) ^ SIGN);
  const int px0 = max(0, (minx - 128 + 255) >> 8), px1 = min((int)W - 1, (maxx - 128) >> 8);
  const int py0 = max(0, (miny - 128 + 255) >> 8), py1 = min((int)H - 1, (maxy - 128) >> 8);
  const bool any_invalid = __any_sync(0xffffffffu, (has0 && !ok0) || (has1 && !ok1));
  return (px1 < px0 || py1 < py0) && !any_invalid;
}
#endif

template <bool PREFETCH_GRAB>
__global__ void __launch_bounds__(TRI_THREADS, OXC_RASTER_MIN_BLOCKS) k_raster_visbuffer(const __grid_constant__ TriParams p) {
  __shared__ float4 clip_all[TRI_WARPS][OXC_MESHLET_MAX_VERTICES];
  __shared__ ScreenVert scr_all[TRI_WARPS][OXC_MESHLET_MAX_VERTICES];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // the meshlet's micro-index run (<= 192 B, scene.slang:336-342) staged in shared memory: 49 words cover it plus the byte skew
  // of its start.  Two coalesced loads per warp, issued before the vertex transform, replace three dependent L1 loads + shifts
  // per triangle.
  __shared__ uint32_t micro_w[TRI_WARPS][52];
  const uint32_t first = p.late ? p.vis->early_visible_meshlet_instances : 0u; // cull_triangles.slang:34-37
  const uint32_t count = p.tri_cmd->x;                                         // dispatch_indirect(cull_triangles_cmd), CullGeometry.cpp:365
  const uint32_t id_base = p.id_base ? __ldg(p.id_base) : 0u;
  float4* clip_s = clip_all[warp];
  ScreenVert* scr_s = scr_all[warp];
  uint32_t kept = 0;
#ifdef OXC_RASTER_STATS
  unsigned long long t_entry, t_chase = 0, t_proc = 0, n_done = 0, n_grabs = 0;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_entry));
#endif
  // warps pull batches of up to RASTER_BATCH consecutive survivors from a global work counter (dynamic balance); lanes
  // 0..nb-1 each chase one meshlet header, so nb pointer chases are in flight together.
  // Guided self-scheduling: the grab size shrinks with the work that is left (remaining / (k x warps in the grid), between 1
  // and RASTER_BATCH), so the kernel ends with single-meshlet grabs.  The early pass divides by the warps (k = 1): its grabs
  // stay at 32 meshlets until 38 % of the list is left instead of 77 % (1 M meshlet instances / 1080p), and each grab costs a
  // header chase.  On H100 SXM that takes the early raster from 355-357 to 325-328 us (BASELINE.md 5.8).  The late
  // pass, which holds a prefetched grab in reserve, keeps k = 2: at k = 1 it took 81 instead of 69 us.
  // A grab is slow (thousands of warps on one L2 atomic address; tools/raster_stats.py times it per warp).  Dealing the list
  // onto 32 interleaved sequences with one counter each would shorten the late pass, but the extra scheduler state is more
  // live registers in a kernel that already spills at its bound, so the single counter stays (not re-timed on H100).
  const uint32_t grab_divisor = gridDim.x * TRI_WARPS * (PREFETCH_GRAB ? 2u : 1u);
  // PREFETCH_GRAB (late pass): the grab for the NEXT batch is issued before the current batch is processed, so the atomic's
  // round trip (long in the late pass: every warp of the GPU on one address, few meshlets per warp) overlaps a batch of
  // rasterisation.  The early pass (many meshlets per warp, few grabs) loses more balance from the batch each warp holds in
  // reserve than it gains, so it keeps the plain grab: its waiting warps cost nothing while the others have instructions to
  // issue.
  uint32_t g_next = 0, batch_next = 1;
  if (PREFETCH_GRAB && lane == 0) {
    batch_next = min((uint32_t)RASTER_BATCH, max(1u, count / grab_divisor));
    g_next = atomicAdd(p.work_counter, batch_next);
  }
  for (;;) {
    uint32_t g0 = 0, batch = 1;
    if (PREFETCH_GRAB) {
      g0 = __shfl_sync(0xffffffffu, g_next, 0);
      batch = __shfl_sync(0xffffffffu, batch_next, 0);
      if (g0 >= count) break;
      if (lane == 0) { // reserve the following batch now; its index is not needed before the next iteration
        const uint32_t seen = g0 + batch; // what had been handed out when this batch was reserved (a lower bound now)
        const uint32_t rem = count > seen ? count - seen : 0u;
        batch_next = min((uint32_t)RASTER_BATCH, max(1u, rem / grab_divisor));
        g_next = atomicAdd(p.work_counter, batch_next);
      }
    } else {
      if (lane == 0) {
        const uint32_t seen = *reinterpret_cast<volatile uint32_t*>(p.work_counter); // heuristic only: a stale value is harmless
        const uint32_t rem = count > seen ? count - seen : 0u;
        batch = min((uint32_t)RASTER_BATCH, max(1u, rem / grab_divisor));
        g0 = atomicAdd(p.work_counter, batch);
      }
      g0 = __shfl_sync(0xffffffffu, g0, 0);
      batch = __shfl_sync(0xffffffffu, batch, 0);
      if (g0 >= count) break;
    }
    const uint32_t nb = min(batch, count - g0);
    const uint32_t my_survivor = g0 + lane;
#ifdef OXC_RASTER_STATS
    unsigned long long t_a, t_b, t_c;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_a));
#endif
    MeshletHeader mine;
    mine.gid = 0; mine.inst = 0; mine.vertex_offset = 0; mine.vertex_count = 0; mine.tri_offset = 0; mine.tri_count = 0;
    mine.micro = nullptr; mine.vidx = nullptr; mine.pos = nullptr;
    if (lane < nb) mine = fetch_header(p, first + my_survivor, id_base);
    // vertex indices of the first meshlet, prefetched one meshlet ahead from here on
    uint32_t vi0, vi1;
    load_vertex_indices(mine, 0, lane, vi0, vi1);
#ifdef OXC_RASTER_STATS
    if (vi0 + vi1 == 0xFFFFFFFFu) kept++; // keep the loads ahead of the timer read
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_b));
#endif
    for (uint32_t j = 0; j < nb; j++) {
      // broadcast again from lane j rather than carried over from the previous meshlet: a header held across the pixel loops
      // costs registers the loops need
      const MeshletHeader w = bcast_header(mine, (int)j);
      {  // words [tri_offset / 4, ...) covering the run: two coalesced loads per warp, in flight during the vertex phase
        const uint32_t n_words = ((w.tri_offset & 3u) + w.tri_count * 3u + 3u) >> 2;
        const uint32_t* src = w.micro + (w.tri_offset >> 2);
        const uint32_t m0 = lane < n_words ? __ldg(src + lane) : 0u;
        const uint32_t m1 = lane + 32u < n_words ? __ldg(src + lane + 32u) : 0u;
        micro_w[warp][lane] = m0;
        if (lane < 20) micro_w[warp][lane + 32] = m1;
      }
      // positions of this meshlet (indices already here) ...
      const uint2 q0 = lane < w.vertex_count ? __ldg(&w.pos[vi0]) : make_uint2(0, 0);
      const uint2 q1 = lane + 32u < w.vertex_count ? __ldg(&w.pos[vi1]) : make_uint2(0, 0);
      // ... and the next meshlet's vertex indices, in flight while this one is rasterised
      if (j + 1 < nb) load_vertex_indices(mine, (int)(j + 1), lane, vi0, vi1);
      const InstCull* ic = p.inst + w.inst;
      const float4 r0 = __ldg(&ic->mvp_row[0]), r1 = __ldg(&ic->mvp_row[1]), r2 = __ldg(&ic->mvp_row[2]), r3 = __ldg(&ic->mvp_row[3]);
      // clip = mvp * (pos,1) once per vertex (visbuffer_encode_ms.slang:135-137), then the screen record
      {
        const float x = dequantize_half_hw(q0.x & 0xFFFFu), y = dequantize_half_hw(q0.x >> 16), z = dequantize_half_hw(q0.y & 0xFFFFu);
        const float4 c = make_float4(row_dot_p1(r0, x, y, z), row_dot_p1(r1, x, y, z), row_dot_p1(r2, x, y, z), row_dot_p1(r3, x, y, z));
        clip_s[lane] = c;
        scr_s[lane] = to_screen(c, p.f_width, p.f_height);
      }
      if (w.vertex_count > 32u) {
        const float x = dequantize_half_hw(q1.x & 0xFFFFu), y = dequantize_half_hw(q1.x >> 16), z = dequantize_half_hw(q1.y & 0xFFFFu);
        const float4 c = make_float4(row_dot_p1(r0, x, y, z), row_dot_p1(r1, x, y, z), row_dot_p1(r2, x, y, z), row_dot_p1(r3, x, y, z));
        clip_s[lane + 32] = c;
        scr_s[lane + 32] = to_screen(c, p.f_width, p.f_height);
      }
      __syncwarp();
      const uint32_t rounds = (w.tri_count + 31u) >> 5;
#if defined(OXC_RASTER_STATS) && OXC_RASTER_STATS == 1
      bool meshlet_draws = false;
      // meshlets that a per-meshlet footprint test could settle without any triangle set-up
      if (meshlet_covers_no_sample(scr_s[lane], scr_s[lane + 32], lane < w.vertex_count, lane + 32u < w.vertex_count, p.width, p.height) &&
          lane == 0)
        atomicAdd(reinterpret_cast<unsigned long long*>(p.big_queue) + (size_t)p.big_capacity * 8 + (p.late ? 64 : 0) + 48, 1ull);
#endif
      for (uint32_t k = 0; k < rounds; k++) {
        const uint32_t t = lane + 32u * k;
        bool pass = false;
        TriSetup s;
        bool draw = false, defer = false, clip = false;
#if defined(OXC_RASTER_STATS) && OXC_RASTER_STATS == 1
        int why_stat = -1;
#endif
        if (t < w.tri_count) {
          const uint8_t* mb = reinterpret_cast<const uint8_t*>(micro_w[warp]) + (w.tri_offset & 3u) + t * 3u;
          const uint32_t i0 = mb[0], i1 = mb[1], i2 = mb[2];
          if (max(i0, max(i1, i2)) < w.vertex_count) { // malformed meshlets never index past the transformed vertices
            const float4 c0 = clip_s[i0], c1 = clip_s[i1], c2 = clip_s[i2];
            pass = c0.z >= 0.0f && c1.z >= 0.0f && c2.z >= 0.0f && !triangle_backface(c0, c1, c2); // cull_triangles.slang:68-69
            if (pass) {
              const int why = tri_setup(scr_s[i0], scr_s[i1], scr_s[i2], p.width, p.height, s);
#if defined(OXC_RASTER_STATS) && OXC_RASTER_STATS == 1
              why_stat = why;
#endif
              draw = why == TRI_DRAW && lane_draws(s);
              // a vertex at w <= 0 / beyond the snap range (clipped later, like a hardware rasteriser would,
              // DrawGeometry.cpp:104-190), 64-bit edge functions or a large box: k_raster_deferred
              clip = why == TRI_INVALID_VERTEX;
              defer = clip || (why == TRI_DRAW && !draw);
              if (why == TRI_NO_SAMPLE && p.small_primitive_cull) pass = false; // north_star small-primitive cull (opt-in)
            }
          }
        }
        kept += pass ? 1u : 0u;
        const uint32_t data = (w.gid << p.prim_bits) | t;
#if defined(OXC_RASTER_STATS) && OXC_RASTER_STATS == 1
        {  // instrumentation build only: per round (32 triangles) histogram of the LARGEST per-lane pixel loop and the round's sums
          const bool set_up = why_stat == TRI_DRAW;
          const int bw = set_up ? s.px1 - s.px0 + 1 : 0, bh = set_up ? s.py1 - s.py0 + 1 : 0;
          const int area = draw ? bw * bh : 0;
          const int mx = __reduce_max_sync(0xffffffffu, area), sm = __reduce_add_sync(0xffffffffu, area);
          const int nd = __popc(__ballot_sync(0xffffffffu, area > 0));
          const int nbig = __popc(__ballot_sync(0xffffffffu, bw * bh > RASTER_BIG_PIXELS));
          const int nwide = __popc(__ballot_sync(0xffffffffu, set_up && !s.narrow));
          const int nclip = __popc(__ballot_sync(0xffffffffu, clip));
          const int ndefer = __popc(__ballot_sync(0xffffffffu, defer));
          const int nsetup = __popc(__ballot_sync(0xffffffffu, set_up));
          const bool setup_round = __any_sync(0xffffffffu, why_stat == TRI_DRAW || why_stat == TRI_BACK_OR_DEGENERATE);
          meshlet_draws |= __any_sync(0xffffffffu, set_up);
          if (lane == 0) {
            unsigned long long* st = reinterpret_cast<unsigned long long*>(p.big_queue) + (size_t)p.big_capacity * 8 + (p.late ? 64 : 0);
            atomicAdd(&st[min(mx, 33)], 1ull);          // [0..33] histogram of max area
            atomicAdd(&st[40], (unsigned long long)sm); // total candidate pixels (per-lane path)
            atomicAdd(&st[41], (unsigned long long)mx); // sum of per-round maxima
            atomicAdd(&st[42], (unsigned long long)nd); // drawing lanes
            atomicAdd(&st[43], 1ull);                   // rounds
            atomicAdd(&st[44], (unsigned long long)nbig);
            if (setup_round) atomicAdd(&st[47], 1ull); // rounds in which some lane runs the set-up past the bounding box
            atomicAdd(&st[49], (unsigned long long)nwide);  // set-up triangles that fail narrow
            atomicAdd(&st[50], (unsigned long long)nclip);  // TRI_INVALID_VERTEX triangles (clipped)
            atomicAdd(&st[51], (unsigned long long)ndefer); // deferred-queue entries
            atomicAdd(&st[52], (unsigned long long)nsetup); // set-up triangles (TRI_DRAW)
          }
        }
#endif
        if (draw) raster_narrow(s, data, p.visbuf, p.width);
        // the rest goes to the deferred queue, one atomic per round from the first deferring lane.  Past the capacity the counter
        // keeps counting, and k_raster_deferred walks the pass again for the triangles the queue could not hold.  A clipped
        // triangle past it also raises OXC_STATUS_CLIP_OVERFLOW: the queue is too small for the frame, and the walk is slow.
        const uint32_t defer_mask = __ballot_sync(0xffffffffu, defer);
        if (defer_mask) {
          const int leader = __ffs(defer_mask) - 1;
          uint32_t base = 0;
          if (lane == (uint32_t)leader) base = atomicAdd(p.deferred_counter, (uint32_t)__popc(defer_mask));
          const uint32_t slot = __shfl_sync(0xffffffffu, base, leader) + __popc(defer_mask & ((1u << lane) - 1u));
          if (defer && slot < p.deferred_capacity) p.deferred_queue[slot] = data;
          else if (clip) atomicOr(p.status, (uint32_t)OXC_STATUS_CLIP_OVERFLOW);
        }
      }
#if defined(OXC_RASTER_STATS) && OXC_RASTER_STATS == 1
      if (lane == 0 && meshlet_draws) // meshlets with at least one drawing triangle
        atomicAdd(reinterpret_cast<unsigned long long*>(p.big_queue) + (size_t)p.big_capacity * 8 + (p.late ? 64 : 0) + 46, 1ull);
#endif
      __syncwarp(); // clip_s / scr_s reuse
    }
#ifdef OXC_RASTER_STATS
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_c));
    t_chase += t_b - t_a; t_proc += t_c - t_b; n_done += nb; n_grabs++;
#endif
  }
#ifdef OXC_RASTER_STATS
  if (lane == 0) { // per-warp record: entry, exit, time in the header chase, time processing, meshlets, grabs
    unsigned long long t_exit;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_exit));
    unsigned long long* rec = reinterpret_cast<unsigned long long*>(p.big_queue) + (size_t)p.big_capacity * 8 + 128 +
                              ((size_t)(p.late ? gridDim.x * TRI_WARPS : 0) + blockIdx.x * TRI_WARPS + warp) * 6;
    rec[0] = t_entry; rec[1] = t_exit; rec[2] = t_chase; rec[3] = t_proc; rec[4] = n_done; rec[5] = n_grabs;
    if (blockIdx.x == 0 && warp == 0) // statistics slot 45: the grid the records are laid out by (tools/raster_stats.py)
      reinterpret_cast<unsigned long long*>(p.big_queue)[(size_t)p.big_capacity * 8 + (p.late ? 64 : 0) + 45] = gridDim.x;
  }
#endif
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
  if (lane == 0 && kept) atomicAdd(p.tri_counter, (unsigned long long)kept);
}

// ---- clipping of the triangles the plain rules drop (specification: oracle/oxc_oracle.c raster_triangle_clipped) ----
// Sutherland-Hodgman in clip space against near (w - z), left (w + x), right (w - x), bottom (w + y), top (w - y); cut points
// evaluated from the inside vertex to the outside vertex with the canonical f32 operation order; the fan (P0, Pi, Pi+1) is
// set up with the plain rules.  Pieces are usually large (geometry around the camera): they go to the chunk queue of
// k_raster_big (inline when the queue is full).
OXC_DI void clip_and_draw(const TriParams& p, float4 c0, float4 c1, float4 c2, uint32_t data, float fW, float fH) {
  float4 poly[2][12];
  int cur;
  const int n = clip_polygon(c0, c1, c2, poly, cur);
  for (int i = 1; i + 1 < n; i++) {
    TriSetup s;
    if (tri_setup(to_screen(poly[cur][0], fW, fH), to_screen(poly[cur][i], fW, fH), to_screen(poly[cur][i + 1], fW, fH), p.width, p.height, s) != TRI_DRAW)
      continue;
    const int bw = s.px1 - s.px0 + 1, bh = s.py1 - s.py0 + 1;
    if (bw * bh > RASTER_BIG_PIXELS && p.big_queue && big_push(p, s, data)) continue; // spread over the GPU by k_raster_big
    s.narrow = false; // pieces may be large: 64-bit edge functions
    raster_small(s, data, p.visbuf, p.width);
  }
}

// The triangle behind a vis data word as k_raster_visbuffer sees it: the three clip-space corners recomputed with the canonical
// operation order (bit-identical to the ones the raster saw), the same near-plane, backface and malformed-index tests and the
// same set-up.  Returns the set-up's TRI_* result, or -1 for a triangle the raster culls or never reaches.
OXC_DI int rebuild_triangle(const TriParams& p, uint32_t data, uint32_t id_base, float4 (&c)[3], TriSetup& s) {
  const uint32_t gid = data >> p.prim_bits, t = data & ((1u << p.prim_bits) - 1u);
  const uint2 mi = __ldg(reinterpret_cast<const uint2*>(p.meshlet_instances) + (gid - id_base));
  const InstGeom* g = p.geom + mi.x;
  const InstCull* ic = p.inst + mi.x;
  const uint4 m = __ldg(reinterpret_cast<const uint4*>(g->meshlets + mi.y));
  if (t >= min(m.w, (uint32_t)OXC_MESHLET_MAX_PRIMITIVES)) return -1;
  const float4 r0 = __ldg(&ic->mvp_row[0]), r1 = __ldg(&ic->mvp_row[1]), r2 = __ldg(&ic->mvp_row[2]), r3 = __ldg(&ic->mvp_row[3]);
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const uint32_t li = micro_index(g->local_triangle_indices, m.y + t * 3u + k);
    if (li >= min(m.z, (uint32_t)OXC_MESHLET_MAX_VERTICES)) return -1;
    const uint32_t vi = __ldg(&g->indirect_vertex_indices[m.x + li]);
    const uint2 q = __ldg(&g->vertex_positions[vi]);
    const float x = dequantize_half_hw(q.x & 0xFFFFu), y = dequantize_half_hw(q.x >> 16), z = dequantize_half_hw(q.y & 0xFFFFu);
    c[k] = make_float4(row_dot_p1(r0, x, y, z), row_dot_p1(r1, x, y, z), row_dot_p1(r2, x, y, z), row_dot_p1(r3, x, y, z));
  }
  if (!(c[0].z >= 0.0f && c[1].z >= 0.0f && c[2].z >= 0.0f) || triangle_backface(c[0], c[1], c[2])) return -1;
  return tri_setup(to_screen(c[0], p.f_width, p.f_height), to_screen(c[1], p.f_width, p.f_height), to_screen(c[2], p.f_width, p.f_height),
                   p.width, p.height, s);
}

// One deferred triangle, drawn by the whole warp (every lane passes the same data word): clipped by lane 0 if a vertex is
// invalid; otherwise a box over RASTER_BIG_PIXELS goes to the chunk queue of k_raster_big, and a smaller box (64-bit edge
// functions), or one the full chunk queue cannot take, is covered in 8x4-pixel tiles right here.
OXC_DI void draw_deferred(const TriParams& p, uint32_t data, uint32_t id_base, uint32_t lane) {
  float4 c[3];
  TriSetup s;
  const int why = rebuild_triangle(p, data, id_base, c, s);
  if (why == TRI_INVALID_VERTEX) {
    if (lane == 0) clip_and_draw(p, c[0], c[1], c[2], data, p.f_width, p.f_height);
    return;
  }
  if (why != TRI_DRAW) return;
  if ((s.px1 - s.px0 + 1) * (s.py1 - s.py0 + 1) > RASTER_BIG_PIXELS && big_push_warp(p, s, data, lane)) return;
  raster_tiles(p, s, data, lane);
}

// One warp per entry of the deferred queue k_raster_visbuffer filled.  Runs after every k_raster_visbuffer and before
// k_raster_big.  When the queue overflowed, the warps then walk the pass's survivors again and draw (or clip) every triangle a
// lane would not draw itself; the queued ones are drawn twice, which the packed max
// leaves unchanged.
__global__ void __launch_bounds__(256) k_raster_deferred(const __grid_constant__ TriParams p) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp0 = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), warps = gridDim.x * (blockDim.x >> 5);
  const uint32_t pushed = *p.deferred_counter;
  const uint32_t n = min(pushed, p.deferred_capacity);
  const uint32_t id_base = p.id_base ? __ldg(p.id_base) : 0u;
  for (uint32_t e = warp0; e < n; e += warps) draw_deferred(p, p.deferred_queue[e], id_base, lane);
  if (pushed <= p.deferred_capacity) return;
  const uint32_t first = p.late ? p.vis->early_visible_meshlet_instances : 0u;
  const uint32_t count = p.tri_cmd->x;
  for (uint32_t g = warp0; g < count; g += warps) {
    const uint32_t gid = __ldg(&p.visible_indices[first + g]);
    for (uint32_t t = lane; t < OXC_MESHLET_MAX_PRIMITIVES; t += 32) {
      const uint32_t data = (gid << p.prim_bits) | t;
      float4 c[3];
      TriSetup s;
      const int why = rebuild_triangle(p, data, id_base, c, s);
      const bool deferred = why == TRI_INVALID_VERTEX || (why == TRI_DRAW && !lane_draws(s));
      for (uint32_t m = __ballot_sync(0xffffffffu, deferred); m; m &= m - 1)
        draw_deferred(p, __shfl_sync(0xffffffffu, data, __ffs(m) - 1), id_base, lane);
    }
  }
}

// ---- stand-alone clip pass (kept for hosts that drive the plain raster themselves): walks every survivor again and clips
//      the triangles the plain rules drop.  oxc_raster_visbuffer no longer needs it — it queues those triangles itself. ----
__global__ void __launch_bounds__(TRI_THREADS) k_raster_clip_pass(const __grid_constant__ TriParams p) {
  __shared__ float4 clip_all[TRI_WARPS][OXC_MESHLET_MAX_VERTICES];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t first = p.late ? p.vis->early_visible_meshlet_instances : 0u;
  const uint32_t count = p.tri_cmd->x;
  const uint32_t id_base = p.id_base ? __ldg(p.id_base) : 0u;
  const float fW = (float)p.width, fH = (float)p.height;
  float4* clip_s = clip_all[warp];
  const uint32_t n_tiles = (count + TRI_WARPS - 1) / TRI_WARPS;
  for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const uint32_t g = tile * TRI_WARPS + warp;
    if (g < count) {
      const MeshletWork w = load_meshlet(p, first + g, id_base, clip_s, lane);
      for (uint32_t t = lane; t < w.tri_count; t += 32) {
        float4 c0, c1, c2;
        if (!triangle_passes(w, t, clip_s, c0, c1, c2)) continue;
        if (to_screen(c0, fW, fH).fx != INT_MIN && to_screen(c1, fW, fH).fx != INT_MIN && to_screen(c2, fW, fH).fx != INT_MIN)
          continue; // drawn by k_raster_visbuffer
        clip_and_draw(p, c0, c1, c2, (w.data_id << p.prim_bits) | t, fW, fH);
      }
    }
    __syncwarp(); // clip_s reuse
  }
}

// visbuffer_clear.slang:20-28 on the packed image: depth 0 | data ~0u
__global__ void k_clear_visbuffer(unsigned long long* vis, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    vis[i] = (unsigned long long)OXC_VIS_CLEAR;
}

// clear + external depth in one pass: max(clear, asuint(depth)<<32 | ~0u) == asuint(depth)<<32 | ~0u for every depth bit
// pattern (the clear value is the smallest word of that form), so the merge after a clear is an unconditional store
__global__ void k_clear_visbuffer_depth(unsigned long long* vis, const float* depth, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    vis[i] = ((unsigned long long)__float_as_uint(__ldg(&depth[i])) << 32) | OXC_VIS_CLEAR;
}

// occluder / external depth merge: vis = max(vis, asuint(depth)<<32 | ~0u)
__global__ void k_merge_depth(unsigned long long* vis, const float* depth, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned long long v = ((unsigned long long)__float_as_uint(depth[i]) << 32) | OXC_VIS_CLEAR;
    if (v > vis[i]) vis[i] = v;
  }
}

// visbuffer.slang:67-70
__global__ void k_resolve_visbuffer(const unsigned long long* vis, uint32_t* vis32, float* depth, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const unsigned long long v = vis[i];
    if (vis32) vis32[i] = (uint32_t)(v & 0xFFFFFFFFull);
    if (depth) depth[i] = __uint_as_float((uint32_t)(v >> 32));
  }
}

} // namespace oxc
