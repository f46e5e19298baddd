// kernels_alpha.cuh — alpha-tested discard of the vis-buffer encode (visbuffer_encode.slang:54-66) for the software raster.
//   k_partition_alpha   splits the pass's survivors by material: meshlets whose material has no albedo image keep the tuned
//                       raster kernel (k_raster_visbuffer, untouched), the others go to k_raster_alpha.
//   k_raster_alpha      one warp per alpha-tested meshlet: same vertex transform, triangle cull, snapping, coverage, depth and
//                       packed max as the plain raster (oxc_raster_core.cuh), plus the per-fragment test of oxc_alpha.cuh;
//                       triangles the plain rules drop are clipped in place, uv carried through the cuts.
// Specification / oracle: orc_raster_visbuffer_alpha (oracle/oxc_oracle.c).  Alpha-tested geometry is a minority of a scene
// (foliage, fences): this kernel favours being small and obviously equal to the specification over the last microsecond.
#pragma once
#include "kernels_tri.cuh"
#include "oxc_alpha.cuh"

namespace oxc {

struct AlphaParams {
  const OxcMeshInstance* mesh_instances;
  const AlphaMaterial* materials; // [material_count]
  uint32_t material_count;
  // this pass's survivors (as TriParams) and the two lists they are split into
  uint32_t* opaque_list;
  uint32_t* masked_list;
  OxcDispatchIndirectCommand* opaque_cmd; // .x = entries of opaque_list (zeroed before the launch)
  OxcDispatchIndirectCommand* masked_cmd;
  uint32_t* overdraw;                     // k_raster_alpha<true>: the W x H fragment counter (RENDER_OVERDRAW)
  uint32_t count_from_visibility;         // k_raster_alpha<true> after the frame: the pass's count from the visibility record
};

OXC_DI bool alpha_material_of(const AlphaParams& a, const TriParams& p, uint32_t gid, uint32_t id_base, uint32_t& mat) {
  const uint2 mi = __ldg(reinterpret_cast<const uint2*>(p.meshlet_instances) + (gid - id_base));
  mat = __ldg(&a.mesh_instances[mi.x].material_index);
  if (mat >= a.material_count) {
    atomicOr(p.status, (uint32_t)OXC_STATUS_BAD_MATERIAL);
    return false;
  }
  return a.materials[mat].texels != nullptr;
}

__global__ void __launch_bounds__(256) k_partition_alpha(const __grid_constant__ TriParams p, const __grid_constant__ AlphaParams a) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t first = p.late ? p.vis->early_visible_meshlet_instances : 0u; // cull_triangles.slang:34-37
  const uint32_t count = p.tri_cmd->x;
  const uint32_t id_base = p.id_base ? __ldg(p.id_base) : 0u;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < count; base += stride) { // warp-uniform trip count
    const uint32_t i = base + lane;
    uint32_t gid = 0, mat = 0;
    bool valid = i < count, masked = false;
    if (valid) {
      gid = __ldg(&p.visible_indices[first + i]);
      masked = alpha_material_of(a, p, gid, id_base, mat);
    }
    const uint32_t bm = __ballot_sync(0xffffffffu, valid && masked), bo = __ballot_sync(0xffffffffu, valid && !masked);
    uint32_t sm = 0, so = 0;
    if (lane == 0) {
      if (bm) sm = atomicAdd(&a.masked_cmd->x, (uint32_t)__popc(bm));
      if (bo) so = atomicAdd(&a.opaque_cmd->x, (uint32_t)__popc(bo));
    }
    sm = __shfl_sync(0xffffffffu, sm, 0);
    so = __shfl_sync(0xffffffffu, so, 0);
    const uint32_t below = (1u << lane) - 1u;
    if (valid && masked) a.masked_list[sm + __popc(bm & below)] = gid;
    if (valid && !masked) a.opaque_list[so + __popc(bo & below)] = gid;
  }
}

// shade one sample: coverage + depth exactly as shade_pixel (oxc_raster_core.cuh), then the alpha test, then the packed max —
// or, OVERDRAW, the fragment counter of the encode pass (visbuffer_encode.slang:68-70: the shader's atomic comes after the discard
// and before any depth comparison)
template <bool OVERDRAW>
OXC_DI void shade_pixel_alpha(const TriSetup& s, const AlphaMaterial& m, const AlphaTri& t, int px, int py, uint32_t data,
                              unsigned long long* vis, uint32_t* overdraw, uint32_t W) {
  const int sx = px * 256 + 128, sy = py * 256 + 128;
  const long long e0 = orient2d(s.bx, s.by, s.cx, s.cy, sx, sy), e1 = orient2d(s.cx, s.cy, s.ax, s.ay, sx, sy),
                  e2 = orient2d(s.ax, s.ay, s.bx, s.by, sx, sy);
  if ((e0 - (s.bias & 1)) < 0 || (e1 - ((s.bias >> 1) & 1)) < 0 || (e2 - ((s.bias >> 2) & 1)) < 0) return;
  const float zz = fa(fa(s.za, fm((float)e1, s.dzb)), fm((float)e2, s.dzc));
  if (!(zz >= 0.0f && zz <= 1.0f)) return;
  if (m.texels) {  // discard (visbuffer_encode.slang:62-64); edge-function increments per pixel as in raster_small (oxc_raster_core.cuh)
    const long long ex[3] = {-(long long)(s.cy - s.by) * 256, -(long long)(s.ay - s.cy) * 256, -(long long)(s.by - s.ay) * 256};
    const long long ey[3] = {(long long)(s.cx - s.bx) * 256, (long long)(s.ax - s.cx) * 256, (long long)(s.bx - s.ax) * 256};
    if (!alpha_keep(m, t, px, py, e0, e1, e2, ex, ey)) return;
  }
  if (OVERDRAW) {
    atomicAdd(overdraw + (size_t)py * W + px, 1u);
    return;
  }
  uint32_t zb = __float_as_uint(zz);
  zb = zb == 0x80000000u ? 0u : zb;
  atomicMax(vis + (size_t)py * W + px, ((unsigned long long)zb << 32) | data);
}

template <bool OVERDRAW>
OXC_DI void raster_box_alpha(const TriSetup& s, const AlphaMaterial& m, const AlphaTri& t, uint32_t data, unsigned long long* vis,
                             uint32_t* overdraw, uint32_t W) {
  for (int py = s.py0; py <= s.py1; py++)
    for (int px = s.px0; px <= s.px1; px++) shade_pixel_alpha<OVERDRAW>(s, m, t, px, py, data, vis, overdraw, W);
}

constexpr int ALPHA_THREADS = 128, ALPHA_WARPS = ALPHA_THREADS / 32;
// bbox area above which the whole warp rasterises the triangle together.  Kept at 32 when the vis-buffer raster's threshold
// rose to 128: every pixel here also samples the alpha texture, and this kernel has not been timed on H100.
constexpr int ALPHA_BIG_PIXELS = 32;

// one triangle's set-up handed from its lane to the whole warp (triangles of more than ALPHA_BIG_PIXELS pixels)
struct AlphaBigRecord {
  TriSetup s;
  AlphaTri t;
  uint32_t data;
};

// OVERDRAW = false: the alpha-tested meshlets of the split (a.masked_list).  OVERDRAW = true: EVERY survivor of the pass (opaque
// materials skip the test; a.materials may be null), fragments counted into a.overdraw instead of drawn.
template <bool OVERDRAW>
__global__ void __launch_bounds__(ALPHA_THREADS) k_raster_alpha(const __grid_constant__ TriParams p, const __grid_constant__ AlphaParams a) {
  __shared__ float4 clip_all[ALPHA_WARPS][OXC_MESHLET_MAX_VERTICES];
  __shared__ float2 uv_all[ALPHA_WARPS][OXC_MESHLET_MAX_VERTICES];
  __shared__ AlphaBigRecord big_all[ALPHA_WARPS];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t first = OVERDRAW ? (p.late ? p.vis->early_visible_meshlet_instances : 0u) : 0u; // cull_triangles.slang:34-37
  // the dispatch command holds the count of the pass that ran LAST; a counter pass issued after the frame takes it from the
  // visibility record instead (early [0, E), late [E, E + L): cull_meshlets_hiz.slang:70-76)
  const uint32_t count = !OVERDRAW ? a.masked_cmd->x
                         : !a.count_from_visibility ? p.tri_cmd->x
                         : (p.late ? p.vis->late_visible_meshlet_instances : p.vis->early_visible_meshlet_instances);
  const uint32_t id_base = p.id_base ? __ldg(p.id_base) : 0u;
  float4* clip_s = clip_all[warp];
  float2* uv_s = uv_all[warp];
  AlphaBigRecord* big_s = &big_all[warp];
  uint32_t kept = 0;
  for (uint32_t g = blockIdx.x * ALPHA_WARPS + warp; g < count; g += gridDim.x * ALPHA_WARPS) {
    // ---- the meshlet: pointer chase, vertices -> clip space (visbuffer_encode.slang:27-38), uv (scene.slang:355-361) ----
    const uint32_t gid = OVERDRAW ? __ldg(&p.visible_indices[first + g]) : a.masked_list[g];
    const uint2 mi = __ldg(reinterpret_cast<const uint2*>(p.meshlet_instances) + (gid - id_base));
    const InstGeom* gm = p.geom + mi.x;
    const InstCull* ic = p.inst + mi.x;
    AlphaMaterial m;
    if (OVERDRAW) { // any material: outside the table or without an image = opaque
      const uint32_t mat = __ldg(&a.mesh_instances[mi.x].material_index);
      m.texels = nullptr;
      if (a.materials && mat < a.material_count) m = a.materials[mat];
    } else {
      m = a.materials[__ldg(&a.mesh_instances[mi.x].material_index)]; // in range and with an image: k_partition_alpha checked it
    }
    const uint4 ml = __ldg(reinterpret_cast<const uint4*>(gm->meshlets + mi.y));
    const uint32_t vertex_count = min(ml.z, (uint32_t)OXC_MESHLET_MAX_VERTICES), tri_count = min(ml.w, (uint32_t)OXC_MESHLET_MAX_PRIMITIVES);
    const float4 r0 = __ldg(&ic->mvp_row[0]), r1 = __ldg(&ic->mvp_row[1]), r2 = __ldg(&ic->mvp_row[2]), r3 = __ldg(&ic->mvp_row[3]);
    const uint32_t* vidx = gm->indirect_vertex_indices + ml.x;
    const uint32_t* tcs = gm->texture_coords;
    for (uint32_t v = lane; v < vertex_count; v += 32) {
      const uint32_t vi = __ldg(&vidx[v]);
      const uint2 q = __ldg(&gm->vertex_positions[vi]);
      const float x = dequantize_half(q.x & 0xFFFFu), y = dequantize_half(q.x >> 16), z = dequantize_half(q.y & 0xFFFFu);
      clip_s[v] = make_float4(row_dot_p1(r0, x, y, z), row_dot_p1(r1, x, y, z), row_dot_p1(r2, x, y, z), row_dot_p1(r3, x, y, z));
      float2 uv = make_float2(0.f, 0.f);
      if (tcs) { const uint32_t t = __ldg(&tcs[vi]); uv = make_float2(dequantize_half(t & 0xFFFFu), dequantize_half(t >> 16)); }
      uv_s[v] = uv;
    }
    __syncwarp();
    const uint32_t rounds = (tri_count + 31u) >> 5;
    for (uint32_t k = 0; k < rounds; k++) {
      const uint32_t t = lane + 32u * k;
      const uint32_t data = (gid << p.prim_bits) | t;
      TriSetup s;
      AlphaTri at;
      bool big = false;
      if (t < tri_count) {
        const uint32_t base = ml.y + t * 3u;
        const uint32_t i0 = micro_index(gm->local_triangle_indices, base + 0u), i1 = micro_index(gm->local_triangle_indices, base + 1u),
                       i2 = micro_index(gm->local_triangle_indices, base + 2u);
        if (max(i0, max(i1, i2)) < vertex_count) {
          const float4 c0 = clip_s[i0], c1 = clip_s[i1], c2 = clip_s[i2];
          if (c0.z >= 0.0f && c1.z >= 0.0f && c2.z >= 0.0f && !triangle_backface(c0, c1, c2)) { // cull_triangles.slang:68-69
            kept++;
            const float2 t0 = uv_s[i0], t1 = uv_s[i1], t2 = uv_s[i2];
            alpha_tri_setup(c0, c1, c2, t0.x, t0.y, t1.x, t1.y, t2.x, t2.y, at);
            const int why = tri_setup(to_screen(c0, p.f_width, p.f_height), to_screen(c1, p.f_width, p.f_height),
                                      to_screen(c2, p.f_width, p.f_height), p.width, p.height, s);
            if (why == TRI_DRAW) {
              big = (s.px1 - s.px0 + 1) * (s.py1 - s.py0 + 1) > ALPHA_BIG_PIXELS;
              if (!big) raster_box_alpha<OVERDRAW>(s, m, at, data, p.visbuf, a.overdraw, p.width);
            } else if (why == TRI_INVALID_VERTEX) { // a vertex at w <= 0 / beyond the snap range: clipped like the plain raster does,
              ClipVertUV poly[2][12];                // with uv carried through the cuts (alpha spec step 3)
              int cur;
              const ClipVertUV a0 = {c0, t0.x, t0.y}, a1 = {c1, t1.x, t1.y}, a2 = {c2, t2.x, t2.y};
              const int n = clip_polygon_uv(a0, a1, a2, poly, cur);
              for (int i = 1; i + 1 < n; i++) {
                const ClipVertUV q0 = poly[cur][0], q1 = poly[cur][i], q2 = poly[cur][i + 1];
                TriSetup ps;
                if (tri_setup(to_screen(q0.c, p.f_width, p.f_height), to_screen(q1.c, p.f_width, p.f_height),
                              to_screen(q2.c, p.f_width, p.f_height), p.width, p.height, ps) != TRI_DRAW)
                  continue;
                AlphaTri pt;
                alpha_tri_setup(q0.c, q1.c, q2.c, q0.u, q0.v, q1.u, q1.v, q2.u, q2.v, pt);
                raster_box_alpha<OVERDRAW>(ps, m, pt, data, p.visbuf, a.overdraw, p.width);
              }
            }
          }
        } // else: malformed meshlet, the triangle is skipped like in the plain raster
      }
      // triangles above ALPHA_BIG_PIXELS pixels: the whole warp covers the bounding box in 8x4-pixel tiles
      uint32_t big_mask = __ballot_sync(0xffffffffu, big);
      while (big_mask) {
        const uint32_t src = (uint32_t)__ffs(big_mask) - 1u;
        big_mask &= big_mask - 1u;
        if (lane == src) { big_s->s = s; big_s->t = at; big_s->data = data; }
        __syncwarp();
        const AlphaBigRecord b = *big_s;
        __syncwarp();
        const int lx = lane & 7, ly = lane >> 3;
        for (int ty = b.s.py0; ty <= b.s.py1; ty += 4)
          for (int tx = b.s.px0; tx <= b.s.px1; tx += 8) {
            const int px = tx + lx, py = ty + ly;
            if (px <= b.s.px1 && py <= b.s.py1) shade_pixel_alpha<OVERDRAW>(b.s, m, b.t, px, py, b.data, p.visbuf, a.overdraw, p.width);
          }
      }
    }
    __syncwarp(); // clip_s / uv_s reuse
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
  if (!OVERDRAW && lane == 0 && kept) atomicAdd(p.tri_counter, (unsigned long long)kept); // the counter pass draws nothing
}

} // namespace oxc
