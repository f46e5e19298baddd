// kernels_decode.cuh — consumers / producers either side of the cull + raster path (SURVEY §8f):
//   k_decode_visbuffer   passes/visbuffer_decode.slang:42-183, geometry part: per-pixel triangle re-fetch, analytic
//                        barycentrics with screen-space derivatives, interpolated uv (+ gradients) and the geometric
//                        world normal (oct encoded).
//   k_decode_gbuffer     the same pass with its material half (:117-183, oxc_gbuffer.cuh): albedo, normal-mapped normal,
//                        emissive, metallic / roughness / occlusion.
//   k_hpb_fused / k_hpb_level   passes/rmvsm_downsample_hpb.slang:15-33 (Shadowmaps.cpp:331-366): page table ->
//                        hierarchical page bitmap that k_cull_meshlets_hpb samples.
// Arithmetic is the canonical binary32 order of oracle/oxc_oracle.c::orc_decode_visbuffer (bit-exact).
#pragma once
#include "oxc_exact.cuh"
#include "oxc_gbuffer.cuh"     // GBufferPixel, vec3_to_oct and the material evaluation of k_decode_gbuffer
#include "oxc_vsm_resolve.cuh" // vsm_unproject: shared with the shadow resolve

namespace oxc {

struct DecodeParams {
  const unsigned long long* vis64; // packed depth|data image (ours), or
  const uint32_t* vis32;           // the reference's R32UI attachment
  const OxcMeshletInstance* meshlet_instances;
  const OxcMeshletInstanceVisibility* vis;
  const InstCull* inst;
  const InstGeom* geom;
  const uint32_t* id_base; // may be null
  float4* lambda;
  float4* ddx;
  float4* ddy;
  float4* uv_normal;
  float4* uv_grad;
  float4 pv_row[4];
  float res_x, res_y;
  uint32_t width, height;
  uint32_t prim_bits; // 8 (visbuffer.slang:9-14) or 6 (OxcCreateInfo::wide_ids)
};

// scene.slang:486-489 decode_normal
OXC_DI void decode_normal(uint32_t packed, float& x, float& y, float& z) {
  const int p = (int)packed;
  x = fs(fd((float)((p >> 20) & 1023), 511.0f), 1.0f);
  y = fs(fd((float)((p >> 10) & 1023), 511.0f), 1.0f);
  z = fs(fd((float)(p & 1023), 511.0f), 1.0f);
}

constexpr int DECODE_TX = 32, DECODE_TY = 8; // one CTA = a 32x8 pixel tile (a triangle's pixels share L1 lines)

// The geometry half of the decode for pixel (x, y), k_decode_visbuffer's arithmetic for k_decode_gbuffer: texel -> triangle, world
// positions, analytic barycentrics with their derivatives, uv with its gradients and the normalized world normal.  Returns the
// status of the lambda plane (0 discarded, 1 decoded, 2 vertex index out of range); L / DX / DY / UN.xy / UG as the planes hold them,
// g (world positions, normal) and *mesh_instance for the material evaluation.  Zero outputs unless decoded.
OXC_DI uint32_t decode_geometry(const DecodeParams& p, uint32_t x, uint32_t y, float4& L, float4& DX, float4& DY, float4& UN, float4& UG,
                                GBufferPixel& g, uint32_t* mesh_instance) {
  const size_t pix = (size_t)y * p.width + x;
  L = make_float4(0.f, 0.f, 0.f, 0.f); DX = L; DY = L; UN = L; UG = L;
  const uint32_t texel = p.vis64 ? (uint32_t)(__ldg(&p.vis64[pix]) & 0xFFFFFFFFull) : __ldg(&p.vis32[pix]); // :96
  const uint32_t gid = texel >> p.prim_bits;                                                                // visbuffer.slang:34
  const uint32_t tri = texel & ((1u << p.prim_bits) - 1u);
  const uint32_t id_base = p.id_base ? __ldg(p.id_base) : 0u;
  const uint32_t mii = gid - id_base;
  const bool discard = texel == 0xFFFFFFFFu || gid == (0xFFFFFFFFu >> p.prim_bits) - 1u /* terrain sentinel TERRAIN_INSTANCE_ID in either packing, visbuffer.slang:16-20 */ || gid < id_base ||
                       mii >= __ldg(&p.vis->total_visible_meshlet_instances); // :97-99 (+ range guard)
  if (discard) return 0u;
  const uint2 mi = __ldg(reinterpret_cast<const uint2*>(p.meshlet_instances) + mii); // :103
  *mesh_instance = mi.x;
  const InstGeom* gm = p.geom + mi.x;                                                // :104-108 (resolved by cull_meshes)
  const InstCull* ic = p.inst + mi.x;
  const uint4 g0 = __ldg(reinterpret_cast<const uint4*>(gm)), g1 = __ldg(reinterpret_cast<const uint4*>(gm) + 1),
              g2 = __ldg(reinterpret_cast<const uint4*>(gm) + 2), g3 = __ldg(reinterpret_cast<const uint4*>(gm) + 3);
  const OxcMeshlet* meshlets = reinterpret_cast<const OxcMeshlet*>(((uint64_t)g0.y << 32) | g0.x);
  const uint32_t* micro = reinterpret_cast<const uint32_t*>(((uint64_t)g0.w << 32) | g0.z);
  const uint32_t* vidx = reinterpret_cast<const uint32_t*>(((uint64_t)g1.y << 32) | g1.x);
  const uint2* pos = reinterpret_cast<const uint2*>(((uint64_t)g1.w << 32) | g1.z);
  const uint32_t* nrm = reinterpret_cast<const uint32_t*>(((uint64_t)g2.y << 32) | g2.x);
  const uint32_t* tcs = reinterpret_cast<const uint32_t*>(((uint64_t)g2.w << 32) | g2.z);
  const uint32_t vertex_count = g3.y;
  const uint4 m = __ldg(reinterpret_cast<const uint4*>(meshlets + mi.y)); // :109
  const uint32_t base = m.y + tri * 3u;                                   // scene.slang:366
  uint32_t idx[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const uint32_t bo = base + (uint32_t)c;
    const uint32_t local = (__ldg(&micro[bo >> 2]) >> ((bo & 3u) * 8u)) & 0xFFu;
    idx[c] = __ldg(&vidx[m.x + local]);
  }
  L.w = 2.0f;
  if (idx[0] > vertex_count - 1u || idx[1] > vertex_count - 1u || idx[2] > vertex_count - 1u) return 2u; // :115-117
  L.w = 1.0f;
  const float4 w0 = __ldg(&ic->world_row[0]), w1 = __ldg(&ic->world_row[1]), w2 = __ldg(&ic->world_row[2]);
  float inv_w[3], nx[3], ny[3], nrx[3], nry[3], nrz[3], tu[3], tv[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const uint2 q = __ldg(&pos[idx[c]]);
    // hardware half decode: identical to the canonical one for all 65536 inputs up to NaN payloads (oxc_exact.cuh)
    const float px = dequantize_half_hw(q.x & 0xFFFFu), py = dequantize_half_hw(q.x >> 16), pz = dequantize_half_hw(q.y & 0xFFFFu);
    const float wx = row_dot_p1(w0, px, py, pz), wy = row_dot_p1(w1, px, py, pz), wz = row_dot_p1(w2, px, py, pz); // :121
    g.wp[c][0] = wx; g.wp[c][1] = wy; g.wp[c][2] = wz;
    const float cx = row_dot_p1(p.pv_row[0], wx, wy, wz), cy = row_dot_p1(p.pv_row[1], wx, wy, wz),
                cw = row_dot_p1(p.pv_row[3], wx, wy, wz); // :45-47
    inv_w[c] = fd(1.0f, cw);                               // :50
    nx[c] = fm(cx, inv_w[c]);                              // :51-53
    ny[c] = fm(cy, inv_w[c]);
    if (nrm) decode_normal(__ldg(&nrm[idx[c]]), nrx[c], nry[c], nrz[c]);
    else { nrx[c] = 0.f; nry[c] = 0.f; nrz[c] = 0.f; }
    if (tcs) { // scene.slang:390-399
      const uint32_t t = __ldg(&tcs[idx[c]]);
      tu[c] = dequantize_half_hw(t & 0xFFFFu); tv[c] = dequantize_half_hw(t >> 16);
    } else { tu[c] = 0.f; tv[c] = 0.f; }
  }
  // fullscreen.slang:11-17 + :122
  const float u = fd(fa((float)x, 0.5f), (float)p.width), v = fd(fa((float)y, 0.5f), (float)p.height);
  const float ndcx = fs(fm(u, 2.0f), 1.0f), ndcy = fs(fm(v, 2.0f), 1.0f);
  // compute_partial_derivatives :55-83
  const float ax = fs(nx[2], nx[1]), ay = fs(ny[2], ny[1]), bx = fs(nx[0], nx[1]), by = fs(ny[0], ny[1]);
  const float inv_det = fd(1.0f, fs(fm(ax, by), fm(ay, bx))); // :58
  float ddx[3], ddy[3], lam[3];
  ddx[0] = fm(fm(fs(ny[1], ny[2]), inv_det), inv_w[0]); // :60
  ddx[1] = fm(fm(fs(ny[2], ny[0]), inv_det), inv_w[1]);
  ddx[2] = fm(fm(fs(ny[0], ny[1]), inv_det), inv_w[2]);
  ddy[0] = fm(fm(fs(nx[2], nx[1]), inv_det), inv_w[0]); // :62
  ddy[1] = fm(fm(fs(nx[0], nx[2]), inv_det), inv_w[1]);
  ddy[2] = fm(fm(fs(nx[1], nx[0]), inv_det), inv_w[2]);
  float ddx_sum = fa(fa(ddx[0], ddx[1]), ddx[2]); // :63 (x * 1.0 is exact)
  float ddy_sum = fa(fa(ddy[0], ddy[1]), ddy[2]); // :64
  const float dvx = fs(ndcx, nx[0]), dvy = fs(ndcy, ny[0]);                            // :66
  const float interp_inv_w = fa(fa(inv_w[0], fm(dvx, ddx_sum)), fm(dvy, ddy_sum));     // :67
  const float interp_w = fd(1.0f, interp_inv_w);                                       // :68
  lam[0] = fm(interp_w, fa(fa(inv_w[0], fm(dvx, ddx[0])), fm(dvy, ddy[0])));           // :69-73
  lam[1] = fm(interp_w, fa(fm(dvx, ddx[1]), fm(dvy, ddy[1])));
  lam[2] = fm(interp_w, fa(fm(dvx, ddx[2]), fm(dvy, ddy[2])));
  const float torx = fd(2.0f, p.res_x), ntory = -fd(2.0f, p.res_y); // :74
#pragma unroll
  for (int c = 0; c < 3; c++) { ddx[c] = fm(ddx[c], torx); ddy[c] = fm(ddy[c], ntory); } // :75-76
  ddx_sum = fm(ddx_sum, torx); ddy_sum = fm(ddy_sum, ntory);                             // :77-78
  const float iddxw = fd(1.0f, fa(interp_inv_w, ddx_sum)), iddyw = fd(1.0f, fa(interp_inv_w, ddy_sum)); // :80-81
#pragma unroll
  for (int c = 0; c < 3; c++) { // :82-83
    ddx[c] = fs(fm(iddxw, fa(fm(lam[c], interp_inv_w), ddx[c])), lam[c]);
    ddy[c] = fs(fm(iddyw, fa(fm(lam[c], interp_inv_w), ddy[c])), lam[c]);
    g.ddx[c] = ddx[c]; g.ddy[c] = ddy[c];
  }
  L.x = lam[0]; L.y = lam[1]; L.z = lam[2];
  DX.x = ddx[0]; DX.y = ddx[1]; DX.z = ddx[2];
  DY.x = ddy[0]; DY.y = ddy[1]; DY.z = ddy[2];
  // gradient_of :33-40
  UN.x = fa(fa(fm(lam[0], tu[0]), fm(lam[1], tu[1])), fm(lam[2], tu[2]));
  UN.y = fa(fa(fm(lam[0], tv[0]), fm(lam[1], tv[1])), fm(lam[2], tv[2]));
  UG.x = fa(fa(fm(ddx[0], tu[0]), fm(ddx[1], tu[1])), fm(ddx[2], tu[2]));
  UG.y = fa(fa(fm(ddx[0], tv[0]), fm(ddx[1], tv[1])), fm(ddx[2], tv[2]));
  UG.z = fa(fa(fm(ddy[0], tu[0]), fm(ddy[1], tu[1])), fm(ddy[2], tu[2]));
  UG.w = fa(fa(fm(ddy[0], tv[0]), fm(ddy[1], tv[1])), fm(ddy[2], tv[2]));
  g.uv[0] = UN.x; g.uv[1] = UN.y; g.uv_ddx[0] = UG.x; g.uv_ddx[1] = UG.y; g.uv_ddy[0] = UG.z; g.uv_ddy[1] = UG.w;
  // :146-147 normalize(mul(lambda, to_world_normals(normals))); cross rows hoisted into InstCull::nrm
  const float4 r0 = __ldg(&ic->nrm[0]), r1 = __ldg(&ic->nrm[1]), r2 = __ldg(&ic->nrm[2]);
  float wnx[3], wny[3], wnz[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    wnx[c] = fa(fa(fm(r0.x, nrx[c]), fm(r1.x, nry[c])), fm(r2.x, nrz[c]));
    wny[c] = fa(fa(fm(r0.y, nrx[c]), fm(r1.y, nry[c])), fm(r2.y, nrz[c]));
    wnz[c] = fa(fa(fm(r0.z, nrx[c]), fm(r1.z, nry[c])), fm(r2.z, nrz[c]));
  }
  const float n0 = fa(fa(fm(lam[0], wnx[0]), fm(lam[1], wnx[1])), fm(lam[2], wnx[2]));
  const float n1 = fa(fa(fm(lam[0], wny[0]), fm(lam[1], wny[1])), fm(lam[2], wny[2]));
  const float n2 = fa(fa(fm(lam[0], wnz[0]), fm(lam[1], wnz[1])), fm(lam[2], wnz[2]));
  const float len = length3(n0, n1, n2);
  g.n[0] = fd(n0, len); g.n[1] = fd(n1, len); g.n[2] = fd(n2, len);
  return 1u;
}

// Written out rather than calling decode_geometry: the shared function changed this kernel's SASS (DESIGN §4.6).
__global__ void __launch_bounds__(DECODE_TX* DECODE_TY) k_decode_visbuffer(const __grid_constant__ DecodeParams p) {
  const uint32_t x = blockIdx.x * DECODE_TX + threadIdx.x, y = blockIdx.y * DECODE_TY + threadIdx.y;
  if (x >= p.width || y >= p.height) return;
  const size_t pix = (size_t)y * p.width + x;
  float4 L = make_float4(0.f, 0.f, 0.f, 0.f), DX = L, DY = L, UN = L, UG = L;
  const uint32_t texel = p.vis64 ? (uint32_t)(__ldg(&p.vis64[pix]) & 0xFFFFFFFFull) : __ldg(&p.vis32[pix]); // :96
  const uint32_t gid = texel >> p.prim_bits;                                                                // visbuffer.slang:34
  const uint32_t tri = texel & ((1u << p.prim_bits) - 1u);
  const uint32_t id_base = p.id_base ? __ldg(p.id_base) : 0u;
  const uint32_t mii = gid - id_base;
  const bool discard = texel == 0xFFFFFFFFu || gid == (0xFFFFFFFFu >> p.prim_bits) - 1u /* terrain sentinel TERRAIN_INSTANCE_ID in either packing, visbuffer.slang:16-20 */ || gid < id_base ||
                       mii >= __ldg(&p.vis->total_visible_meshlet_instances); // :97-99 (+ range guard)
  if (!discard) {
    const uint2 mi = __ldg(reinterpret_cast<const uint2*>(p.meshlet_instances) + mii); // :103
    const InstGeom* g = p.geom + mi.x;                                                 // :104-108 (resolved by cull_meshes)
    const InstCull* ic = p.inst + mi.x;
    const uint4 g0 = __ldg(reinterpret_cast<const uint4*>(g)), g1 = __ldg(reinterpret_cast<const uint4*>(g) + 1),
                g2 = __ldg(reinterpret_cast<const uint4*>(g) + 2), g3 = __ldg(reinterpret_cast<const uint4*>(g) + 3);
    const OxcMeshlet* meshlets = reinterpret_cast<const OxcMeshlet*>(((uint64_t)g0.y << 32) | g0.x);
    const uint32_t* micro = reinterpret_cast<const uint32_t*>(((uint64_t)g0.w << 32) | g0.z);
    const uint32_t* vidx = reinterpret_cast<const uint32_t*>(((uint64_t)g1.y << 32) | g1.x);
    const uint2* pos = reinterpret_cast<const uint2*>(((uint64_t)g1.w << 32) | g1.z);
    const uint32_t* nrm = reinterpret_cast<const uint32_t*>(((uint64_t)g2.y << 32) | g2.x);
    const uint32_t* tcs = reinterpret_cast<const uint32_t*>(((uint64_t)g2.w << 32) | g2.z);
    const uint32_t vertex_count = g3.y;
    const uint4 m = __ldg(reinterpret_cast<const uint4*>(meshlets + mi.y)); // :109
    const uint32_t base = m.y + tri * 3u;                                   // scene.slang:366
    uint32_t idx[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const uint32_t bo = base + (uint32_t)c;
      const uint32_t local = (__ldg(&micro[bo >> 2]) >> ((bo & 3u) * 8u)) & 0xFFu;
      idx[c] = __ldg(&vidx[m.x + local]);
    }
    L.w = 2.0f;
    if (!(idx[0] > vertex_count - 1u || idx[1] > vertex_count - 1u || idx[2] > vertex_count - 1u)) { // :115-117
      L.w = 1.0f;
      const float4 w0 = __ldg(&ic->world_row[0]), w1 = __ldg(&ic->world_row[1]), w2 = __ldg(&ic->world_row[2]);
      float inv_w[3], nx[3], ny[3], nrx[3], nry[3], nrz[3], tu[3], tv[3];
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const uint2 q = __ldg(&pos[idx[c]]);
        // hardware half decode: identical to the canonical one for all 65536 inputs up to NaN payloads (oxc_exact.cuh)
        const float px = dequantize_half_hw(q.x & 0xFFFFu), py = dequantize_half_hw(q.x >> 16), pz = dequantize_half_hw(q.y & 0xFFFFu);
        const float wx = row_dot_p1(w0, px, py, pz), wy = row_dot_p1(w1, px, py, pz), wz = row_dot_p1(w2, px, py, pz); // :121
        const float cx = row_dot_p1(p.pv_row[0], wx, wy, wz), cy = row_dot_p1(p.pv_row[1], wx, wy, wz),
                    cw = row_dot_p1(p.pv_row[3], wx, wy, wz); // :45-47
        inv_w[c] = fd(1.0f, cw);                               // :50
        nx[c] = fm(cx, inv_w[c]);                              // :51-53
        ny[c] = fm(cy, inv_w[c]);
        if (nrm) decode_normal(__ldg(&nrm[idx[c]]), nrx[c], nry[c], nrz[c]);
        else { nrx[c] = 0.f; nry[c] = 0.f; nrz[c] = 0.f; }
        if (tcs) { // scene.slang:390-399
          const uint32_t t = __ldg(&tcs[idx[c]]);
          tu[c] = dequantize_half_hw(t & 0xFFFFu); tv[c] = dequantize_half_hw(t >> 16);
        } else { tu[c] = 0.f; tv[c] = 0.f; }
      }
      // fullscreen.slang:11-17 + :122
      const float u = fd(fa((float)x, 0.5f), (float)p.width), v = fd(fa((float)y, 0.5f), (float)p.height);
      const float ndcx = fs(fm(u, 2.0f), 1.0f), ndcy = fs(fm(v, 2.0f), 1.0f);
      // compute_partial_derivatives :55-83
      const float ax = fs(nx[2], nx[1]), ay = fs(ny[2], ny[1]), bx = fs(nx[0], nx[1]), by = fs(ny[0], ny[1]);
      const float inv_det = fd(1.0f, fs(fm(ax, by), fm(ay, bx))); // :58
      float ddx[3], ddy[3], lam[3];
      ddx[0] = fm(fm(fs(ny[1], ny[2]), inv_det), inv_w[0]); // :60
      ddx[1] = fm(fm(fs(ny[2], ny[0]), inv_det), inv_w[1]);
      ddx[2] = fm(fm(fs(ny[0], ny[1]), inv_det), inv_w[2]);
      ddy[0] = fm(fm(fs(nx[2], nx[1]), inv_det), inv_w[0]); // :62
      ddy[1] = fm(fm(fs(nx[0], nx[2]), inv_det), inv_w[1]);
      ddy[2] = fm(fm(fs(nx[1], nx[0]), inv_det), inv_w[2]);
      float ddx_sum = fa(fa(ddx[0], ddx[1]), ddx[2]); // :63 (x * 1.0 is exact)
      float ddy_sum = fa(fa(ddy[0], ddy[1]), ddy[2]); // :64
      const float dvx = fs(ndcx, nx[0]), dvy = fs(ndcy, ny[0]);                            // :66
      const float interp_inv_w = fa(fa(inv_w[0], fm(dvx, ddx_sum)), fm(dvy, ddy_sum));     // :67
      const float interp_w = fd(1.0f, interp_inv_w);                                       // :68
      lam[0] = fm(interp_w, fa(fa(inv_w[0], fm(dvx, ddx[0])), fm(dvy, ddy[0])));           // :69-73
      lam[1] = fm(interp_w, fa(fm(dvx, ddx[1]), fm(dvy, ddy[1])));
      lam[2] = fm(interp_w, fa(fm(dvx, ddx[2]), fm(dvy, ddy[2])));
      const float torx = fd(2.0f, p.res_x), ntory = -fd(2.0f, p.res_y); // :74
#pragma unroll
      for (int c = 0; c < 3; c++) { ddx[c] = fm(ddx[c], torx); ddy[c] = fm(ddy[c], ntory); } // :75-76
      ddx_sum = fm(ddx_sum, torx); ddy_sum = fm(ddy_sum, ntory);                             // :77-78
      const float iddxw = fd(1.0f, fa(interp_inv_w, ddx_sum)), iddyw = fd(1.0f, fa(interp_inv_w, ddy_sum)); // :80-81
#pragma unroll
      for (int c = 0; c < 3; c++) { // :82-83
        ddx[c] = fs(fm(iddxw, fa(fm(lam[c], interp_inv_w), ddx[c])), lam[c]);
        ddy[c] = fs(fm(iddyw, fa(fm(lam[c], interp_inv_w), ddy[c])), lam[c]);
      }
      L.x = lam[0]; L.y = lam[1]; L.z = lam[2];
      DX.x = ddx[0]; DX.y = ddx[1]; DX.z = ddx[2];
      DY.x = ddy[0]; DY.y = ddy[1]; DY.z = ddy[2];
      // gradient_of :33-40
      UN.x = fa(fa(fm(lam[0], tu[0]), fm(lam[1], tu[1])), fm(lam[2], tu[2]));
      UN.y = fa(fa(fm(lam[0], tv[0]), fm(lam[1], tv[1])), fm(lam[2], tv[2]));
      UG.x = fa(fa(fm(ddx[0], tu[0]), fm(ddx[1], tu[1])), fm(ddx[2], tu[2]));
      UG.y = fa(fa(fm(ddx[0], tv[0]), fm(ddx[1], tv[1])), fm(ddx[2], tv[2]));
      UG.z = fa(fa(fm(ddy[0], tu[0]), fm(ddy[1], tu[1])), fm(ddy[2], tu[2]));
      UG.w = fa(fa(fm(ddy[0], tv[0]), fm(ddy[1], tv[1])), fm(ddy[2], tv[2]));
      // :146-147 normalize(mul(lambda, to_world_normals(normals))); cross rows hoisted into InstCull::nrm
      {
        const float4 r0 = __ldg(&ic->nrm[0]), r1 = __ldg(&ic->nrm[1]), r2 = __ldg(&ic->nrm[2]);
        float wnx[3], wny[3], wnz[3];
#pragma unroll
        for (int c = 0; c < 3; c++) {
          wnx[c] = fa(fa(fm(r0.x, nrx[c]), fm(r1.x, nry[c])), fm(r2.x, nrz[c]));
          wny[c] = fa(fa(fm(r0.y, nrx[c]), fm(r1.y, nry[c])), fm(r2.y, nrz[c]));
          wnz[c] = fa(fa(fm(r0.z, nrx[c]), fm(r1.z, nry[c])), fm(r2.z, nrz[c]));
        }
        const float n0 = fa(fa(fm(lam[0], wnx[0]), fm(lam[1], wnx[1])), fm(lam[2], wnx[2]));
        const float n1 = fa(fa(fm(lam[0], wny[0]), fm(lam[1], wny[1])), fm(lam[2], wny[2]));
        const float n2 = fa(fa(fm(lam[0], wnz[0]), fm(lam[1], wnz[1])), fm(lam[2], wnz[2]));
        const float len = length3(n0, n1, n2);
        const float vx = fd(n0, len), vy = fd(n1, len), vz = fd(n2, len);
        // common/encoding.slang:17-21 vec3_to_oct
        const float inv = fd(1.0f, fa(fa(fabsf(vx), fabsf(vy)), fabsf(vz)));
        const float ox = fm(vx, inv), oy = fm(vy, inv);
        if (vz <= 0.0f) {
          UN.z = fm(fs(1.0f, fabsf(oy)), ox >= 0.0f ? 1.0f : -1.0f);
          UN.w = fm(fs(1.0f, fabsf(ox)), oy >= 0.0f ? 1.0f : -1.0f);
        } else {
          UN.z = ox; UN.w = oy;
        }
      }
    }
  }
  if (p.lambda) p.lambda[pix] = L;
  if (p.ddx) p.ddx[pix] = DX;
  if (p.ddy) p.ddy[pix] = DY;
  if (p.uv_normal) p.uv_normal[pix] = UN;
  if (p.uv_grad) p.uv_grad[pix] = UG;
}

// ---- G-buffer decode (visbuffer_decode.slang:88-183): the geometry above, then the material evaluation of oxc_gbuffer.cuh ----
struct GBufferParams {
  DecodeParams d; // geometry inputs (its targets stay null)
  const OxcMeshInstance* mesh_instances;
  const GBufMaterial* materials;
  const GBufImage* images; // [material_count][GB_SLOTS]
  uint32_t material_count;
  uint32_t want;           // bit k: target k is written
  float cam[3];            // camera.position
  float4* albedo;
  float4* normal;
  float4* emissive;
  float4* mro;
  uint32_t* status;
};

__global__ void __launch_bounds__(DECODE_TX* DECODE_TY) k_decode_gbuffer(const __grid_constant__ GBufferParams p) {
  const uint32_t x = blockIdx.x * DECODE_TX + threadIdx.x, y = blockIdx.y * DECODE_TY + threadIdx.y;
  if (x >= p.d.width || y >= p.d.height) return;
  const size_t pix = (size_t)y * p.d.width + x;
  float4 L, DX, DY, UN, UG;
  GBufferPixel g;
  uint32_t mesh_instance = 0;
  const uint32_t st = decode_geometry(p.d, x, y, L, DX, DY, UN, UG, g, &mesh_instance);
  if (st == 0u) return; // discard: the targets keep their contents
  float4 albedo = make_float4(0.f, 0.f, 0.f, 0.f), normal = albedo, emissive = albedo, mro = albedo;
  if (st == 1u) {
    const uint32_t mat = __ldg(&p.mesh_instances[mesh_instance].material_index);
    if (mat < p.material_count)
      gbuffer_shade(ldg_struct(p.materials + mat), p.images + (size_t)mat * GB_SLOTS, g, p.cam[0], p.cam[1], p.cam[2], p.want, albedo, normal,
                    emissive, mro);
    else
      atomicOr(p.status, (uint32_t)OXC_STATUS_BAD_MATERIAL);
  }
  if (p.albedo) p.albedo[pix] = albedo;
  if (p.normal) p.normal[pix] = normal;
  if (p.emissive) p.emissive[pix] = emissive;
  if (p.mro) p.mro[pix] = mro;
}

// ---- hierarchical page bitmap (rmvsm_downsample_hpb.slang) ----
struct HpbBuildParams {
  const uint32_t* page_table; // layers x size x size (R32UI, VSMPageMetadata bits rmvsm.slang:16-28)
  uint8_t* hpb;               // level l at level_offset(l): layers x s_l x s_l bytes
  uint32_t size, layers, levels;
};

OXC_DI uint8_t hpb_cached(uint32_t page) { return (uint8_t)((page & 7u) == 7u); } // visible && backed && dirty (:24-26)

// One CTA per layer: level 0 from the page table, every further level out of shared memory (size <= 256).
__global__ void __launch_bounds__(1024) k_hpb_fused(const __grid_constant__ HpbBuildParams p) {
  extern __shared__ uint8_t lv[]; // ping: size^2, pong: (size/2)^2
  const uint32_t z = blockIdx.x, s0 = p.size;
  uint8_t* cur = lv;
  uint8_t* nxt = lv + (size_t)s0 * s0;
  const uint32_t* pt = p.page_table + (size_t)z * s0 * s0;
  uint8_t* out = p.hpb + (size_t)z * s0 * s0;
  for (uint32_t i = threadIdx.x; i < s0 * s0; i += blockDim.x) {
    const uint8_t c = hpb_cached(__ldg(&pt[i]));
    cur[i] = c;
    out[i] = c;
  }
  __syncthreads();
  size_t off = (size_t)p.layers * s0 * s0;
  uint32_t ps = s0;
  for (uint32_t l = 1; l < p.levels; l++) {
    const uint32_t s = max(1u, s0 >> l);
    uint8_t* dst = p.hpb + off + (size_t)z * s * s;
    for (uint32_t i = threadIdx.x; i < s * s; i += blockDim.x) {
      const uint32_t x = i % s, y = i / s, x0 = x * 2u, y0 = y * 2u;
      // :27-32; loads past the source extent return 0 (only reachable when the source side is 1)
      const uint8_t tl = cur[(size_t)y0 * ps + x0];
      const uint8_t tr = (y0 + 1u < ps) ? cur[(size_t)(y0 + 1u) * ps + x0] : 0;
      const uint8_t bl = (x0 + 1u < ps) ? cur[(size_t)y0 * ps + x0 + 1u] : 0;
      const uint8_t br = (x0 + 1u < ps && y0 + 1u < ps) ? cur[(size_t)(y0 + 1u) * ps + x0 + 1u] : 0;
      const uint8_t c = (uint8_t)((tl | tr | bl | br) == 1);
      nxt[i] = c;
      dst[i] = c;
    }
    __syncthreads();
    uint8_t* t = cur; cur = nxt; nxt = t;
    off += (size_t)p.layers * s * s;
    ps = s;
  }
}

// Generic per-level kernel for page tables too large for shared memory.
__global__ void k_hpb_level(const uint32_t* page_table, const uint8_t* src, uint8_t* dst, uint32_t ps, uint32_t s, uint32_t layers,
                            int first) {
  const size_t n = (size_t)layers * s * s;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (first) { dst[i] = hpb_cached(__ldg(&page_table[i])); continue; }
    const uint32_t x = (uint32_t)(i % s), y = (uint32_t)((i / s) % s), z = (uint32_t)(i / ((size_t)s * s));
    const uint8_t* sl = src + (size_t)z * ps * ps;
    const uint32_t x0 = x * 2u, y0 = y * 2u;
    const uint8_t tl = sl[(size_t)y0 * ps + x0];
    const uint8_t tr = (y0 + 1u < ps) ? sl[(size_t)(y0 + 1u) * ps + x0] : 0;
    const uint8_t bl = (x0 + 1u < ps) ? sl[(size_t)y0 * ps + x0 + 1u] : 0;
    const uint8_t br = (x0 + 1u < ps && y0 + 1u < ps) ? sl[(size_t)(y0 + 1u) * ps + x0 + 1u] : 0;
    dst[i] = (uint8_t)((tl | tr | bl | br) == 1);
  }
}

// ------------------------------------------------------------------------------------------------
// VSM page marking — passes/rmvsm_mark_visible_pages.slang:19-84 (+ rmvsm.slang:116-221).  One thread per depth pixel.
// Lanes of a warp that hit the same page table entry elect one of them for the atomic (the reference's scalarisation loop,
// :64-74, done with match.any): pixels are coherent, so a warp usually touches one or two pages.
// ------------------------------------------------------------------------------------------------
struct VsmMarkParams {
  float4 inv_pv_row[4];       // rows of Camera::inv_projection_view
  float inv_res_half[2];      // (1 / resolution) * 0.5
  float clipmap_row[10][4][4];// rows of every clipmap's projection_view_mat
  int page_offset[10][2];
  const float* depth;
  uint32_t* page_tables;
  uint32_t* page_occupancy;
  uint32_t* request_count;
  int* requests;
  uint32_t request_capacity;
  int width, height, size, clipmap_count;
  float texel_length, bias;
};

__global__ void __launch_bounds__(256) k_vsm_mark_visible_pages(const __grid_constant__ VsmMarkParams p) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  uint32_t address = 0xFFFFFFFFu; // page table entry this pixel marks (none)
  int wx = 0, wy = 0, ci_out = 0;
  if (x < p.width && y < p.height) {
    const float d = __ldg(&p.depth[(size_t)y * p.width + x]);
    if (d != 0.0f) {                                                                             // :43-45
      const float u = fd(fa((float)x, 0.5f), (float)p.width), v = fd(fa((float)y, 0.5f), (float)p.height); // :47
      float wxp, wyp, wzp;
      vsm_unproject(p, u, v, d, wxp, wyp, wzp);
      float ax, ay, az, bx, by, bz;                                                              // :156-186
      vsm_unproject(p, fs(u, p.inv_res_half[0]), fa(v, p.inv_res_half[1]), d, ax, ay, az);
      vsm_unproject(p, fa(u, p.inv_res_half[0]), fa(v, p.inv_res_half[1]), d, bx, by, bz);
      const float dx = fs(ax, bx), dy = fs(ay, by), dz = fs(az, bz);
      const float dist = fsq(fa(fa(fm(dx, dx), fm(dy, dy)), fm(dz, dz)));
      float level_f = canonical_log2(fd(dist, p.texel_length));
      level_f = level_f > 0.0f ? level_f : 0.0f;
      const float lf = ceilf(fa(p.bias, level_f));
      uint32_t ci = lf >= 4294967296.0f ? 0xFFFFFFFFu : (lf > 0.0f ? __float2uint_rz(lf) : 0u);
      ci = ci > (uint32_t)(p.clipmap_count - 1) ? (uint32_t)(p.clipmap_count - 1) : ci;
      const float(*cr)[4] = p.clipmap_row[ci];
      const float lx = fa(fa(fa(fm(cr[0][0], wxp), fm(cr[0][1], wyp)), fm(cr[0][2], wzp)), fm(cr[0][3], 1.0f));
      const float ly = fa(fa(fa(fm(cr[1][0], wxp), fm(cr[1][1], wyp)), fm(cr[1][2], wzp)), fm(cr[1][3], 1.0f));
      const float lw = fa(fa(fa(fm(cr[3][0], wxp), fm(cr[3][1], wyp)), fm(cr[3][2], wzp)), fm(cr[3][3], 1.0f));
      const float cu = fm(fa(fd(lx, lw), 1.0f), 0.5f), cv = fm(fa(fd(ly, lw), 1.0f), 0.5f);     // :214-221
      if (!(cu < 0.0f || cv < 0.0f || cu > 1.0f || cv > 1.0f)) {                                  // :200-203
        const float fsz = (float)p.size;
        const float fxv = floorf(fm(cu, fsz)), fyv = floorf(fm(cv, fsz));
        const int vx = !(fxv == fxv) ? 0 : (fxv >= 2147483648.0f ? INT_MAX : (fxv <= -2147483648.0f ? INT_MIN : (int)fxv));
        const int vy = !(fyv == fyv) ? 0 : (fyv >= 2147483648.0f ? INT_MAX : (fyv <= -2147483648.0f ? INT_MIN : (int)fyv));
        if (!(vx < 0 || vy < 0 || vx > p.size - 1 || vy > p.size - 1)) {                          // :129-133
          const float fox = (float)(vx + p.page_offset[ci][0]), foy = (float)(vy + p.page_offset[ci][1]);
          wx = (int)fs(fox, fm(fsz, floorf(fd(fox, fsz))));                                       // com::mod, common/math.slang:99-101
          wy = (int)fs(foy, fm(fsz, floorf(fd(foy, fsz))));
          if (!(wx < 0 || wy < 0 || wx > p.size - 1 || wy > p.size - 1)) {
            address = ((uint32_t)ci * p.size + (uint32_t)wy) * p.size + (uint32_t)wx;
            ci_out = (int)ci;
          }
        }
      }
    }
  }
  // one atomic per distinct page table entry per warp (:64-74)
  const uint32_t peers = __match_any_sync(0xffffffffu, address);
  if (address != 0xFFFFFFFFu && (threadIdx.x & 31) == (uint32_t)(__ffs(peers) - 1)) {
    const uint32_t prev = atomicOr(&p.page_tables[address], 1u); // VSMPageState.Visible
    if (!(prev & 1u)) {                                          // the page became visible this frame (:76-83)
      if (prev & 4u) p.page_occupancy[prev >> 16] = 1u;          // already backed: keep the allocator off it
      else {
        const uint32_t k = atomicAdd(p.request_count, 1u);
        if (k < p.request_capacity) { p.requests[k * 3 + 0] = wx; p.requests[k * 3 + 1] = wy; p.requests[k * 3 + 2] = ci_out; }
      }
    }
  }
}

} // namespace oxc
