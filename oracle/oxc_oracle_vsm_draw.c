/*
 * oxc_oracle_vsm_draw.c — CPU ORACLE (test infrastructure) of the VSM shadow raster into the physical atlas: the last step of
 * RendererInstance::draw_virtual_shadowmap (Passes/Shadowmaps.cpp:433-754, passes/rmvsm_build_draw_commands.slang,
 * passes/rmvsm_draw_physical_pages.slang).  Same rules as oxc_oracle.c.  It is one translation unit with oxc_oracle.c and
 * oxc_oracle_vsm.c, included below, so that it runs the raster specification's own helpers (tri_clip / tri_passes of the
 * triangle cull, orient2d, edge_bias, the alpha test) rather than copies of them.  Built into liboxc_oracle_vsm_draw.so by
 * oracle/pyoracle_vsm_draw.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_vsm_draw.c
 *
 * SPECIFICATION of orc_vsm_draw_pages (include/oxcull.h oxc_vsm_draw_pages repeats it):
 *   1. triangles: exactly those orc_cull_triangles keeps with the COARSE camera over the HPB cull's survivors (all three clip.z >= 0
 *      and det(xyw) < 1e-4 of mul(coarse PV, world) . p, cull_triangles.slang:62-69).
 *   2. rmvsm_build_draw_commands.slang:21-31: one draw of that list per clipmap c with dirty_flags[c] != 0, highest c first.
 *   3. vertex shader (rmvsm_draw_physical_pages.slang:37-43): clip = mul(clipmap PV, (mul(world, (p, 1)).xyz, 1)), canonical order.
 *      Viewport W = H = physical_page_table_size (P), culling off, no depth attachment.
 *   4. the raster specification of oxc_oracle.c (comment above raster_triangle) steps 3, 5 and 6 — 24.8 snapping, pixel-centre
 *      samples, top-left tie-break, z = (za + E_b*dzb) + E_c*dzc — with two changes:
 *        - both windings are drawn: area2 < 0 swaps vertices 1 and 2 as step 4 does; area2 > 0 keeps the order (a, b, c = 0, 1, 2);
 *          area2 == 0 draws nothing;
 *        - the sink is a minimum: z outside [0, 1] is dropped, -0 is stored as +0, texel = min(texel bits, asuint(z)) as u32.
 *      A triangle with a vertex at w <= 0 or beyond the 2^22 snap range takes the clip path of raster_triangle_clipped (same planes,
 *      same cut arithmetic, same fan), with uv carried as raster_triangle_clipped_uv carries it.
 *   5. fragment shader (:55-87), per sample, f32, in the shader's order: virtual_uv = (px + 0.5, py + 0.5) / P; virtual page =
 *      i32(floor(virtual_uv * page_table_size)), no page outside [0, size - 1], wrapped by the clipmap's page_offset (vsm_wrap);
 *      only a Backed && Dirty entry is written (nothing is inferred from Visible or the HPB); texel = (address % n, address / n) *
 *      page_size + i32(mod(f32(i32(floor(virtual_uv * P))), page_size)), n = P / page_size; a texel outside the atlas is not written.
 *   6. the alpha test of the vis-buffer encode (visbuffer_encode.slang:54-66 == :73-84 here) when a material table is given.
 *   Depth: NDC z = clip.z / clip.w.  The reference writes SV_Position.z / SV_Position.w, which is NDC z for its orthographic
 *   clipmaps (Shadowmaps.cpp:41-59, w = 1) under either convention for SV_Position.w.
 *   Only pixels of dirty pages are visited: each triangle's sample box is cut into the pixel ranges of the Backed && Dirty pages it
 *   touches (the virtual page of a pixel is monotone in the pixel coordinate, so a page's pixels form one range per axis).
 */
#include "oxc_oracle.c"
#define to_i32_f32 vsm_to_i32_f32 /* oxc_oracle_vsm.c has its own copy of this helper */
#include "oxc_oracle_vsm.c"
#undef to_i32_f32

#include "oxc_oracle_vsm_draw.h"

typedef struct VsmDrawTarget {
  const uint32_t* layer; /* page table layer of the clipmap being drawn */
  int32_t size, page_size, P, n, off[2];
  const int32_t* page_of;  /* [P]: virtual page of a pixel coordinate (-1: none) */
  const int32_t* first_px; /* [size + 1]: first pixel whose page is >= v */
  const OrcAlphaMaterial* am;
  uint32_t* atlas;
  uint64_t written;        /* fragments that reached the sink */
} VsmDrawTarget;

/* :60-61 and :67-68 for one pixel coordinate */
static int32_t vsm_draw_page_of(int32_t px, int32_t P, int32_t size) {
  const float uv = ((float)px + 0.5f) / (float)P;
  return to_i32_f32(floorf(uv * (float)size));
}
static int32_t vsm_draw_in_page(int32_t px, int32_t P, int32_t page_size) {
  const float uv = ((float)px + 0.5f) / (float)P;
  const float t = (float)to_i32_f32(floorf(uv * (float)P)), ps = (float)page_size;
  return to_i32_f32(t - ps * floorf(t / ps)); /* com::mod */
}

/* step 4 plain rules + step 5 + step 6 for one triangle (uv may be NULL when am is NULL) */
static void vsm_draw_triangle(const float clip[3][4], const float (*uv)[2], VsmDrawTarget* g) {
  const int64_t W = g->P;
  int64_t fx[3], fy[3];
  float z[3], rws[3];
  if (!(clip[0][3] > 0.0f && clip[1][3] > 0.0f && clip[2][3] > 0.0f)) return;
  for (int i = 0; i < 3; i++) {
    float rw = 1.0f / clip[i][3];
    rws[i] = rw;
    float nx = clip[i][0] * rw, ny = clip[i][1] * rw;
    z[i] = clip[i][2] * rw;
    float sx = (nx * 0.5f + 0.5f) * (float)W, sy = (ny * 0.5f + 0.5f) * (float)W;
    float qx = floorf(sx * 256.0f + 0.5f), qy = floorf(sy * 256.0f + 0.5f);
    if (!(fabsf(qx) <= 4194304.0f && fabsf(qy) <= 4194304.0f)) return;
    fx[i] = (int64_t)qx;
    fy[i] = (int64_t)qy;
  }
  int64_t area2 = orient2d(fx[0], fy[0], fx[1], fy[1], fx[2], fy[2]);
  if (area2 == 0) return;
  const int o[3] = {0, area2 < 0 ? 2 : 1, area2 < 0 ? 1 : 2}; /* a, b, c */
  if (area2 < 0) area2 = -area2;
  const int64_t ax = fx[o[0]], ay = fy[o[0]], bx = fx[o[1]], by = fy[o[1]], cx = fx[o[2]], cy = fy[o[2]];
  const float za = z[o[0]], zb = z[o[1]], zc = z[o[2]];
  int64_t minx = ax < bx ? (ax < cx ? ax : cx) : (bx < cx ? bx : cx);
  int64_t maxx = ax > bx ? (ax > cx ? ax : cx) : (bx > cx ? bx : cx);
  int64_t miny = ay < by ? (ay < cy ? ay : cy) : (by < cy ? by : cy);
  int64_t maxy = ay > by ? (ay > cy ? ay : cy) : (by > cy ? by : cy);
  int64_t px0 = (minx - 128 + 255) >> 8, px1 = (maxx - 128) >> 8;
  int64_t py0 = (miny - 128 + 255) >> 8, py1 = (maxy - 128) >> 8;
  if (px0 < 0) px0 = 0;
  if (py0 < 0) py0 = 0;
  if (px1 > W - 1) px1 = W - 1;
  if (py1 > W - 1) py1 = W - 1;
  if (px1 < px0 || py1 < py0) return;
  const int b0 = edge_bias(bx, by, cx, cy), b1 = edge_bias(cx, cy, ax, ay), b2 = edge_bias(ax, ay, bx, by);
  const float fa = (float)area2;
  const float dzb = (zb - za) / fa, dzc = (zc - za) / fa;
  const int64_t ex[3] = {-(cy - by) * 256, -(ay - cy) * 256, -(by - ay) * 256};
  const int64_t ey[3] = {(cx - bx) * 256, (ax - cx) * 256, (bx - ax) * 256};
  float rwo[3], uvo[3][2];
  for (int k = 0; k < 3; k++) { rwo[k] = rws[o[k]]; uvo[k][0] = uv ? uv[o[k]][0] : 0.0f; uvo[k][1] = uv ? uv[o[k]][1] : 0.0f; }
  /* the pixel ranges of the dirty pages inside the box */
  const int32_t vx0 = g->page_of[px0], vx1 = g->page_of[px1], vy0 = g->page_of[py0], vy1 = g->page_of[py1];
  for (int32_t vy = vy0 < 0 ? 0 : vy0; vy <= vy1 && vy < g->size; vy++)
    for (int32_t vx = vx0 < 0 ? 0 : vx0; vx <= vx1 && vx < g->size; vx++) {
      int32_t wx, wy;
      if (!vsm_wrap(vx, g->off[0], g->size, &wx) || !vsm_wrap(vy, g->off[1], g->size, &wy)) continue;
      const uint32_t e = g->layer[(size_t)wy * g->size + wx];
      if (!((e & VSM_BACKED) && (e & VSM_DIRTY))) continue; /* :65 */
      const uint32_t phys = e >> 16;
      const int64_t base_x = (int64_t)(phys % (uint32_t)g->n) * g->page_size, base_y = (int64_t)(phys / (uint32_t)g->n) * g->page_size;
      const int64_t x0 = px0 > g->first_px[vx] ? px0 : g->first_px[vx], x1 = px1 < g->first_px[vx + 1] - 1 ? px1 : g->first_px[vx + 1] - 1;
      const int64_t y0 = py0 > g->first_px[vy] ? py0 : g->first_px[vy], y1 = py1 < g->first_px[vy + 1] - 1 ? py1 : g->first_px[vy + 1] - 1;
      for (int64_t py = y0; py <= y1; py++)
        for (int64_t px = x0; px <= x1; px++) {
          const int64_t sxp = px * 256 + 128, syp = py * 256 + 128;
          const int64_t e0 = orient2d(bx, by, cx, cy, sxp, syp), e1 = orient2d(cx, cy, ax, ay, sxp, syp), e2 = orient2d(ax, ay, bx, by, sxp, syp);
          if ((e0 + b0) < 0 || (e1 + b1) < 0 || (e2 + b2) < 0) continue;
          const float zz = (za + (float)e1 * dzb) + (float)e2 * dzc;
          if (!(zz >= 0.0f && zz <= 1.0f)) continue;
          if (g->am) {
            const int64_t ev[3] = {e0, e1, e2};
            if (!alpha_keep_fragment(g->am, px, py, ev, ex, ey, rwo, (const float(*)[2])uvo)) continue;
          }
          const int64_t X = base_x + vsm_draw_in_page((int32_t)px, g->P, g->page_size), Y = base_y + vsm_draw_in_page((int32_t)py, g->P, g->page_size);
          if (X >= W || Y >= W) continue; /* an out-of-bounds image atomic is discarded */
          uint32_t zbits = f2bits(zz);
          if (zbits == 0x80000000u) zbits = 0u;
          uint32_t* t = &g->atlas[(size_t)Y * (size_t)W + (size_t)X];
          if (zbits < *t) *t = zbits; /* :86 atomic_min */
          g->written++;
        }
    }
}

/* raster_triangle_clipped_uv's Sutherland-Hodgman (vertex = x y z w u v), pieces through vsm_draw_triangle */
static void vsm_draw_triangle_clipped(const float clip[3][4], const float uv[3][2], VsmDrawTarget* g) {
  float poly[2][12][6];
  int n = 3, cur = 0;
  for (int i = 0; i < 3; i++) { memcpy(poly[0][i], clip[i], 16); poly[0][i][4] = uv[i][0]; poly[0][i][5] = uv[i][1]; }
  for (int plane = 0; plane < 5 && n >= 3; plane++) {
    float(*in)[6] = poly[cur];
    float(*out)[6] = poly[cur ^ 1];
    int m = 0;
    for (int i = 0; i < n; i++) {
      const float* A = in[i];
      const float* B = in[(i + 1) % n];
      const float dA = clip_plane_distance(A, plane), dB = clip_plane_distance(B, plane);
      const int inA = dA >= 0.0f, inB = dB >= 0.0f;
      if (inA) { memcpy(out[m], A, 24); m++; }
      if (inA != inB) {
        const float* I = inA ? A : B;
        const float* O = inA ? B : A;
        const float dI = inA ? dA : dB, dO = inA ? dB : dA;
        const float t = dI / (dI - dO);
        for (int k = 0; k < 6; k++) out[m][k] = I[k] + t * (O[k] - I[k]);
        m++;
      }
    }
    n = m;
    cur ^= 1;
  }
  for (int i = 1; i + 1 < n; i++) {
    float tri[3][4], tuv[3][2];
    const int idx[3] = {0, i, i + 1};
    for (int k = 0; k < 3; k++) { memcpy(tri[k], poly[cur][idx[k]], 16); tuv[k][0] = poly[cur][idx[k]][4]; tuv[k][1] = poly[cur][idx[k]][5]; }
    vsm_draw_triangle(tri, (const float(*)[2])tuv, g);
  }
}

/* step 3: clip positions of triangle `tri` in the clipmap (PV . (W . p)), as tri_clip fetches the vertices */
static void vsm_tri_clip_world(const OrcScene* s, const TriMeshlet* t, const float world[16], const float pv[16], uint32_t tri, float clip[3][4]) {
  const uint32_t* micro = (const uint32_t*)(s->blob + t->lod->local_triangle_indices);
  const uint32_t* vidx = (const uint32_t*)(s->blob + t->lod->indirect_vertex_indices);
  const uint16_t* pos = (const uint16_t*)(s->blob + t->mesh->vertex_positions);
  const uint32_t base = t->meshlet.local_triangle_index_offset + tri * 3;
  for (int c = 0; c < 3; c++) {
    const uint32_t v = vidx[t->meshlet.indirect_vertex_index_offset + micro_index(micro, base + (uint32_t)c)];
    const Vec4_f32 p = {orc_dequantize_half(pos[v * 4 + 0]), orc_dequantize_half(pos[v * 4 + 1]), orc_dequantize_half(pos[v * 4 + 2]), 1.0f};
    const Vec4_f32 w = mul_mv_f32(world, p); /* Transform::to_world_position, scene.slang:288-290 */
    const Vec4_f32 wp = {w.x, w.y, w.z, 1.0f};
    const Vec4_f32 cp = mul_mv_f32(pv, wp);  /* rmvsm_draw_physical_pages.slang:42-43 */
    clip[c][0] = cp.x; clip[c][1] = cp.y; clip[c][2] = cp.z; clip[c][3] = cp.w;
  }
}

uint64_t orc_vsm_draw_pages(const OrcScene* scene, const OxcMeshletInstance* meshlet_instances, const uint32_t* survivors,
                            uint32_t survivor_count, const OxcCullCamera* coarse, const OxcVsmContext* vsm, const OxcVirtualClipmap* clipmaps,
                            const uint32_t* dirty_flags, const uint32_t* page_tables, const OxcMaterialTable* table, float* atlas) {
  const int32_t size = vsm->page_table_size, P = vsm->physical_page_table_size;
  int32_t* page_of = (int32_t*)malloc(sizeof(int32_t) * (size_t)(P > 0 ? P : 1));
  int32_t* first_px = (int32_t*)malloc(sizeof(int32_t) * (size_t)(size + 1));
  for (int32_t px = 0; px < P; px++) page_of[px] = vsm_draw_page_of(px, P, size);
  for (int32_t v = 0, px = 0; v <= size; v++) {
    while (px < P && page_of[px] < v) px++;
    first_px[v] = px;
  }
  VsmDrawTarget g;
  memset(&g, 0, sizeof g);
  g.size = size; g.page_size = vsm->page_size; g.P = P; g.n = P / vsm->page_size; g.page_of = page_of; g.first_px = first_px;
  g.atlas = (uint32_t*)atlas;
  for (uint32_t k = 0; k < survivor_count; k++) {
    const uint32_t mii = survivors[k];
    TriMeshlet t;
    fetch_tri_meshlet(scene, meshlet_instances, mii, coarse, &t); /* t.mvp = coarse PV . W */
    const OxcMeshInstance* inst = &scene->mesh_instances[meshlet_instances[mii].mesh_instance_index];
    const float* world = scene->transforms[inst->transform_index].world;
    OrcAlphaMaterial am;
    g.am = alpha_material_setup(table, inst->material_index, &am) ? &am : NULL;
    uint64_t keep = 0;
    for (uint32_t tri = 0; tri < t.meshlet.triangle_count && tri < 64; tri++) { /* step 1 */
      float cc[3][4];
      if (tri_clip(scene, &t, tri, cc) && tri_passes(cc)) keep |= 1ull << tri;
    }
    for (int32_t c = vsm->clipmap_count - 1; c >= 0 && keep; c--) { /* step 2 */
      if (!dirty_flags[c]) continue;
      g.layer = page_tables + (size_t)c * size * size;
      g.off[0] = clipmaps[c].page_offset[0]; g.off[1] = clipmaps[c].page_offset[1];
      for (uint32_t tri = 0; tri < 64; tri++) {
        if (!(keep >> tri & 1u)) continue;
        float clip[3][4], uv[3][2] = {{0.0f, 0.0f}, {0.0f, 0.0f}, {0.0f, 0.0f}};
        vsm_tri_clip_world(scene, &t, world, clipmaps[c].projection_view_mat, tri, clip);
        if (g.am) tri_uv(scene, &t, tri, uv);
        if (tri_dropped_by_range(clip, (uint32_t)P, (uint32_t)P)) vsm_draw_triangle_clipped(clip, (const float(*)[2])uv, &g);
        else vsm_draw_triangle(clip, (const float(*)[2])uv, &g);
      }
    }
  }
  free(page_of);
  free(first_px);
  return g.written;
}
