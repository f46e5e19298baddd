// terrain_draw_vs_oracle.cpp — HOST run of the terrain draw's device source (oxylus_b200/csrc/oxc_terrain.cuh: corners, factors,
// rounding, the bisected merge walk, heights, clip positions, with the raster core of oxc_raster_core.cuh), for the comparison with the
// oracle's specification (oracle/oxc_oracle_terrain_draw.c) that tests/test_terrain_draw_source_cpu.py makes pixel for pixel, without a
// GPU.  The device headers are compiled for the host through tests/host_shim/ (each __f*_rn intrinsic = one IEEE binary32 operation
// under -ffp-contract=off; atomicMax = max).  The parameters come from the header's builder, as in oxc_draw_terrain.  Every triangle is
// drawn the way k_draw_terrain draws a small one (the chunks k_raster_big draws for the large ones apply the same per-pixel rule, which
// tests/raster_core_vs_oracle.cpp checks).  Test infrastructure only.
//
//   terrain_draw_vs_oracle <inputs.bin> <outputs.bin>
// inputs.bin: res_x u32, res_y u32, heightmap (u16), OxcTerrainDrawSettings, OxcCullCamera, width, height, prim_bits, instance_count,
// n u32, then n visible patch indices (u32).  outputs.bin receives the vis buffer (width x height u64), then the number of triangles
// each slot drew (u32, n of them).
#include <cstdint>
#include <cstdio>
#include <vector>

static inline unsigned long long atomicMax(unsigned long long* p, unsigned long long v) {
  const unsigned long long old = *p;
  if (v > old) *p = v;
  return old;
}

#include "oxc_terrain.cuh"

using namespace oxc;

static void draw(const TerrainDrawParams& p, float4 c0, float4 c1, float4 c2) {
  TriSetup s;
  const int why = tri_setup(to_screen(c0, p.fW, p.fH), to_screen(c1, p.fW, p.fH), to_screen(c2, p.fW, p.fH), p.width, p.height, s);
  if (why == TRI_DRAW) {
    raster_small(s, p.data, p.vis, p.width);
  } else if (why == TRI_INVALID_VERTEX) {
    float4 poly[2][12];
    int cur;
    const int m = clip_polygon(c0, c1, c2, poly, cur);
    for (int i = 1; i + 1 < m; i++) {
      TriSetup ps;
      if (tri_setup(to_screen(poly[cur][0], p.fW, p.fH), to_screen(poly[cur][i], p.fW, p.fH), to_screen(poly[cur][i + 1], p.fW, p.fH),
                    p.width, p.height, ps) != TRI_DRAW)
        continue;
      ps.narrow = false;
      raster_small(ps, p.data, p.vis, p.width);
    }
  }
}

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s inputs.bin outputs.bin\n", argv[0]); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  uint32_t res[2];
  if (std::fread(res, 4, 2, f) != 2) return 2;
  std::vector<uint16_t> hm((size_t)res[0] * res[1]);
  OxcTerrainDrawSettings st;
  OxcCullCamera cam;
  uint32_t hdr[5];
  if (std::fread(hm.data(), 2, hm.size(), f) != hm.size() || std::fread(&st, sizeof st, 1, f) != 1 || std::fread(&cam, sizeof cam, 1, f) != 1 ||
      std::fread(hdr, 4, 5, f) != 5)
    return 2;
  const uint32_t w = hdr[0], h = hdr[1], prim_bits = hdr[2], instance_count = hdr[3], n = hdr[4];
  std::vector<uint32_t> visible(n ? n : 1);
  if (n && std::fread(visible.data(), 4, n, f) != n) return 2;
  std::fclose(f);
  std::vector<uint64_t> vis((size_t)w * h, 0xFFFFFFFFull);
  OxcDrawIndirectCommand cmd = {4, instance_count, 0, 0};
  const TerrainDrawParams p = terrain_make_params(hm.data(), res[0], res[1], st, visible.data(), &cmd, cam, w, h, vis.data(), prim_bits);
  const uint32_t count = instance_count < p.patch_total ? instance_count : p.patch_total;
  std::vector<uint32_t> drawn(n, 0);
  for (uint32_t slot = 0; slot < n; slot++) {
    const uint32_t idx = terrain_slot_patch(p, slot, count);
    if (idx >= p.patch_total) continue;
    TerrainPatch t;
    terrain_patch_setup(p, idx, t);
    for (uint32_t k = 0; k < t.tri_count; k++) {
      float2 d[3];
      terrain_triangle_domain(t, k, d);
      draw(p, terrain_clip(p, t, d[0]), terrain_clip(p, t, d[1]), terrain_clip(p, t, d[2]));
    }
    drawn[slot] = t.tri_count;
  }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o || std::fwrite(vis.data(), 8, vis.size(), o) != vis.size() || (n && std::fwrite(drawn.data(), 4, n, o) != n)) return 2;
  std::fclose(o);
  return 0;
}
