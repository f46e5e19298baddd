// gtao_vs_oracle.cpp — HOST run of the GTAO's per-pixel source (oxylus_b200/csrc/oxc_gtao.cuh), for the comparison with the oracle's
// specification (oracle/oxc_oracle_gtao.c) that tests/test_gtao_source_cpu.py makes pixel for pixel, without a GPU.  The device header
// is compiled for the host through tests/host_shim/ (each __f*_rn intrinsic = one IEEE binary32 operation under -ffp-contract=off; the
// binary64 operations of canonical_sincos / canonical_pow are plain C++ operations under the same flag).  The parameters come
// from the header's gtao_make_params, as in oxc_generate_ambient_occlusion; the pyramid's stored texels come from the header's recursive virtual-pyramid
// rule (the prefilter kernel computes the same values in shared memory).  Test infrastructure only.
//
//   gtao_vs_oracle <inputs.bin> <outputs.bin>
// inputs.bin: OxcGtaoCamera, OxcGtaoSettings, width u32, height u32, depth[W*H] f32, normals[W*H*4] f32;
// outputs.bin receives mips[total] f32, edges[W*H] u32, noisy[W*H] u16, ao[W*H] f32.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "oxc_gtao.cuh"

using namespace oxc;

template <typename T>
static bool rd(FILE* f, T* p, size_t n) { return std::fread(p, sizeof(T), n, f) == n; }
template <typename T>
static bool wr(FILE* f, const std::vector<T>& v) { return std::fwrite(v.data(), sizeof(T), v.size(), f) == v.size(); }

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s inputs.bin outputs.bin\n", argv[0]); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  OxcGtaoCamera cam;
  OxcGtaoSettings st;
  uint32_t W, H;
  if (!rd(f, &cam, 1) || !rd(f, &st, 1) || !rd(f, &W, 1) || !rd(f, &H, 1)) return 2;
  std::vector<float> depth((size_t)W * H), normals((size_t)W * H * 4);
  if (!rd(f, depth.data(), depth.size()) || !rd(f, normals.data(), normals.size())) return 2;
  std::fclose(f);
  std::vector<float> mips((size_t)gtao_mip_texels(W, H)), ao((size_t)W * H);
  std::vector<uint32_t> edges((size_t)W * H);
  std::vector<uint16_t> noisy((size_t)W * H);
  const OxcGtaoTargets t{mips.data(), edges.data(), noisy.data(), ao.data()};
  const GtaoParams p = gtao_make_params(cam, st, depth.data(), normals.data(), W, H, t);
  float (*const level[GTAO_LEVELS])(const GtaoParams&, long long, long long) = {gtao_virtual_level<0>, gtao_virtual_level<1>, gtao_virtual_level<2>,
                                                                                 gtao_virtual_level<3>, gtao_virtual_level<4>};
  for (int k = 0; k < GTAO_LEVELS; k++)
    for (int ty = 0; ty < p.mip_h[k]; ty++)
      for (int tx = 0; tx < p.mip_w[k]; tx++) mips[(size_t)p.mip_off[k] + (size_t)ty * p.mip_w[k] + tx] = nan_canonical(level[k](p, tx, ty));
  size_t sky = 0;
  for (int y = 0; y < (int)H; y++)
    for (int x = 0; x < (int)W; x++) {
      float centre;
      edges[(size_t)y * W + x] = gtao_edges(p, x, y, &centre);
      sky += centre >= fm(p.far_clip, 0.999f);
      noisy[(size_t)y * W + x] = half_bits(gtao_occlusion(p, x, y, centre));
    }
  for (int y = 0; y < (int)H; y++)
    for (int x = 0; x < (int)W; x++) ao[(size_t)y * W + x] = gtao_denoise(p, x, y);
  FILE* o = std::fopen(argv[2], "wb");
  if (!o || !wr(o, mips) || !wr(o, edges) || !wr(o, noisy) || !wr(o, ao)) return 2;
  std::fclose(o);
  std::printf("%u x %u pixels, %zu sky\n", W, H, sky);
  return 0;
}
