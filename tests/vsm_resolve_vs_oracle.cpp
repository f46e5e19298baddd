// vsm_resolve_vs_oracle.cpp — HOST run of the VSM shadow resolve's per-pixel source (oxylus_b200/csrc/oxc_vsm_resolve.cuh), for the
// comparison with the oracle's specification (oracle/oxc_oracle_vsm_resolve.c) that tests/test_vsm_resolve_source_cpu.py makes pixel
// for pixel, without a GPU.  The device header is compiled for the host through tests/host_shim/ (each __f*_rn intrinsic = one IEEE
// binary32 operation under -ffp-contract=off; the binary64 operations of canonical_sincos are plain C++ operations under the same
// flag).  The kernel's parameters come from the header's vsm_resolve_make_params, as in oxc_vsm_resolve_shadows; the per-CTA tangent basis
// is computed once.
// Test infrastructure only.
//
//   vsm_resolve_vs_oracle <inputs.bin> <shadow.bin>
// inputs.bin: OxcVsmContext, inv_projection_view[16] f32, resolution[2] f32, clipmaps[clipmap_count] OxcVirtualClipmap, depth[W*H] f32,
// normals[W*H*4] f32, page_tables[clipmap_count*size*size] u32, atlas[P*P] f32; shadow.bin receives W*H f32.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "oxc_vsm_resolve.cuh"

using namespace oxc;

template <typename T>
static bool rd(FILE* f, T* p, size_t n) { return std::fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s inputs.bin shadow.bin\n", argv[0]); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  OxcVsmContext vsm;
  float inv_pv[16], res[2];
  if (!rd(f, &vsm, 1) || !rd(f, inv_pv, 16) || !rd(f, res, 2)) return 2;
  std::vector<OxcVirtualClipmap> cm(vsm.clipmap_count);
  const size_t W = (size_t)vsm.depth_extent[0], H = (size_t)vsm.depth_extent[1], S = (size_t)vsm.page_table_size, P = (size_t)vsm.physical_page_table_size;
  std::vector<float> depth(W * H), normals(W * H * 4), atlas(P * P), shadow(W * H);
  std::vector<uint32_t> pt((size_t)vsm.clipmap_count * S * S);
  if (!rd(f, cm.data(), cm.size()) || !rd(f, depth.data(), depth.size()) || !rd(f, normals.data(), normals.size()) || !rd(f, pt.data(), pt.size()) ||
      !rd(f, atlas.data(), atlas.size()))
    return 2;
  std::fclose(f);
  const VsmResolveParams p = vsm_resolve_make_params(vsm, inv_pv, res, cm.data(), depth.data(), normals.data(), pt.data(), atlas.data(),
                                                      shadow.data());
  const VsmBasis b = vsm_perpendicular_basis(p.light[0], p.light[1], p.light[2]);
  size_t pcf_pixels = 0;
  for (size_t y = 0; y < H; y++)
    for (size_t x = 0; x < W; x++) {
      bool pcf = false;
      shadow[y * W + x] = vsm_resolve_pixel(p, b, (int)x, (int)y, &pcf);
      pcf_pixels += pcf;
    }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o || std::fwrite(shadow.data(), sizeof(float), shadow.size(), o) != shadow.size()) return 2;
  std::fclose(o);
  std::printf("%zu pixels, %zu ran the PCF loop\n", W * H, pcf_pixels);
  return 0;
}
