// vsm_resolve_vs_oracle.cpp — HOST run of the VSM shadow resolve's per-pixel source (oxylus_b200/csrc/oxc_vsm_resolve.cuh), for the
// comparison with the oracle's specification (oracle/oxc_oracle_vsm_resolve.c) that tests/test_vsm_resolve_source_cpu.py makes pixel
// for pixel, without a GPU.  The device header is compiled for the host through tests/host_shim/ (each __f*_rn intrinsic = one IEEE
// binary32 operation under -ffp-contract=off; the binary64 operations of canonical_sincos are plain C++ operations under the same
// flag).  The kernel's parameters are filled the way oxc_vsm_resolve_shadows fills them; the per-CTA tangent basis is computed once.
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
  std::vector<float> depth(W * H), atlas(P * P), shadow(W * H);
  std::vector<float4> normals(W * H);
  std::vector<uint32_t> pt((size_t)vsm.clipmap_count * S * S);
  if (!rd(f, cm.data(), cm.size()) || !rd(f, depth.data(), depth.size()) || !rd(f, normals.data(), normals.size()) || !rd(f, pt.data(), pt.size()) ||
      !rd(f, atlas.data(), atlas.size()))
    return 2;
  std::fclose(f);
  // oxcull.cu oxc_vsm_resolve_shadows
  VsmResolveParams p{};
  for (int i = 0; i < 4; i++) p.inv_pv_row[i] = make_float4(inv_pv[i], inv_pv[4 + i], inv_pv[8 + i], inv_pv[12 + i]);
  p.inv_res_half[0] = (1.0f / res[0]) * 0.5f; p.inv_res_half[1] = (1.0f / res[1]) * 0.5f;
  for (int k = 0; k < vsm.clipmap_count; k++) {
    const float* m = cm[k].projection_view_mat;
    for (int i = 0; i < 4; i++)
      for (int j = 0; j < 4; j++) p.clipmap_row[k][i][j] = m[j * 4 + i];
    p.page_offset[k][0] = cm[k].page_offset[0]; p.page_offset[k][1] = cm[k].page_offset[1];
    p.ortho[k] = m[3] == 0.0f && m[7] == 0.0f && m[11] == 0.0f && m[15] == 1.0f;
  }
  for (int i = 0; i < VSM_RESOLVE_BLOCKER_SAMPLES; i++) vsm_hammersley((uint32_t)i, VSM_RESOLVE_BLOCKER_SAMPLES, p.ham[i][0], p.ham[i][1]);
  for (int i = 0; i < VSM_RESOLVE_PCF_SAMPLES; i++)
    vsm_hammersley((uint32_t)i, VSM_RESOLVE_PCF_SAMPLES, p.ham[VSM_RESOLVE_BLOCKER_SAMPLES + i][0], p.ham[VSM_RESOLVE_BLOCKER_SAMPLES + i][1]);
  for (int i = 0; i < 3; i++) p.light[i] = vsm.directional_light_dir[i];
  p.depth = depth.data(); p.normals = normals.data(); p.page_tables = pt.data(); p.atlas = atlas.data(); p.shadow = shadow.data();
  p.width = (int)W; p.height = (int)H; p.size = (int)S; p.clipmap_count = vsm.clipmap_count;
  p.page_size = vsm.page_size; p.atlas_size = (int)P; p.phys_per_row = (int)P / vsm.page_size;
  {
    volatile float scale_ratio = (float)(vsm.page_table_size - 1) / (float)vsm.page_table_size;
    volatile float effective_width = vsm.first_clipmap_width * scale_ratio;
    volatile float twice = effective_width * 2.0f;
    p.texel_length = twice / vsm.virtual_extent;
  }
  p.bias = vsm.clipmap_selection_bias; p.z_length = vsm.z_length;
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
