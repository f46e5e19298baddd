// pbr_vs_oracle.cpp — HOST run of PBR apply's per-pixel source (oxylus_b200/csrc/oxc_pbr.cuh), for the comparison with the oracle's
// specification (oracle/oxc_oracle_pbr.c) that tests/test_pbr_source_cpu.py makes pixel for pixel, without a GPU.  The device header
// is compiled for the host through tests/host_shim/ (each __f*_rn intrinsic = one IEEE binary32 operation under -ffp-contract=off; the
// binary64 operations of canonical_sincos / canonical_pow / canonical_pow5 are plain C++ operations under the same flag).  The
// parameters come from the header's pbr_make_params, as in oxc_apply_pbr, and the lights are staged once, as the kernel stages them
// per CTA.  Test infrastructure only.
//
//   pbr_vs_oracle <inputs.bin> <outputs.bin>
// inputs.bin: OxcPbrCamera, OxcPbrSettings, width u32, height u32, optional-plane mask u32 (1 ao, 2 shadow, 4 contact),
// lights[light_count] OxcLight, depth[W*H] f32, albedo, normal, emissive, mro [W*H*4] f32 each, then ao, shadow, contact [W*H] f32
// each when present; outputs.bin receives out[W*H*4] f32.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "oxc_pbr.cuh"

using namespace oxc;

template <typename T>
static bool rd(FILE* f, T* p, size_t n) { return n == 0 || std::fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s inputs.bin outputs.bin\n", argv[0]); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  OxcPbrCamera cam;
  OxcPbrSettings st;
  uint32_t W, H, mask;
  if (!rd(f, &cam, 1) || !rd(f, &st, 1) || !rd(f, &W, 1) || !rd(f, &H, 1) || !rd(f, &mask, 1) || st.light_count > 256) return 2;
  const size_t px = (size_t)W * H;
  std::vector<OxcLight> lights(st.light_count);
  std::vector<float> depth(px), albedo(px * 4), normal(px * 4), emissive(px * 4), mro(px * 4), ao(px), shadow(px), contact(px);
  if (!rd(f, lights.data(), lights.size()) || !rd(f, depth.data(), px) || !rd(f, albedo.data(), px * 4) || !rd(f, normal.data(), px * 4) ||
      !rd(f, emissive.data(), px * 4) || !rd(f, mro.data(), px * 4))
    return 2;
  if (((mask & 1u) && !rd(f, ao.data(), px)) || ((mask & 2u) && !rd(f, shadow.data(), px)) || ((mask & 4u) && !rd(f, contact.data(), px))) return 2;
  std::fclose(f);
  OxcPbrInputs in{};
  in.depth = depth.data(); in.albedo = albedo.data(); in.normal = normal.data(); in.emissive = emissive.data();
  in.metallic_roughness_occlusion = mro.data();
  in.ambient_occlusion = (mask & 1u) ? ao.data() : nullptr;
  in.shadow = (mask & 2u) ? shadow.data() : nullptr;
  in.contact_shadow = (mask & 4u) ? contact.data() : nullptr;
  std::vector<float> out(px * 4);
  // oxcull.cu oxc_apply_pbr
  PbrParams p = pbr_make_params(cam, st, lights.data(), in, W, H, out.data());
  if (!(st.scene_flags & OXC_SCENE_HAS_CONTACT_SHADOWS)) p.contact = nullptr;
  // kernels_pbr.cuh k_apply_pbr: the staged lights, then every pixel
  std::vector<PbrLight> staged(st.light_count);
  for (uint32_t i = 0; i < st.light_count; i++) {
    const float4* r = p.lights + (size_t)i * 4;
    staged[i] = pbr_stage_light(r[0], r[1], r[2], r[3]);
  }
  for (int y = 0; y < (int)H; y++)
    for (int x = 0; x < (int)W; x++) p.out[(size_t)y * W + x] = pbr_pixel(p, staged.data(), x, y);
  FILE* o = std::fopen(argv[2], "wb");
  if (!o || std::fwrite(out.data(), 4, out.size(), o) != out.size()) return 2;
  std::fclose(o);
  std::printf("%u x %u pixels, %u lights\n", W, H, st.light_count);
  return 0;
}
