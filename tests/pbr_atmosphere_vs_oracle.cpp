// pbr_atmosphere_vs_oracle.cpp — HOST run of the atmospheric PBR apply's per-pixel source (oxylus_b200/csrc/oxc_pbr_atmosphere.cuh), for
// the comparison with the oracle's specification (oracle/oxc_oracle_pbr_atmosphere.c) that tests/test_pbr_atmosphere_source_cpu.py makes
// pixel for pixel, without a GPU.  The device header is compiled for the host through tests/host_shim/ (each __f*_rn intrinsic = one IEEE
// binary32 operation under -ffp-contract=off).  The parameters come from the header's pbr_atmosphere_make_params, as in
// oxc_apply_pbr_atmosphere, and the lights are staged once, as the kernel stages them per CTA.  Test infrastructure only.
//
//   pbr_atmosphere_vs_oracle <inputs.bin> <outputs.bin>
// inputs.bin: OxcPbrCamera, OxcPbrSettings, OxcAtmosphere, width u32, height u32, optional-plane mask u32 (1 ao, 2 shadow, 4 contact),
// lights[light_count] OxcLight, depth[W*H] f32, albedo, normal, emissive, mro [W*H*4] f32 each, then ao, shadow, contact [W*H] f32 each
// when present, then the transmittance, sky-view and aerial-perspective LUTs and the cube (binary16 RGBA at the record's sizes);
// outputs.bin receives out[W*H*4] f32.
//   pbr_atmosphere_vs_oracle --constants <outputs.bin>
// outputs.bin receives the bits of the constants the pass reads: 0x3C8EFA35's float, its canonical_cos (min_cos), half_slice_depth and
// near_depth_fade_out, 4 x u32.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "oxc_pbr_atmosphere.cuh"

using namespace oxc;

template <typename T>
static bool rd(FILE* f, T* p, size_t n) { return n == 0 || std::fread(p, sizeof(T), n, f) == n; }

static uint32_t bits(float v) { uint32_t u; std::memcpy(&u, &v, 4); return u; }

int main(int argc, char** argv) {
  if (argc == 3 && std::strcmp(argv[1], "--constants") == 0) {
    const uint32_t c[4] = {bits(PBRA_SUN_RADIANS), bits(canonical_cos(PBRA_SUN_RADIANS)), bits(PBRA_HALF_SLICE), bits(PBRA_NEAR_FADE)};
    FILE* o = std::fopen(argv[2], "wb");
    if (!o || std::fwrite(c, 4, 4, o) != 4) return 2;
    std::fclose(o);
    return 0;
  }
  if (argc != 3) { std::fprintf(stderr, "usage: %s inputs.bin outputs.bin\n", argv[0]); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  OxcPbrCamera cam;
  OxcPbrSettings st;
  OxcAtmosphere at;
  uint32_t W, H, mask;
  if (!rd(f, &cam, 1) || !rd(f, &st, 1) || !rd(f, &at, 1) || !rd(f, &W, 1) || !rd(f, &H, 1) || !rd(f, &mask, 1) || st.light_count > 256) return 2;
  const size_t px = (size_t)W * H;
  std::vector<OxcLight> lights(st.light_count);
  std::vector<float> depth(px), albedo(px * 4), normal(px * 4), emissive(px * 4), mro(px * 4), ao(px), shadow(px), contact(px);
  if (!rd(f, lights.data(), lights.size()) || !rd(f, depth.data(), px) || !rd(f, albedo.data(), px * 4) || !rd(f, normal.data(), px * 4) ||
      !rd(f, emissive.data(), px * 4) || !rd(f, mro.data(), px * 4))
    return 2;
  if (((mask & 1u) && !rd(f, ao.data(), px)) || ((mask & 2u) && !rd(f, shadow.data(), px)) || ((mask & 4u) && !rd(f, contact.data(), px))) return 2;
  const uint32_t* t = at.transmittance_lut_size;
  const uint32_t* v = at.sky_view_lut_size;
  const uint32_t* a = at.aerial_perspective_lut_size;
  std::vector<uint16_t> tl((size_t)t[0] * t[1] * 4), sv((size_t)v[0] * v[1] * 4), ap((size_t)a[0] * a[1] * a[2] * 4), cube(6 * 32 * 32 * 4);
  if (!rd(f, tl.data(), tl.size()) || !rd(f, sv.data(), sv.size()) || !rd(f, ap.data(), ap.size()) || !rd(f, cube.data(), cube.size())) return 2;
  std::fclose(f);
  OxcPbrInputs in{};
  in.depth = depth.data(); in.albedo = albedo.data(); in.normal = normal.data(); in.emissive = emissive.data();
  in.metallic_roughness_occlusion = mro.data();
  in.ambient_occlusion = (mask & 1u) ? ao.data() : nullptr;
  in.shadow = (mask & 2u) ? shadow.data() : nullptr;
  in.contact_shadow = (mask & 4u) ? contact.data() : nullptr;
  const OxcPbrSky sky{tl.data(), sv.data(), ap.data(), cube.data()};
  std::vector<float> out(px * 4);
  // oxcull.cu oxc_apply_pbr_atmosphere
  const PbrAtmParams p = pbr_atmosphere_make_params(cam, st, at, lights.data(), in, sky, W, H, out.data());
  // kernels_pbr_atmosphere.cuh k_apply_pbr_atmosphere: the staged lights, then every pixel
  std::vector<PbrLight> staged(st.light_count);
  for (uint32_t i = 0; i < st.light_count; i++) {
    const float4* r = p.pbr.lights + (size_t)i * 4;
    staged[i] = pbr_stage_light(r[0], r[1], r[2], r[3]);
  }
  for (int y = 0; y < (int)H; y++)
    for (int x = 0; x < (int)W; x++) p.pbr.out[(size_t)y * W + x] = pbr_atmosphere_pixel(p, staged.data(), x, y);
  FILE* o = std::fopen(argv[2], "wb");
  if (!o || std::fwrite(out.data(), 4, out.size(), o) != out.size()) return 2;
  std::fclose(o);
  std::printf("%u x %u pixels, %u lights\n", W, H, st.light_count);
  return 0;
}
