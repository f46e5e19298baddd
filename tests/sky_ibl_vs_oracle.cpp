// sky_ibl_vs_oracle.cpp — HOST run of the sky IBL's per-texel source (oxylus_b200/csrc/oxc_sky_ibl.cuh) and of canonical_acos /
// canonical_atan2 (oxc_exact.cuh), for the comparison with the oracle's specification (oracle/oxc_oracle_sky_ibl.c) that
// tests/test_sky_ibl_source_cpu.py makes texel for texel, without a GPU.  The device header is compiled for the host through
// tests/host_shim/ (each __f*_rn intrinsic = one IEEE binary32 operation under -ffp-contract=off).  The parameters come from the
// header's sky_ibl_make_params, as in oxc_atmosphere_sky_ibl.  Test infrastructure only.
//
//   sky_ibl_vs_oracle <inputs.bin> <outputs.bin>
// inputs.bin: OxcAtmosphere, OxcPbrCamera, sun[3] f32, sun_intensity f32, sun_ambient_strength f32, frame_index u32, the transmittance
// and sky-view planes (binary16 RGBA at the record's sizes), the cube (6 x 32 x 32 binary16 RGBA).  outputs.bin receives the cube.
//   sky_ibl_vs_oracle --functions <inputs.bin> <outputs.bin>
// inputs.bin: n u64, then n f32 y and n f32 x; outputs.bin receives canonical_atan2(y, x) and canonical_acos(x), n f32 each.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "oxc_sky_ibl.cuh"

using namespace oxc;

static int functions(const char* in, const char* out) {
  FILE* f = std::fopen(in, "rb");
  uint64_t n = 0;
  if (!f || std::fread(&n, 8, 1, f) != 1) return 2;
  std::vector<float> y(n), x(n), r(2 * n);
  if (std::fread(y.data(), 4, n, f) != n || std::fread(x.data(), 4, n, f) != n) return 2;
  std::fclose(f);
  for (uint64_t i = 0; i < n; i++) { r[i] = canonical_atan2(y[i], x[i]); r[n + i] = canonical_acos(x[i]); }
  FILE* o = std::fopen(out, "wb");
  if (!o || std::fwrite(r.data(), 4, r.size(), o) != r.size()) return 2;
  std::fclose(o);
  return 0;
}

int main(int argc, char** argv) {
  if (argc == 4 && std::strcmp(argv[1], "--functions") == 0) return functions(argv[2], argv[3]);
  if (argc != 3) { std::fprintf(stderr, "usage: %s [--functions] inputs.bin outputs.bin\n", argv[0]); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  OxcAtmosphere a;
  OxcPbrCamera cam;
  float v[5];
  uint32_t frame_index;
  if (std::fread(&a, sizeof a, 1, f) != 1 || std::fread(&cam, sizeof cam, 1, f) != 1 || std::fread(v, 4, 5, f) != 5 ||
      std::fread(&frame_index, 4, 1, f) != 1)
    return 2;
  std::vector<uint16_t> t((size_t)a.transmittance_lut_size[0] * a.transmittance_lut_size[1] * 4);
  std::vector<uint16_t> sv((size_t)a.sky_view_lut_size[0] * a.sky_view_lut_size[1] * 4), cube((size_t)SKY_IBL_TEXELS * 4);
  if (std::fread(t.data(), 2, t.size(), f) != t.size() || std::fread(sv.data(), 2, sv.size(), f) != sv.size() ||
      std::fread(cube.data(), 2, cube.size(), f) != cube.size())
    return 2;
  std::fclose(f);
  const SkyIblParams p = sky_ibl_make_params(a, cam, v, v[3], v[4], frame_index, t.data(), sv.data(), cube.data());
  for (int face = 0; face < 6; face++)
    for (int y = 0; y < SKY_IBL_RES; y++)
      for (int x = 0; x < SKY_IBL_RES; x++) sky_ibl_texel_serial(p, face, x, y);
  FILE* o = std::fopen(argv[2], "wb");
  if (!o || std::fwrite(cube.data(), 2, cube.size(), o) != cube.size()) return 2;
  std::fclose(o);
  return 0;
}
