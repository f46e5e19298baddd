// atmosphere_vs_oracle.cpp — HOST run of the atmosphere's per-texel source (oxylus_b200/csrc/oxc_atmosphere.cuh), for the comparison
// with the oracle's specification (oracle/oxc_oracle_atmosphere.c) that tests/test_atmosphere_source_cpu.py makes texel for texel,
// without a GPU.  The device header is compiled for the host through tests/host_shim/ (each __f*_rn intrinsic = one IEEE binary32
// operation under -ffp-contract=off).  The parameters come from the header's atmosphere_make_params, as in oxc_atmosphere_transmittance
// and oxc_atmosphere_sky_luts.  Test infrastructure only.
//
//   atmosphere_vs_oracle <inputs.bin> <outputs.bin>
// inputs.bin: OxcAtmosphere of the bake, OxcAtmosphere of the frame, OxcPbrCamera, sun[3] f32, sun_intensity f32.
// outputs.bin receives the transmittance, sky-view and aerial-perspective planes (binary16 RGBA, each at its record's sizes).
#include <cstdint>
#include <cstdio>
#include <vector>

#include "oxc_atmosphere.cuh"

using namespace oxc;

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s inputs.bin outputs.bin\n", argv[0]); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  OxcAtmosphere bake, frame;
  OxcPbrCamera cam;
  float sun[4];
  if (std::fread(&bake, sizeof bake, 1, f) != 1 || std::fread(&frame, sizeof frame, 1, f) != 1 || std::fread(&cam, sizeof cam, 1, f) != 1 ||
      std::fread(sun, 4, 4, f) != 4)
    return 2;
  std::fclose(f);
  const size_t nt = (size_t)bake.transmittance_lut_size[0] * bake.transmittance_lut_size[1];
  const size_t nsv = (size_t)frame.sky_view_lut_size[0] * frame.sky_view_lut_size[1];
  const size_t nap = (size_t)frame.aerial_perspective_lut_size[0] * frame.aerial_perspective_lut_size[1] * frame.aerial_perspective_lut_size[2];
  std::vector<uint16_t> t(nt * 4), sv(nsv * 4), ap(nap * 4);
  const AtmosphereParams pb = atmosphere_make_params(bake, nullptr, nullptr, 0.0f, nullptr, t.data(), nullptr, nullptr, 0);
  for (int y = 0; y < pb.t_h; y++)
    for (int x = 0; x < pb.t_w; x++) atm_transmittance_texel(pb, x, y);
  const AtmosphereParams p = atmosphere_make_params(frame, &cam, sun, sun[3], t.data(), nullptr, sv.data(), ap.data(), 0);
  for (int y = 0; y < p.sv_h; y++)
    for (int x = 0; x < p.sv_w; x++) atm_sky_view_texel(p, x, y);
  for (int z = 0; z < p.ap_d; z++)
    for (int y = 0; y < p.ap_h; y++)
      for (int x = 0; x < p.ap_w; x++) atm_aerial_texel(p, x, y, z);
  FILE* o = std::fopen(argv[2], "wb");
  if (!o || std::fwrite(t.data(), 2, t.size(), o) != t.size() || std::fwrite(sv.data(), 2, sv.size(), o) != sv.size() ||
      std::fwrite(ap.data(), 2, ap.size(), o) != ap.size())
    return 2;
  std::fclose(o);
  std::printf("%zu + %zu + %zu texels\n", nt, nsv, nap);
  return 0;
}
