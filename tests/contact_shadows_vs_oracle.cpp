// contact_shadows_vs_oracle.cpp — HOST run of the contact-shadow pass's per-pixel source (oxylus_b200/csrc/oxc_contact_shadows.cuh),
// for the comparison with the oracle's specification (oracle/oxc_oracle_contact_shadows.c) that tests/test_contact_shadows_source_cpu.py
// makes pixel for pixel, without a GPU.  The device header is compiled for the host through tests/host_shim/ (each __f*_rn intrinsic =
// one IEEE binary32 operation under -ffp-contract=off).  The parameters come from the header's cs_make_params, as in
// oxc_contact_shadows.  Test infrastructure only.
//
//   contact_shadows_vs_oracle <inputs.bin> <outputs.bin>
// inputs.bin: OxcContactShadowCamera, OxcContactShadowSettings, width u32, height u32, depth[W*H] f32; outputs.bin receives out[W*H] f32.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "oxc_contact_shadows.cuh"

using namespace oxc;

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s inputs.bin outputs.bin\n", argv[0]); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  OxcContactShadowCamera cam;
  OxcContactShadowSettings st;
  uint32_t W, H;
  if (std::fread(&cam, sizeof cam, 1, f) != 1 || std::fread(&st, sizeof st, 1, f) != 1 || std::fread(&W, 4, 1, f) != 1 ||
      std::fread(&H, 4, 1, f) != 1)
    return 2;
  std::vector<float> depth((size_t)W * H), out((size_t)W * H);
  if (std::fread(depth.data(), 4, depth.size(), f) != depth.size()) return 2;
  std::fclose(f);
  const ContactShadowParams p = cs_make_params(cam, st, depth.data(), W, H, out.data());
  size_t shadowed = 0;
  for (int y = 0; y < (int)H; y++)
    for (int x = 0; x < (int)W; x++) {
      const float v = cs_pixel(p, cs_constants(p), x, y);
      out[(size_t)y * W + x] = v;
      shadowed += v < 1.0f;
    }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o || std::fwrite(out.data(), 4, out.size(), o) != out.size()) return 2;
  std::fclose(o);
  std::printf("%u x %u pixels, %zu in contact\n", W, H, shadowed);
  return 0;
}
