// fxaa_vs_oracle.cpp — HOST run of FXAA's device source (oxylus_b200/csrc/oxc_fxaa.cuh), for the comparison with the oracle's
// specification (oracle/oxc_oracle_fxaa.c) that tests/test_fxaa_source_cpu.py makes pixel for pixel, without a GPU.  The device header
// is compiled for the host through tests/host_shim/ (each __f*_rn intrinsic = one IEEE binary32 operation under -ffp-contract=off).
// The parameters come from the header's builder, as in oxc_fxaa.  Test infrastructure only.
//
//   fxaa_vs_oracle <inputs.bin> <outputs.bin>
// inputs.bin: width u32, height u32, the frame (width x height float4).  outputs.bin receives the header's four constants (f32), the
// output plane (width x height float4), then each pixel's tap count (u8).
#include <cstdint>
#include <cstdio>
#include <vector>

#include "oxc_fxaa.cuh"

using namespace oxc;

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s inputs.bin outputs.bin\n", argv[0]); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  uint32_t wh[2];
  if (std::fread(wh, 4, 2, f) != 2) return 2;
  const uint32_t w = wh[0], h = wh[1];
  std::vector<float> frame((size_t)w * h * 4), out((size_t)w * h * 4);
  std::vector<uint8_t> taps((size_t)w * h);
  if (std::fread(frame.data(), 4, frame.size(), f) != frame.size()) return 2;
  std::fclose(f);
  const FxaaParams p = fxaa_make_params(frame.data(), w, h, out.data());
  for (int y = 0; y < p.height; y++)
    for (int x = 0; x < p.width; x++) {
      int n;
      p.out[(size_t)y * p.width + x] = fxaa_pixel(p, x, y, n);
      taps[(size_t)y * p.width + x] = (uint8_t)n;
    }
  const float table[4] = {FXAA_EDGE_THRESHOLD_MIN, FXAA_EDGE_THRESHOLD_MAX, FXAA_SUBPIXEL_QUALITY, FXAA_ONE_TWELFTH};
  FILE* o = std::fopen(argv[2], "wb");
  if (!o || std::fwrite(table, 4, 4, o) != 4 || std::fwrite(out.data(), 4, out.size(), o) != out.size() ||
      std::fwrite(taps.data(), 1, taps.size(), o) != taps.size())
    return 2;
  std::fclose(o);
  return 0;
}
