// tonemap_vs_oracle.cpp — HOST run of the tonemap's device source (oxylus_b200/csrc/oxc_tonemap.cuh), for the comparison with the
// oracle's specification (oracle/oxc_oracle_tonemap.c) that tests/test_tonemap_source_cpu.py makes pixel for pixel, without a GPU.  The
// device header is compiled for the host through tests/host_shim/ (each __f*_rn intrinsic = one IEEE binary32 operation under
// -ffp-contract=off).  The parameters come from the header's builder, as in oxc_tonemap.  Test infrastructure only.
//
//   tonemap_vs_oracle <inputs.bin> <outputs.bin>
// inputs.bin: width u32, height u32, OxcTonemapSettings, OxcExposure, the frame (width x height float4), the bloom image
// ((width / 2) x (height / 2) float4).  outputs.bin receives the header's constant table (TonemapConstants, 33 f32), then the output
// plane (width x height float4).
#include <cstdint>
#include <cstdio>
#include <vector>

#include "oxc_tonemap.cuh"

using namespace oxc;

template <uint32_t TYPE>
static void run(const TonemapParams& p) {
  for (int y = 0; y < p.height; y++)
    for (int x = 0; x < p.width; x++) p.out[(size_t)y * p.width + x] = tonemap_pixel<TYPE>(p, x, y);
}

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s inputs.bin outputs.bin\n", argv[0]); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  uint32_t wh[2];
  OxcTonemapSettings s;
  OxcExposure record;
  if (std::fread(wh, 4, 2, f) != 2 || std::fread(&s, sizeof s, 1, f) != 1 || std::fread(&record, sizeof record, 1, f) != 1) return 2;
  const uint32_t w = wh[0], h = wh[1];
  std::vector<float> frame((size_t)w * h * 4), bloom((size_t)(w / 2) * (h / 2) * 4 + 4), out((size_t)w * h * 4);
  if (std::fread(frame.data(), 4, frame.size(), f) != frame.size() || std::fread(bloom.data(), 4, bloom.size() - 4, f) != bloom.size() - 4)
    return 2;
  std::fclose(f);
  const TonemapParams p = tonemap_make_params(frame.data(), w, h, s, &record, bloom.data(), out.data());
  switch (s.tonemap_type) {
  case OXC_TONEMAP_NONE: run<OXC_TONEMAP_NONE>(p); break;
  case OXC_TONEMAP_ACES: run<OXC_TONEMAP_ACES>(p); break;
  case OXC_TONEMAP_AGX: run<OXC_TONEMAP_AGX>(p); break;
  default: run<OXC_TONEMAP_GT7>(p); break;
  }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o || std::fwrite(&p.k, sizeof p.k, 1, o) != 1 || std::fwrite(out.data(), 4, out.size(), o) != out.size()) return 2;
  std::fclose(o);
  return 0;
}
