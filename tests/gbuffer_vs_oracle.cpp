// gbuffer_vs_oracle.cpp — HOST run of the G-buffer decode's material half (oxylus_b200/csrc/oxc_gbuffer.cuh: the device table that
// oxc_set_materials builds, and gbuffer_shade per pixel), for the comparison with the oracle's specification
// (oracle/oxc_oracle_gbuffer.c) that tests/test_gbuffer_source_cpu.py makes pixel for pixel, without a GPU.  The device header is
// compiled for the host through tests/host_shim/ (each __f*_rn intrinsic = one IEEE binary32 operation under -ffp-contract=off).  The
// per-pixel geometry records come from the oracle (orc_decode_gbuffer_pixels), which runs orc_decode_visbuffer's arithmetic.
// Test infrastructure only.
//
//   gbuffer_vs_oracle <inputs.bin> <planes.bin>
// inputs.bin: u32 material_count, OxcMaterial[material_count]; u32 image_count, per image u32 width, height, format, level_count,
// u64 bytes, the texels; u32 sampler_count, OxcSamplerDesc[sampler_count]; f32 camera position[3]; u64 pixel count n,
// f32 records[n][24], i32 material[n] (-1 discarded, -2 vertex index out of range).  planes.bin receives f32 [n][16]: albedo, normal,
// emissive, metallic_roughness_occlusion (zeros for -1 / -2 and for a material outside the table).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "oxc_gbuffer.cuh"

using namespace oxc;

template <typename T>
static bool rd(FILE* f, T* p, size_t n) { return std::fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv) {
  if (argc != 3) { std::fprintf(stderr, "usage: %s inputs.bin planes.bin\n", argv[0]); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  uint32_t nm = 0, ni = 0, ns = 0;
  if (!rd(f, &nm, 1)) return 2;
  std::vector<OxcMaterial> mats(nm);
  if (!rd(f, mats.data(), nm) || !rd(f, &ni, 1)) return 2;
  std::vector<OxcAlphaImage> images(ni);
  std::vector<std::vector<uint32_t>> texels(ni); // 4-byte aligned storage, as the decode requires
  for (uint32_t i = 0; i < ni; i++) {
    uint32_t hdr[4];
    uint64_t bytes = 0;
    if (!rd(f, hdr, 4) || !rd(f, &bytes, 1)) return 2;
    texels[i].assign((bytes + 3) / 4, 0u);
    if (!rd(f, reinterpret_cast<uint8_t*>(texels[i].data()), bytes)) return 2;
    images[i].texels_dev = texels[i].data();
    images[i].width = hdr[0]; images[i].height = hdr[1]; images[i].format = hdr[2]; images[i].level_count = hdr[3];
  }
  if (!rd(f, &ns, 1)) return 2;
  std::vector<OxcSamplerDesc> samplers(ns);
  float cam[3];
  uint64_t n = 0;
  if (!rd(f, samplers.data(), ns) || !rd(f, cam, 3) || !rd(f, &n, 1)) return 2;
  std::vector<GBufferPixel> px(n);
  std::vector<int32_t> material(n);
  static_assert(sizeof(GBufferPixel) == 24 * sizeof(float), "the oracle's 24-float record");
  if (!rd(f, px.data(), n) || !rd(f, material.data(), n)) return 2;
  std::fclose(f);
  // oxcull.cu oxc_set_materials / oxc_decode_gbuffer
  OxcMaterialTable t{};
  t.materials = mats.data(); t.material_count = nm;
  t.images = ni ? images.data() : nullptr; t.image_count = ni;
  t.samplers = ns ? samplers.data() : nullptr; t.sampler_count = ns;
  std::string error;
  const std::vector<uint8_t> table = gbuffer_table(&t, &error);
  if (!error.empty()) { std::fprintf(stderr, "table refused: %s\n", error.c_str()); return 3; }
  const GBufMaterial* gm = reinterpret_cast<const GBufMaterial*>(table.data());
  const GBufImage* gi = reinterpret_cast<const GBufImage*>(table.data() + (size_t)nm * sizeof(GBufMaterial));
  std::vector<float4> out(n * 4);
  size_t shaded = 0;
  for (uint64_t i = 0; i < n; i++) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a, e = a, m = a;
    if (material[i] >= 0 && (uint32_t)material[i] < nm) {
      const uint32_t k = (uint32_t)material[i];
      gbuffer_shade(gm[k], gi + (size_t)k * GB_SLOTS, px[i], cam[0], cam[1], cam[2], 15u, a, b, e, m);
      shaded++;
    }
    out[i * 4 + 0] = a; out[i * 4 + 1] = b; out[i * 4 + 2] = e; out[i * 4 + 3] = m;
  }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o || std::fwrite(out.data(), sizeof(float4), out.size(), o) != out.size()) return 2;
  std::fclose(o);
  std::printf("%llu pixels, %zu shaded\n", (unsigned long long)n, shaded);
  return 0;
}
