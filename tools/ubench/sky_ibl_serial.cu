// sky_ibl_serial.cu — the sky IBL cube in the one-thread-per-texel form, the comparison point of the shipped (texel, sample) layout of
// k_atmosphere_sky_ibl: 6,144 threads, each running its texel's 64 samples in one serial loop (oxc_sky_ibl.cuh sky_ibl_texel_serial, the
// same functions, so the same bits).  tools/bench_sky_ibl.py compiles it into a temporary directory with the library's flags and loads
// it through ctypes; the library does not contain it.
#include "../../oxylus_b200/csrc/oxc_sky_ibl.cuh"

namespace {
constexpr int kThreads = 64;

__global__ void __launch_bounds__(kThreads) k_sky_ibl_serial(const __grid_constant__ oxc::SkyIblParams p) {
  const int texel = (int)(blockIdx.x * kThreads + threadIdx.x);
  if (texel >= oxc::SKY_IBL_TEXELS) return;
  oxc::sky_ibl_texel_serial(p, texel / (oxc::SKY_IBL_RES * oxc::SKY_IBL_RES), texel % oxc::SKY_IBL_RES,
                            texel / oxc::SKY_IBL_RES % oxc::SKY_IBL_RES);
}
} // namespace

// oxc_atmosphere_sky_ibl's arguments, without its checks; returns the launch's cudaError_t
extern "C" int sky_ibl_serial(const OxcAtmosphere* atmosphere, const OxcPbrCamera* camera, const float sun_direction[3], float sun_intensity,
                              float sun_ambient_strength, uint32_t frame_index, const uint16_t* transmittance_dev,
                              const uint16_t* sky_view_dev, uint16_t* cube_dev, void* stream) {
  const oxc::SkyIblParams p = oxc::sky_ibl_make_params(*atmosphere, *camera, sun_direction, sun_intensity, sun_ambient_strength, frame_index,
                                                       transmittance_dev, sky_view_dev, cube_dev);
  k_sky_ibl_serial<<<(oxc::SKY_IBL_TEXELS + kThreads - 1) / kThreads, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return (int)cudaGetLastError();
}
