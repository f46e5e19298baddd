// renderer_instance.cpp — see renderer_instance.hpp.  Host code only: every byte of compute goes through
// the C ABI of include/oxcull.h.
#include "renderer_instance.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

namespace ox {

namespace {
// OXR_TRACE=1: per-frame device timeline of the pipelined path (frame start / compute end / copy start / copy end),
// printed by oxr_wait relative to the first traced frame.  Debug aid for tools/e2e_probe.py.
struct Trace {
  bool on = false, have_base = false;
  cudaEvent_t base = nullptr;
  cudaEvent_t ev[2][4] = {};
  cudaEvent_t stage[2][8] = {}; // OXR_TRACE=1: after clear+merge, cull_meshes+early cull, early raster, hiz, late cull, late raster
  int cur_slot = 0, n_stage = 0;
  void mark(cudaStream_t s) {
    if (!on || n_stage >= 8) return;
    if (!stage[cur_slot][n_stage]) cudaEventCreate(&stage[cur_slot][n_stage]);
    cudaEventRecord(stage[cur_slot][n_stage++], s);
  }
  Trace() {
    const char* e = std::getenv("OXR_TRACE");
    on = e && e[0] == '1';
  }
} g_trace;

struct Readback {
  OxcMeshletInstanceVisibility visibility;
  uint32_t draw_index_count[2];
  unsigned long long raster_triangles;
};

// the atmosphere's LUTs at the reference's extents (RendererInstance.hpp: 256 x 64, 312 x 192, 32 x 32 x 32), binary16 RGBA
constexpr uint32_t kTransmittanceLut[2] = {256, 64}, kSkyViewLut[2] = {312, 192}, kMultiscatteringLut[2] = {32, 32}, kAerialLut[3] = {32, 32, 32};
constexpr size_t kTransmittanceTexels = (size_t)kTransmittanceLut[0] * kTransmittanceLut[1], kSkyViewTexels = (size_t)kSkyViewLut[0] * kSkyViewLut[1],
                 kAerialTexels = (size_t)kAerialLut[0] * kAerialLut[1] * kAerialLut[2];

// the three LUTs of the renderer's atmosphere block, in this order
struct AtmosphereLuts {
  uint16_t *transmittance, *sky_view, *aerial_perspective;
};
AtmosphereLuts lut_planes(uint16_t* block) {
  return {block, block + kTransmittanceTexels * 4, block + (kTransmittanceTexels + kSkyViewTexels) * 4};
}

// the caller's record with the sizes of those LUTs
OxcAtmosphere sized_atmosphere(const OxcAtmosphere& atmosphere) {
  OxcAtmosphere sized = atmosphere;
  for (int i = 0; i < 3; i++) {
    sized.transmittance_lut_size[i] = i < 2 ? kTransmittanceLut[i] : 1; sized.sky_view_lut_size[i] = i < 2 ? kSkyViewLut[i] : 1;
    sized.multiscattering_lut_size[i] = i < 2 ? kMultiscatteringLut[i] : 1; sized.aerial_perspective_lut_size[i] = kAerialLut[i];
  }
  return sized;
}
} // namespace

int RendererInstance::fail(int rc) {
  if (rc != OXC_OK && error_.empty()) error_ = oxc_last_error();
  return rc;
}

template <typename T>
int RendererInstance::optional_plane(T** p, size_t bytes) {
  if (*p) return OXC_OK;
  if (cudaMalloc(reinterpret_cast<void**>(p), bytes) != cudaSuccess) {
    cudaGetLastError(); // clear the allocation error so that the next launch check does not report it
    *p = nullptr;
    return OXC_E_CAPACITY;
  }
  return OXC_OK;
}

int RendererInstance::copy_to_host(std::initializer_list<HostCopy> copies) {
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  for (const HostCopy& c : copies)
    if (c.host && cudaMemcpyAsync(c.host, c.dev, c.bytes, cudaMemcpyDeviceToHost, s) != cudaSuccess) return fail(OXC_E_CUDA);
  if (cudaStreamSynchronize(s) != cudaSuccess) return fail(OXC_E_CUDA);
  return OXC_OK;
}

RendererInstance::RendererInstance(int device, const OxcCreateInfo& info, uint32_t width, uint32_t height)
    : width_(width), height_(height) {
  if (oxc_create(device, &info, &ctx_) != OXC_OK) {
    error_ = oxc_last_error();
    ctx_ = nullptr;
    return;
  }
  { // the shadow draw's context; a card without room for it keeps the camera path (oxr_vsm_draw_shadows then refuses)
    OxcCreateInfo si = info;
    si.max_views = si.max_views > 10 ? si.max_views : 10;
    if (oxc_create(device, &si, &shadow_ctx_) != OXC_OK) shadow_ctx_ = nullptr;
  }
  cudaStream_t s = nullptr;
  const size_t px = (size_t)width * height;
  if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void**>(&d_vis64_), px * 8) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void**>(&d_vis32_), px * 4) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void**>(&d_depth_), px * 4) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void**>(&d_occluder_), px * 4) != cudaSuccess ||
      cudaMallocHost(&h_pinned_, sizeof(Readback)) != cudaSuccess) {
    error_ = std::string("RendererInstance allocation failed: ") + cudaGetErrorString(cudaGetLastError());
  }
  stream_ = s;
  ids_capacity_ = info.max_meshlet_instances ? info.max_meshlet_instances : 1;
  cudaStream_t cs = nullptr;
  bool ok = cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking) == cudaSuccess;
  copy_stream_ = cs;
  {
    cudaEvent_t ew = nullptr;
    ok = ok && cudaEventCreateWithFlags(&ew, cudaEventDisableTiming) == cudaSuccess;
    ev_window_ = ew;
  }
  for (auto& sl : slots_) {
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    ok = ok && cudaMalloc(reinterpret_cast<void**>(&sl.d_vis32), px * 4) == cudaSuccess &&
         cudaMalloc(reinterpret_cast<void**>(&sl.d_depth), px * 4) == cudaSuccess &&
         cudaMalloc(reinterpret_cast<void**>(&sl.d_ids), (size_t)ids_capacity_ * 4) == cudaSuccess &&
         cudaMalloc(&sl.d_counters, sizeof(Readback)) == cudaSuccess &&
         cudaMemset(sl.d_counters, 0, sizeof(Readback)) == cudaSuccess &&
         cudaMallocHost(&sl.h_readback, sizeof(Readback)) == cudaSuccess &&
         cudaEventCreateWithFlags(&e0, cudaEventDisableTiming) == cudaSuccess &&
         cudaEventCreateWithFlags(&e1, cudaEventDisableTiming) == cudaSuccess;
    sl.ev_compute = e0;
    sl.ev_copy = e1;
  }
  for (int k = 0; k < 2; k++) {
    ok = ok && cudaMalloc(&d_cam_[k], sizeof(OxcCullCamera)) == cudaSuccess && cudaMallocHost(&h_cam_[k], sizeof(OxcCullCamera)) == cudaSuccess;
  }
  {
    const char* e = std::getenv("OXR_NO_GRAPH");
    use_graphs_ = !(e && e[0] == '1');
  }
  if (!ok && error_.empty()) error_ = std::string("RendererInstance pipeline allocation failed: ") + cudaGetErrorString(cudaGetLastError());
}

RendererInstance::~RendererInstance() {
  if (stream_) cudaStreamSynchronize(static_cast<cudaStream_t>(stream_));
  cudaFree(d_vis64_); cudaFree(d_vis32_); cudaFree(d_depth_); cudaFree(d_occluder_); cudaFree(d_overdraw_); cudaFree(d_gbuffer_);
  cudaFree(d_uv_normal_); cudaFree(d_gtao_); cudaFree(d_pbr_); cudaFree(d_lights_); cudaFree(d_contact_); cudaFree(d_atmosphere_); cudaFree(d_sky_ibl_cube_);
  cudaFree(d_post_); cudaFree(d_bloom_); cudaFree(d_tonemap_); cudaFree(d_fxaa_);
  terrain_release();
  if (h_pinned_) cudaFreeHost(h_pinned_);
  if (copy_stream_) cudaStreamSynchronize(static_cast<cudaStream_t>(copy_stream_));
  for (auto& sl : slots_) {
    cudaFree(sl.d_vis32); cudaFree(sl.d_depth); cudaFree(sl.d_ids); cudaFree(sl.d_counters);
    if (sl.h_readback) cudaFreeHost(sl.h_readback);
    if (sl.ev_compute) cudaEventDestroy(static_cast<cudaEvent_t>(sl.ev_compute));
    if (sl.ev_copy) cudaEventDestroy(static_cast<cudaEvent_t>(sl.ev_copy));
  }
  drop_graphs();
  vsm_release();
  cudaFree(d_transforms_previous_);
  for (int k = 0; k < 2; k++) { cudaFree(d_cam_[k]); if (h_cam_[k]) cudaFreeHost(h_cam_[k]); }
  if (ev_window_) cudaEventDestroy(static_cast<cudaEvent_t>(ev_window_));
  if (copy_stream_) cudaStreamDestroy(static_cast<cudaStream_t>(copy_stream_));
  if (stream_) cudaStreamDestroy(static_cast<cudaStream_t>(stream_));
  oxc_destroy(shadow_ctx_);
  oxc_destroy(ctx_);
}

// RendererInstance::update (RendererInstance.cpp:1333-1788): table uploads + mask (re)allocation / zero fill
auto RendererInstance::update(const RendererInstanceUpdateInfo& info) -> int {
  if (!ctx_) return OXC_E_STATE;
  error_.clear();
  drop_graphs(); // the scene tables may be reallocated: captured launches would keep the old addresses
  oxc_bind_camera_buffer(ctx_, nullptr);
  int rc = oxc_set_scene(ctx_, &info.scene, stream_);
  if (rc != OXC_OK) return fail(rc);
  if (shadow_ctx_ && oxc_set_scene(shadow_ctx_, &info.scene, stream_) != OXC_OK) drop_shadow_context(); // camera path unaffected
  // a new scene has no motion yet: previous transforms = current
  const uint32_t n = info.scene.transform_count;
  transforms_.assign(info.scene.transforms, info.scene.transforms + n);
  if (n > transforms_previous_capacity_) {
    cudaFree(d_transforms_previous_);
    d_transforms_previous_ = nullptr;
    transforms_previous_capacity_ = 0;
    if (cudaMalloc(reinterpret_cast<void**>(&d_transforms_previous_), (size_t)n * sizeof(OxcTransformWorld)) != cudaSuccess) return fail(OXC_E_CUDA);
    transforms_previous_capacity_ = n;
  }
  if (n && cudaMemcpyAsync(d_transforms_previous_, transforms_.data(), (size_t)n * sizeof(OxcTransformWorld), cudaMemcpyHostToDevice,
                           static_cast<cudaStream_t>(stream_)) != cudaSuccess)
    return fail(OXC_E_CUDA);
  return OXC_OK;
}

auto RendererInstance::update_transforms(const OxcTransformWorld* transforms, uint32_t first, uint32_t count) -> int {
  if (!ctx_) return OXC_E_STATE;
  int rc = oxc_update_transforms(ctx_, transforms, first, count, stream_);
  if (rc != OXC_OK) return fail(rc);
  if (shadow_ctx_ && oxc_update_transforms(shadow_ctx_, transforms, first, count, stream_) != OXC_OK) drop_shadow_context();
  // the replaced values become the previous transforms (pageable source: the copy has left transforms_ when the call returns)
  if (count && cudaMemcpyAsync(d_transforms_previous_ + first, transforms_.data() + first, (size_t)count * sizeof(OxcTransformWorld),
                               cudaMemcpyHostToDevice, static_cast<cudaStream_t>(stream_)) != cudaSuccess)
    return fail(OXC_E_CUDA);
  std::memcpy(transforms_.data() + first, transforms, (size_t)count * sizeof(OxcTransformWorld));
  return OXC_OK;
}

void RendererInstance::vsm_release() {
  OxrVsmPages& v = vsm_.pages;
  cudaFree(v.page_tables); cudaFree(v.hpb); cudaFree(v.page_occupancy); cudaFree(v.requests); cudaFree(v.allocator);
  cudaFree(v.free_page_list); cudaFree(v.dirty_physical_page_coords); cudaFree(v.clipmap_dirty_flags); cudaFree(v.physical_atlas);
  cudaFree(vsm_.d_dirty_instances); cudaFree(vsm_.d_shadow);
  vsm_ = Vsm();
}

// RendererInstance's vsm_* attachments (created with the renderer in the reference) and the transient buffers of
// Shadowmaps.cpp:100-128, sized from the VSM context; a new shape starts from a cleared table and a zeroed atlas
int RendererInstance::vsm_allocate(const OxcVsmContext& vsm, uint32_t hpb_levels) {
  const uint32_t size = (uint32_t)vsm.page_table_size, layers = (uint32_t)vsm.clipmap_count;
  const uint32_t per_row = (uint32_t)(vsm.physical_page_table_size / vsm.page_size), atlas = (uint32_t)vsm.physical_page_table_size;
  OxrVsmPages& v = vsm_.pages;
  if (v.page_tables && v.page_table_size == size && v.clipmap_count == layers && v.physical_atlas_size == atlas &&
      v.physical_page_count == per_row * per_row && v.hpb_levels == hpb_levels && vsm_.shape.page_size == vsm.page_size)
    return OXC_OK;
  vsm_release();
  const size_t entries = (size_t)layers * size * size, pages = (size_t)per_row * per_row;
  size_t hpb_bytes = 0;
  for (uint32_t l = 0; l < hpb_levels; l++) { const size_t sl = (size >> l) ? (size >> l) : 1u; hpb_bytes += layers * sl * sl; }
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  bool ok = cudaMalloc(reinterpret_cast<void**>(&v.page_tables), entries * 4) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void**>(&v.hpb), hpb_bytes) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void**>(&v.page_occupancy), pages * 4) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void**>(&v.requests), entries * 12) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void**>(&v.allocator), sizeof(OxcVsmAllocator)) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void**>(&v.free_page_list), pages * 4) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void**>(&v.dirty_physical_page_coords), entries * 8) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void**>(&v.clipmap_dirty_flags), layers * 4) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void**>(&v.physical_atlas), (size_t)atlas * atlas * 4) == cudaSuccess;
  ok = ok && cudaMemsetAsync(v.page_tables, 0, entries * 4, s) == cudaSuccess && cudaMemsetAsync(v.hpb, 0, hpb_bytes, s) == cudaSuccess &&
       cudaMemsetAsync(v.allocator, 0, sizeof(OxcVsmAllocator), s) == cudaSuccess &&
       cudaMemsetAsync(v.clipmap_dirty_flags, 0, layers * 4, s) == cudaSuccess &&
       cudaMemsetAsync(v.physical_atlas, 0, (size_t)atlas * atlas * 4, s) == cudaSuccess;
  if (!ok) {
    vsm_release();
    error_ = std::string("virtual shadow map allocation failed: ") + cudaGetErrorString(cudaGetLastError());
    return OXC_E_CUDA;
  }
  v.page_table_size = size; v.clipmap_count = layers; v.physical_page_count = (uint32_t)pages; v.physical_atlas_size = atlas;
  v.hpb_levels = hpb_levels; v.request_capacity = (uint32_t)entries; // every entry is requested at most once per frame
  vsm_.shape = vsm;
  return OXC_OK;
}

// Shadowmaps.cpp:100-430 up to the shadow raster, on stream_, from the depth of the last frame.  The vuk passes become the
// oxc_vsm_* calls; step numbers as in include/oxcull.h.
auto RendererInstance::update_virtual_shadow_pages(VsmPageContext& context) -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  const OxcVsmContext& vsm = context.vsm;
  if (context.hpb_levels < 1 || context.hpb_levels > 16) return OXC_E_INVALID;
  if (context.dirty_mesh_instance_count && !context.dirty_mesh_instances) return OXC_E_INVALID;
  if (vsm.clipmap_count < 1 || vsm.clipmap_count > 10 || vsm.page_table_size < 1 || vsm.page_size < 1 ||
      vsm.physical_page_table_size % vsm.page_size != 0)
    return OXC_E_INVALID;
  if (vsm.depth_extent[0] != (int32_t)width_ || vsm.depth_extent[1] != (int32_t)height_) return OXC_E_INVALID;
  vsm_.updated = false;
  int rc = vsm_allocate(vsm, context.hpb_levels);
  if (rc != OXC_OK) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  OxrVsmPages& v = vsm_.pages;
  if (context.dirty_mesh_instance_count > vsm_.dirty_capacity) {
    cudaFree(vsm_.d_dirty_instances);
    vsm_.d_dirty_instances = nullptr;
    vsm_.dirty_capacity = 0;
    if (cudaMalloc(reinterpret_cast<void**>(&vsm_.d_dirty_instances), (size_t)context.dirty_mesh_instance_count * 4) != cudaSuccess)
      return fail(OXC_E_CUDA);
    vsm_.dirty_capacity = context.dirty_mesh_instance_count;
  }
  const bool invalidate = !context.sun_moved && context.dirty_mesh_instance_count > 0; // :203
  if (invalidate && cudaMemcpyAsync(vsm_.d_dirty_instances, context.dirty_mesh_instances, (size_t)context.dirty_mesh_instance_count * 4,
                                    cudaMemcpyHostToDevice, s) != cudaSuccess)
    return fail(OXC_E_CUDA);
  // the frame's depth attachment: the depth half of the packed vis buffer
  if ((rc = oxc_resolve_visbuffer(ctx_, d_vis64_, width_, height_, nullptr, d_depth_, stream_)) != OXC_OK) return fail(rc);
  // steps 0, 1, 3
  if ((rc = oxc_vsm_begin_frame(ctx_, &vsm, (int)context.sun_moved, v.page_tables, v.page_occupancy, v.physical_page_count,
                                &v.allocator->active_request_count, stream_)) != OXC_OK) return fail(rc);
  // step 2
  if (invalidate && (rc = oxc_vsm_invalidate_pages(ctx_, &vsm, context.clipmaps, vsm_.d_dirty_instances, context.dirty_mesh_instance_count,
                                                   d_transforms_previous_, v.page_tables, stream_)) != OXC_OK) return fail(rc);
  // step 4
  if ((rc = oxc_mark_visible_pages(ctx_, context.inv_projection_view, context.resolution, context.clipmaps, &vsm, d_depth_, v.page_tables,
                                   v.page_occupancy, &v.allocator->active_request_count, v.requests, v.request_capacity, stream_)) != OXC_OK)
    return fail(rc);
  // steps 5, 6, 7, 9
  if ((rc = oxc_vsm_allocate_pages(ctx_, &vsm, v.page_tables, v.page_occupancy, v.physical_page_count, v.requests, v.request_capacity,
                                   v.allocator, v.free_page_list, v.dirty_physical_page_coords, v.clipmap_dirty_flags, stream_)) != OXC_OK)
    return fail(rc);
  // step 8
  if ((rc = oxc_build_hpb(ctx_, v.page_tables, v.page_table_size, v.clipmap_count, v.hpb, v.hpb_levels, stream_)) != OXC_OK) return fail(rc);
  // step 10
  if ((rc = oxc_vsm_clear_dirty_pages(ctx_, &vsm, v.allocator, v.dirty_physical_page_coords, v.physical_atlas, stream_)) != OXC_OK)
    return fail(rc);
  if (cudaStreamSynchronize(s) != cudaSuccess) {
    error_ = cudaGetErrorString(cudaGetLastError());
    return OXC_E_CUDA;
  }
  std::memcpy(vsm_.clipmaps, context.clipmaps, sizeof vsm_.clipmaps);
  std::memcpy(vsm_.inv_projection_view, context.inv_projection_view, sizeof vsm_.inv_projection_view);
  std::memcpy(vsm_.resolution, context.resolution, sizeof vsm_.resolution);
  vsm_.updated = true;
  return OXC_OK;
}

// Shadowmaps.cpp:433-754 after the page loop: cull_geometry(use_hpb) for the coarse camera (cull_meshes, the HPB cull on the device
// dirty flags), then rmvsm_build_draw_commands + rmvsm_draw_physical_pages as one oxc_vsm_draw_pages, on stream_, synchronous
auto RendererInstance::draw_virtual_shadows(const OxcCullCamera& coarse) -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  if (!shadow_ctx_) return OXC_E_CAPACITY; // its context could not be created or kept in step with the scene
  if (!vsm_.updated) return OXC_E_STATE;
  const OxrVsmPages& v = vsm_.pages;
  int rc;
  if ((rc = oxc_cull_meshes(shadow_ctx_, &coarse, OXC_CULL_TEST_ALL, stream_)) != OXC_OK) return fail(rc);
  if ((rc = oxc_cull_meshlets_hpb_dirty_dev(shadow_ctx_, &coarse, vsm_.clipmaps, v.clipmap_dirty_flags, v.clipmap_count, v.hpb, v.page_table_size,
                                            v.hpb_levels, stream_)) != OXC_OK) return fail(rc);
  if ((rc = oxc_vsm_draw_pages(shadow_ctx_, &vsm_.shape, &coarse, vsm_.clipmaps, v.clipmap_dirty_flags, v.page_tables, v.physical_atlas,
                               stream_)) != OXC_OK) return fail(rc);
  if (cudaStreamSynchronize(static_cast<cudaStream_t>(stream_)) != cudaSuccess) {
    error_ = cudaGetErrorString(cudaGetLastError());
    return OXC_E_CUDA;
  }
  return OXC_OK;
}

// Shadowmaps.cpp:756-822 resolve_shadowmap on stream_, synchronous: the vis decode's normals of the last frame (the reference's
// normal_attachment), its depth, then the fullscreen resolve with the VSM state of the last update
auto RendererInstance::resolve_shadowmap(const OxcCullCamera& camera, float* shadow_host) -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  if (!shadow_host) return OXC_E_INVALID;
  if (!vsm_.updated) return OXC_E_STATE;
  const size_t px = (size_t)width_ * height_;
  // the resolve's own planes are an optional part, as the shadow draw's context is
  if (optional_plane(&d_uv_normal_, px * 16) != OXC_OK || optional_plane(&vsm_.d_shadow, px * 4) != OXC_OK) return OXC_E_CAPACITY;
  int rc;
  if ((rc = oxc_bind_camera_buffer(ctx_, nullptr)) != OXC_OK) return fail(rc); // as render(): the camera comes from the argument
  OxcDecodeTargets targets{};
  targets.uv_normal = d_uv_normal_;
  if ((rc = oxc_decode_visbuffer(ctx_, &camera, d_vis64_, nullptr, width_, height_, &targets, stream_)) != OXC_OK) return fail(rc);
  if ((rc = resolve_shadowmap_device(d_uv_normal_)) != OXC_OK) return rc;
  return copy_to_host({{shadow_host, vsm_.d_shadow, px * 4}});
}

// the frame's depth, then the fullscreen resolve into vsm_.d_shadow with the VSM state of the last update, from `normals` (float4 per
// pixel, oct(world normal) in .zw), enqueued on stream_
int RendererInstance::resolve_shadowmap_device(const float* normals) {
  const OxrVsmPages& v = vsm_.pages;
  int rc;
  if ((rc = oxc_resolve_visbuffer(ctx_, d_vis64_, width_, height_, nullptr, d_depth_, stream_)) != OXC_OK) return fail(rc);
  if ((rc = oxc_vsm_resolve_shadows(ctx_, &vsm_.shape, vsm_.inv_projection_view, vsm_.resolution, vsm_.clipmaps, d_depth_, normals,
                                    v.page_tables, v.physical_atlas, vsm_.d_shadow, stream_)) != OXC_OK) return fail(rc);
  return OXC_OK;
}

// the vis decode pass (RendererInstance's "vis decode", visbuffer_decode.slang:88-183) on stream_, synchronous: the G-buffer of the
// frame rendered last, from its packed vis buffer and the material table of the last set_materials
auto RendererInstance::decode_visbuffer(const OxcCullCamera& camera, float* albedo_host, float* normal_host, float* emissive_host, float* mro_host)
    -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  const size_t px = (size_t)width_ * height_;
  if (optional_plane(&d_gbuffer_, px * 64) != OXC_OK) return OXC_E_CAPACITY;
  float* const host[4] = {albedo_host, normal_host, emissive_host, mro_host};
  OxcGBufferTargets targets{};
  float** const dev[4] = {&targets.albedo, &targets.normal, &targets.emissive, &targets.metallic_roughness_occlusion};
  for (int k = 0; k < 4; k++) *dev[k] = host[k] ? d_gbuffer_ + (size_t)k * px * 4 : nullptr;
  const int rc = decode_gbuffer_device(camera, targets);
  if (rc != OXC_OK) return rc;
  return copy_to_host({{albedo_host, targets.albedo, px * 16}, {normal_host, targets.normal, px * 16}, {emissive_host, targets.emissive, px * 16},
                       {mro_host, targets.metallic_roughness_occlusion, px * 16}});
}

// the cleared attachments, then the G-buffer decode of the last frame into `targets` (planes of d_gbuffer_), enqueued on stream_
int RendererInstance::decode_gbuffer_device(const OxcCullCamera& camera, const OxcGBufferTargets& targets) {
  int rc;
  if ((rc = oxc_bind_camera_buffer(ctx_, nullptr)) != OXC_OK) return fail(rc); // as render(): the camera comes from the argument
  if (cudaMemsetAsync(d_gbuffer_, 0, (size_t)width_ * height_ * 64, static_cast<cudaStream_t>(stream_)) != cudaSuccess)
    return fail(OXC_E_CUDA); // discarded pixels: the cleared attachment
  rc = oxc_decode_gbuffer(ctx_, &camera, d_vis64_, nullptr, width_, height_, &targets, stream_);
  if (rc == OXC_E_STATE || rc == OXC_E_INVALID) return rc; // no or unreadable material table: the frame state is intact
  if (rc != OXC_OK) return fail(rc);
  return OXC_OK;
}

// PBR.cpp:143-311 generate_ambient_occlusion on stream_, synchronous: the vis decode's normals of the last frame (the reference's
// normal_attachment .zw), its depth, then prefilter, sector pass and denoise into the renderer's own planes
auto RendererInstance::generate_ambient_occlusion(const OxcCullCamera& camera, const OxcGtaoCamera& gtao_camera, const OxcGtaoSettings& settings,
                                                  float* ao_host) -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  if (!ao_host) return OXC_E_INVALID;
  const size_t px = (size_t)width_ * height_;
  if (optional_plane(&d_uv_normal_, px * 16) != OXC_OK || optional_plane(&d_gtao_, gtao_mip_texels() * 4 + px * 10) != OXC_OK)
    return OXC_E_CAPACITY;
  int rc;
  if ((rc = oxc_bind_camera_buffer(ctx_, nullptr)) != OXC_OK) return fail(rc); // as render(): the camera comes from the argument
  OxcDecodeTargets decode{};
  decode.uv_normal = d_uv_normal_;
  if ((rc = oxc_decode_visbuffer(ctx_, &camera, d_vis64_, nullptr, width_, height_, &decode, stream_)) != OXC_OK) return fail(rc);
  OxcGtaoTargets targets;
  if ((rc = generate_ambient_occlusion_device(gtao_camera, settings, d_uv_normal_, &targets)) != OXC_OK) return rc;
  return copy_to_host({{ao_host, targets.ambient_occlusion, px * 4}});
}

size_t RendererInstance::gtao_mip_texels() const {
  size_t mip_texels = 0;
  for (uint32_t k = 0; k < 5; k++) mip_texels += (size_t)std::max(1u, width_ >> k) * std::max(1u, height_ >> k);
  return mip_texels;
}

// the frame's depth, then prefilter, sector pass and denoise into the renderer's own planes from `normals` (float4 per pixel, oct(world
// normal) in .zw), enqueued on stream_; *targets receives the planes
int RendererInstance::generate_ambient_occlusion_device(const OxcGtaoCamera& gtao_camera, const OxcGtaoSettings& settings, const float* normals,
                                                        OxcGtaoTargets* targets) {
  const size_t px = (size_t)width_ * height_;
  *targets = OxcGtaoTargets{};
  targets->depth_mips = static_cast<float*>(d_gtao_);
  targets->edges = reinterpret_cast<uint32_t*>(targets->depth_mips + gtao_mip_texels());
  targets->ambient_occlusion = reinterpret_cast<float*>(targets->edges + px);
  targets->noisy_occlusion = reinterpret_cast<uint16_t*>(targets->ambient_occlusion + px);
  int rc;
  if ((rc = oxc_resolve_visbuffer(ctx_, d_vis64_, width_, height_, nullptr, d_depth_, stream_)) != OXC_OK) return fail(rc);
  rc = oxc_generate_ambient_occlusion(ctx_, &gtao_camera, &settings, d_depth_, normals, width_, height_, targets, stream_);
  if (rc == OXC_E_INVALID) return rc; // refused settings: nothing was launched, the frame state is intact
  if (rc != OXC_OK) return fail(rc);
  return OXC_OK;
}

// apply_pbr (PBR.cpp:435-531, no atmosphere) on stream_, synchronous, with the passes before it in RendererInstance::render: the
// G-buffer of the last frame, the shadow resolve and the GTAO on its normal plane (whose .zw is the vis decode's uv_normal.zw), then
// the lighting into the renderer's output plane
auto RendererInstance::apply_pbr(const OxcCullCamera& camera, const OxcPbrCamera& pbr_camera, const OxcPbrSettings& settings, const OxcLight* lights_host,
                                 bool cast_shadows, const OxcGtaoCamera* gtao_camera, const OxcGtaoSettings* gtao_settings, float* rgba_host,
                                 const OxcContactShadowCamera* contact_camera, const OxcContactShadowSettings* contact_settings,
                                 const OxcAtmosphere* atmosphere) -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  const bool gtao = (settings.scene_flags & OXC_SCENE_HAS_GTAO) != 0;
  const bool contact = (settings.scene_flags & OXC_SCENE_HAS_CONTACT_SHADOWS) != 0;
  if (!rgba_host || (gtao && (!gtao_camera || !gtao_settings)) || (settings.light_count > 0 && !lights_host)) return OXC_E_INVALID;
  if (contact && (!contact_camera || !contact_settings || contact_settings->steps < 1u || contact_settings->steps > OXC_CONTACT_SHADOW_MAX_STEPS))
    return OXC_E_INVALID; // refused before anything is enqueued
  if (settings.light_count > OXC_MAX_LIGHTS || (!atmosphere && (settings.scene_flags & OXC_SCENE_HAS_ATMOSPHERE)))
    return OXC_E_INVALID; // the atmosphere variant takes a record: refused before anything is enqueued
  // the atmosphere variant: HasAtmosphere selects it, and the reference makes its sky tables only under HasDirectionalLight
  // (RendererInstance.cpp:1022), so without a sun it would read tables no pass wrote that frame
  if (atmosphere && (settings.scene_flags & (OXC_SCENE_HAS_ATMOSPHERE | OXC_SCENE_HAS_DIRECTIONAL_LIGHT)) !=
                        (OXC_SCENE_HAS_ATMOSPHERE | OXC_SCENE_HAS_DIRECTIONAL_LIGHT))
    return OXC_E_INVALID;
  if (cast_shadows && !vsm_.updated) return OXC_E_STATE;
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  const size_t px = (size_t)width_ * height_;
  if (optional_plane(&d_gbuffer_, px * 64) != OXC_OK || (cast_shadows && optional_plane(&vsm_.d_shadow, px * 4) != OXC_OK) ||
      (gtao && optional_plane(&d_gtao_, gtao_mip_texels() * 4 + px * 10) != OXC_OK) || (contact && optional_plane(&d_contact_, px * 4) != OXC_OK))
    return OXC_E_CAPACITY;
  // the output plane and the lights buffer: both or neither
  if (optional_plane(&d_pbr_, px * 16) != OXC_OK || optional_plane(&d_lights_, OXC_MAX_LIGHTS * sizeof(OxcLight)) != OXC_OK) {
    cudaFree(d_pbr_); d_pbr_ = nullptr;
    return OXC_E_CAPACITY;
  }
  int rc;
  // RendererInstance.cpp:1022: the per-frame LUTs and the cube update before the geometry's lighting chain
  if (atmosphere && (rc = sky_ibl_device(*atmosphere, pbr_camera, settings.sun_direction, settings.sun_intensity)) != OXC_OK) return rc;
  OxcGBufferTargets gb{};
  gb.albedo = d_gbuffer_; gb.normal = d_gbuffer_ + px * 4; gb.emissive = d_gbuffer_ + px * 8; gb.metallic_roughness_occlusion = d_gbuffer_ + px * 12;
  if ((rc = decode_gbuffer_device(camera, gb)) != OXC_OK) return rc;
  OxcPbrInputs in{};
  in.albedo = gb.albedo; in.normal = gb.normal; in.emissive = gb.emissive; in.metallic_roughness_occlusion = gb.metallic_roughness_occlusion;
  if (cast_shadows) {
    if ((rc = resolve_shadowmap_device(gb.normal)) != OXC_OK) return rc;
    in.shadow = vsm_.d_shadow;
  }
  if (contact) { // RendererInstance.cpp:990-1020: after the shadow resolve, before the GTAO
    if ((rc = contact_shadows_device(*contact_camera, *contact_settings)) != OXC_OK) return rc;
    in.contact_shadow = d_contact_;
  }
  if (gtao) {
    OxcGtaoTargets t;
    if ((rc = generate_ambient_occlusion_device(*gtao_camera, *gtao_settings, gb.normal, &t)) != OXC_OK) return rc;
    in.ambient_occlusion = t.ambient_occlusion;
  }
  if ((rc = oxc_resolve_visbuffer(ctx_, d_vis64_, width_, height_, nullptr, d_depth_, stream_)) != OXC_OK) return fail(rc);
  in.depth = d_depth_;
  if (settings.light_count &&
      cudaMemcpyAsync(d_lights_, lights_host, settings.light_count * sizeof(OxcLight), cudaMemcpyHostToDevice, s) != cudaSuccess)
    return fail(OXC_E_CUDA);
  if (atmosphere) {
    const AtmosphereLuts luts = lut_planes(d_atmosphere_);
    const OxcPbrSky sky{luts.transmittance, luts.sky_view, luts.aerial_perspective, d_sky_ibl_cube_};
    const OxcAtmosphere sized = sized_atmosphere(*atmosphere);
    rc = oxc_apply_pbr_atmosphere(ctx_, &pbr_camera, &settings, &sized, d_lights_, &in, &sky, width_, height_, d_pbr_, stream_);
  } else {
    rc = oxc_apply_pbr(ctx_, &pbr_camera, &settings, d_lights_, &in, width_, height_, d_pbr_, stream_);
  }
  if (rc != OXC_OK) return fail(rc);
  if ((rc = copy_to_host({{rgba_host, d_pbr_, px * 16}})) != OXC_OK) return rc;
  post_source_ = d_pbr_;
  return OXC_OK;
}

// eye adaptation on stream_, synchronous: the histogram and the record are allocated at the first call, the record filled with 1.0
auto RendererInstance::eye_adaptation(const OxcEyeAdaptationSettings& settings, float delta_time, OxcExposure* exposure_host) -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  if (!post_source_) return OXC_E_INVALID; // no lit plane yet
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  const bool first = !d_post_;
  if (optional_plane(&d_post_, OXC_HISTOGRAM_BIN_COUNT * 4 + sizeof(OxcExposure)) != OXC_OK) return OXC_E_CAPACITY;
  OxcExposure* record = reinterpret_cast<OxcExposure*>(d_post_ + OXC_HISTOGRAM_BIN_COUNT);
  const OxcExposure one{1.0f, 1.0f};
  if (first && (cudaMemcpyAsync(record, &one, sizeof one, cudaMemcpyHostToDevice, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess))
    return fail(OXC_E_CUDA);
  int rc;
  if ((rc = oxc_eye_adaptation(ctx_, post_source_, width_, height_, &settings, delta_time, record, d_post_, stream_)) != OXC_OK) return fail(rc);
  return copy_to_host({{exposure_host, record, sizeof(OxcExposure)}});
}

// bloom on stream_, synchronous: the two chains are allocated at the first call
auto RendererInstance::bloom(const OxcBloomSettings& settings, float* bloom_host) -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  if (!post_source_ || width_ < 2 || height_ < 2) return OXC_E_INVALID;
  const bool adapt = (settings.scene_flags & OXC_SCENE_HAS_EYE_ADAPTATION) != 0;
  if (adapt && !d_post_) return OXC_E_STATE; // no exposure record before an eye_adaptation
  const uint64_t texels = oxc_bloom_chain_texels(width_, height_);
  if (optional_plane(&d_bloom_, texels * 32) != OXC_OK) return OXC_E_CAPACITY;
  const OxcBloomTargets targets{d_bloom_, d_bloom_ + texels * 4};
  const OxcExposure* record = adapt ? reinterpret_cast<const OxcExposure*>(d_post_ + OXC_HISTOGRAM_BIN_COUNT) : nullptr;
  int rc;
  if ((rc = oxc_bloom(ctx_, post_source_, width_, height_, &settings, record, &targets, stream_)) != OXC_OK) return fail(rc);
  if ((rc = copy_to_host({{bloom_host, targets.upsampled, (size_t)(width_ / 2) * (height_ / 2) * 16}})) != OXC_OK) return rc;
  bloomed_ = true;
  return OXC_OK;
}

// tonemap on stream_, synchronous: the output plane is allocated at the first call
auto RendererInstance::tonemap(const OxcTonemapSettings& settings, float* rgba_host) -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  if (!post_source_ || settings.tonemap_type > OXC_TONEMAP_GT7) return OXC_E_INVALID; // no lit plane yet, or no such curve
  const bool adapt = (settings.scene_flags & OXC_SCENE_HAS_EYE_ADAPTATION) != 0, bloom = (settings.scene_flags & OXC_SCENE_HAS_BLOOM) != 0;
  if ((adapt && !d_post_) || (bloom && !bloomed_)) return OXC_E_STATE; // no record before an eye_adaptation, no image before a bloom
  const size_t px = (size_t)width_ * height_;
  if (optional_plane(&d_tonemap_, px * 16) != OXC_OK) return OXC_E_CAPACITY;
  const OxcExposure* record = adapt ? reinterpret_cast<const OxcExposure*>(d_post_ + OXC_HISTOGRAM_BIN_COUNT) : nullptr;
  const float* image = bloom ? d_bloom_ + oxc_bloom_chain_texels(width_, height_) * 4 : nullptr; // upsampled level 0
  int rc;
  if ((rc = oxc_tonemap(ctx_, post_source_, width_, height_, &settings, record, image, d_tonemap_, stream_)) != OXC_OK) return fail(rc);
  return copy_to_host({{rgba_host, d_tonemap_, px * 16}});
}

// FXAA on stream_, synchronous: the output plane is allocated at the first call and becomes the post chain's source
auto RendererInstance::fxaa(float* rgba_host) -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  if (!post_source_) return OXC_E_INVALID; // no lit plane yet
  const size_t px = (size_t)width_ * height_;
  if (optional_plane(&d_fxaa_, px * 16) != OXC_OK) return OXC_E_CAPACITY;
  int rc;
  if ((rc = oxc_fxaa(ctx_, d_pbr_, width_, height_, d_fxaa_, stream_)) != OXC_OK) return fail(rc);
  if ((rc = copy_to_host({{rgba_host, d_fxaa_, px * 16}})) != OXC_OK) return rc;
  post_source_ = d_fxaa_;
  return OXC_OK;
}

// the contact_shadows pass (RendererInstance.cpp:990-1020) on stream_, synchronous: the last frame's depth, the pass into the renderer's
// own plane, width x height floats to the host
auto RendererInstance::contact_shadows(const OxcContactShadowCamera& contact_camera, const OxcContactShadowSettings& settings, float* contact_host)
    -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  if (!contact_host) return OXC_E_INVALID;
  const size_t px = (size_t)width_ * height_;
  if (optional_plane(&d_contact_, px * 4) != OXC_OK) return OXC_E_CAPACITY;
  int rc;
  if ((rc = contact_shadows_device(contact_camera, settings)) != OXC_OK) return rc;
  return copy_to_host({{contact_host, d_contact_, px * 4}});
}

// the atmosphere's LUTs on stream_, without a copy: the bake once with the default record (RendererInstance.cpp:203-226), then the two
// per-frame LUTs with the caller's record at the renderer's extents (:1456-1459, PBR.cpp:11-50 and :96-140)
int RendererInstance::atmosphere_luts_device(const OxcAtmosphere& atmosphere, const OxcPbrCamera& camera, const float sun_direction[3],
                                             float sun_intensity) {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  if (!sun_direction) return OXC_E_INVALID;
  if (optional_plane(&d_atmosphere_, (kTransmittanceTexels + kSkyViewTexels + kAerialTexels) * 8) != OXC_OK) return OXC_E_CAPACITY;
  const AtmosphereLuts luts = lut_planes(d_atmosphere_);
  const OxcAtmosphere sized = sized_atmosphere(atmosphere);
  int rc;
  if (!transmittance_baked_) {
    // GPU::Atmosphere{} with only the transmittance and multiple-scattering sizes set, as the reference's init bakes it
    OxcAtmosphere def = {{0.005802f, 0.013558f, 0.033100f}, 8.0f, {0.003996f, 0.003996f, 0.003996f}, 1.2f, 0.004440f, 3.6f,
                         {0.000650f, 0.001881f, 0.000085f}, 25.0f, 15.0f, {0.3f, 0.3f, 0.3f}, 6360.0f, 6460.0f, 8.0f, 1.0f,
                         {kTransmittanceLut[0], kTransmittanceLut[1], 1}, {0, 0, 0}, {kMultiscatteringLut[0], kMultiscatteringLut[1], 1},
                         {0, 0, 0}};
    if ((rc = oxc_atmosphere_transmittance(ctx_, &def, luts.transmittance, stream_)) != OXC_OK) return fail(rc);
    transmittance_baked_ = true;
  }
  if ((rc = oxc_atmosphere_sky_luts(ctx_, &sized, &camera, sun_direction, sun_intensity, luts.transmittance, luts.sky_view, luts.aerial_perspective,
                                    stream_)) != OXC_OK)
    return fail(rc);
  return OXC_OK;
}

// atmosphere_luts_device, then the copies to the host, synchronous
auto RendererInstance::atmosphere_luts(const OxcAtmosphere& atmosphere, const OxcPbrCamera& camera, const float sun_direction[3],
                                       float sun_intensity, uint16_t* transmittance_host, uint16_t* sky_view_host,
                                       uint16_t* aerial_perspective_host) -> int {
  int rc;
  if ((rc = atmosphere_luts_device(atmosphere, camera, sun_direction, sun_intensity)) != OXC_OK) return rc;
  const AtmosphereLuts luts = lut_planes(d_atmosphere_);
  return copy_to_host({{transmittance_host, luts.transmittance, kTransmittanceTexels * 8}, {sky_view_host, luts.sky_view, kSkyViewTexels * 8},
                       {aerial_perspective_host, luts.aerial_perspective, kAerialTexels * 8}});
}

// the per-frame LUTs as atmosphere_luts makes them, then the sky IBL cube (PBR.cpp:52-94) into the renderer's cube with
// sun_ambient_strength 0.15 and frame_index = the count of earlier calls, on stream_ without a copy
int RendererInstance::sky_ibl_device(const OxcAtmosphere& atmosphere, const OxcPbrCamera& camera, const float sun_direction[3],
                                     float sun_intensity) {
  int rc;
  if ((rc = atmosphere_luts_device(atmosphere, camera, sun_direction, sun_intensity)) != OXC_OK) return rc;
  const bool first = !d_sky_ibl_cube_;
  if (optional_plane(&d_sky_ibl_cube_, OXC_SKY_IBL_CUBE_BYTES) != OXC_OK) return OXC_E_CAPACITY;
  // cleared to black, as RendererInstance.cpp:197-201 clears the reference's: no texel has history
  if (first && cudaMemsetAsync(d_sky_ibl_cube_, 0, OXC_SKY_IBL_CUBE_BYTES, static_cast<cudaStream_t>(stream_)) != cudaSuccess) return fail(OXC_E_CUDA);
  const AtmosphereLuts luts = lut_planes(d_atmosphere_);
  const OxcAtmosphere sized = sized_atmosphere(atmosphere);
  if ((rc = oxc_atmosphere_sky_ibl(ctx_, &sized, &camera, sun_direction, sun_intensity, 0.15f, sky_ibl_calls_, luts.transmittance, luts.sky_view,
                                   d_sky_ibl_cube_, stream_)) != OXC_OK)
    return fail(rc);
  sky_ibl_calls_++;
  return OXC_OK;
}

// sky_ibl_device, then the cube to the host, synchronous
auto RendererInstance::atmosphere_sky_ibl(const OxcAtmosphere& atmosphere, const OxcPbrCamera& camera, const float sun_direction[3],
                                          float sun_intensity, uint16_t* cube_host) -> int {
  int rc;
  if ((rc = sky_ibl_device(atmosphere, camera, sun_direction, sun_intensity)) != OXC_OK) return rc;
  return copy_to_host({{cube_host, d_sky_ibl_cube_, OXC_SKY_IBL_CUBE_BYTES}});
}

int RendererInstance::contact_shadows_device(const OxcContactShadowCamera& contact_camera, const OxcContactShadowSettings& settings) {
  if (settings.steps < 1u || settings.steps > OXC_CONTACT_SHADOW_MAX_STEPS) return OXC_E_INVALID; // refused before anything is enqueued
  int rc;
  if ((rc = oxc_resolve_visbuffer(ctx_, d_vis64_, width_, height_, nullptr, d_depth_, stream_)) != OXC_OK) return fail(rc);
  rc = oxc_contact_shadows(ctx_, &contact_camera, &settings, d_depth_, width_, height_, d_contact_, stream_);
  if (rc != OXC_OK) return fail(rc);
  return OXC_OK;
}

// the shadow context is an optional part: losing it must not take the camera path down with it
void RendererInstance::drop_shadow_context() {
  cudaStreamSynchronize(static_cast<cudaStream_t>(stream_));
  oxc_destroy(shadow_ctx_);
  shadow_ctx_ = nullptr;
}

auto RendererInstance::virtual_shadow_pages(OxrVsmPages* out) const -> int {
  if (!out) return OXC_E_INVALID;
  if (!vsm_.pages.page_tables) return OXC_E_STATE;
  *out = vsm_.pages;
  return OXC_OK;
}

// MainGeometryContext::draw_overdraw (RendererInstance.cpp:771-776; debug view "Overdraw"): the encode pass's fragment counter for
// the frame that was rendered last — both passes' survivor lists are still in place, so this runs after the frame, not inside it
auto RendererInstance::overdraw(const OxcCullCamera& camera, uint32_t* overdraw_host) -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  if (!overdraw_host) return OXC_E_INVALID;
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  const size_t px = (size_t)width_ * height_;
  if (!d_overdraw_ && cudaMalloc(reinterpret_cast<void**>(&d_overdraw_), px * 4) != cudaSuccess) return fail(OXC_E_CUDA);
  int rc;
  if ((rc = oxc_bind_camera_buffer(ctx_, nullptr)) != OXC_OK) return fail(rc); // as render(): the camera comes from the argument
  if ((rc = oxc_clear_overdraw(ctx_, d_overdraw_, width_, height_, s)) != OXC_OK) return fail(rc);
  if ((rc = oxc_raster_overdraw(ctx_, &camera, OXC_CULL_TEST_ALL, width_, height_, d_overdraw_, /*after_frame=*/1, s)) != OXC_OK) return fail(rc);
  if ((rc = oxc_raster_overdraw(ctx_, &camera, OXC_CULL_TEST_ALL | OXC_CULL_LATE_PASS, width_, height_, d_overdraw_, /*after_frame=*/1, s)) != OXC_OK) return fail(rc);
  return copy_to_host({{overdraw_host, d_overdraw_, px * 4}});
}

// the reference uploads its material table with the scene (RendererInstance.cpp:1333-1788); the vis-buffer encode reads it for
// the alpha-tested discard (visbuffer_encode.slang:54-66)
auto RendererInstance::set_materials(const OxcMaterialTable* table) -> int {
  if (!ctx_) return OXC_E_STATE;
  error_.clear();
  drop_graphs(); // the raster's launch sequence depends on whether a table is set
  int rc = oxc_set_materials(ctx_, table, stream_);
  if (rc == OXC_OK && shadow_ctx_ && oxc_set_materials(shadow_ctx_, table, stream_) != OXC_OK) drop_shadow_context(); // the shadow alpha test
  return fail(rc);
}

auto RendererInstance::set_external_depth(const float* depth_host) -> int {
  if (!ctx_) return OXC_E_STATE;
  has_external_depth_ = depth_host != nullptr;
  if (!depth_host) return OXC_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  if (cudaMemcpyAsync(d_occluder_, depth_host, (size_t)width_ * height_ * 4, cudaMemcpyHostToDevice, s) != cudaSuccess ||
      cudaStreamSynchronize(s) != cudaSuccess)
    return fail(OXC_E_CUDA);
  return OXC_OK;
}

void RendererInstance::terrain_release() {
  cudaFree(terrain_.d_heightmap); cudaFree(terrain_.d_minmax); cudaFree(terrain_.d_visible); cudaFree(terrain_.d_mask); cudaFree(terrain_.d_cmd);
  terrain_ = Terrain();
}

auto RendererInstance::set_terrain(const uint16_t* heightmap_host, uint32_t res_x, uint32_t res_y, const float* patch_minmax_host,
                                   const OxcTerrainDrawSettings* settings) -> int {
  if (!ctx_) return OXC_E_STATE;
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  if (cudaStreamSynchronize(s) != cudaSuccess) return fail(OXC_E_CUDA); // no frame in flight reads the buffers released below
  drop_graphs(); // a captured frame holds the old terrain's launches (or none)
  terrain_release();
  if (!heightmap_host) return OXC_OK;
  if (!patch_minmax_host || !settings || res_x == 0 || res_y == 0 || res_x > 65536 || res_y > 65536) return OXC_E_INVALID;
  const uint64_t total = (uint64_t)settings->terrain.patch_count[0] * settings->terrain.patch_count[1];
  if (total == 0 || total > 0xFFFFFFFFull) return OXC_E_INVALID;
  if (!std::isfinite(settings->target_edge_pixels) || !(settings->target_edge_pixels >= 1.0f) || !std::isfinite(settings->max_tessellation) ||
      !(settings->max_tessellation >= 1.0f))
    return OXC_E_INVALID;
  const size_t texels = (size_t)res_x * res_y, words = (size_t)((total + 31) / 32);
  Terrain t;
  t.res_x = res_x; t.res_y = res_y; t.settings = *settings;
  if (cudaMalloc(&t.d_heightmap, texels * 2) != cudaSuccess || cudaMalloc(&t.d_minmax, (size_t)total * 8) != cudaSuccess ||
      cudaMalloc(&t.d_visible, (size_t)total * 4) != cudaSuccess || cudaMalloc(&t.d_mask, words * 4) != cudaSuccess ||
      cudaMalloc(&t.d_cmd, sizeof(OxcDrawIndirectCommand)) != cudaSuccess) {
    cudaGetLastError();
    terrain_ = t;
    terrain_release();
    return OXC_E_CAPACITY;
  }
  t.set = true;
  terrain_ = t;
  if (cudaMemcpyAsync(t.d_heightmap, heightmap_host, texels * 2, cudaMemcpyHostToDevice, s) != cudaSuccess ||
      cudaMemcpyAsync(t.d_minmax, patch_minmax_host, (size_t)total * 8, cudaMemcpyHostToDevice, s) != cudaSuccess ||
      cudaMemsetAsync(t.d_mask, 0, words * 4, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess)
    return fail(OXC_E_CUDA);
  return OXC_OK;
}

int RendererInstance::terrain_pass(const OxcCullCamera& camera, bool late) {
  const uint32_t flags = OXC_CULL_TEST_FRUSTUM | OXC_CULL_TEST_OCCLUSION | (late ? OXC_CULL_LATE_PASS : 0u);
  int rc = oxc_cull_terrain(ctx_, &terrain_.settings.terrain, terrain_.d_minmax, &camera, flags, terrain_.d_visible, terrain_.d_mask,
                            terrain_.d_cmd, stream_);
  if (rc != OXC_OK) return rc;
  return oxc_draw_terrain(ctx_, terrain_.d_heightmap, terrain_.res_x, terrain_.res_y, &terrain_.settings, terrain_.d_visible, terrain_.d_cmd,
                          &camera, width_, height_, d_vis64_, stream_);
}

// CullGeometry.cpp:61-404
auto RendererInstance::cull_geometry(CullGeometryContext& context) -> int {
  int rc;
  // --- Stage 1: cull_meshes (only on the first cull of a sequence), :68-117
  if (context.init_cull_meshes)
    if ((rc = oxc_cull_meshes(ctx_, &context.cull_camera, context.cull_flags, stream_)) != OXC_OK) return fail(rc);
  // --- Stage 2: cull_meshlets, :124-335.  The plain variant is dispatched with TestFrustum only (:275).
  if (context.use_hiz) rc = oxc_cull_meshlets(ctx_, &context.cull_camera, context.cull_flags, 1, stream_);
  else rc = oxc_cull_meshlets(ctx_, &context.cull_camera, OXC_CULL_TEST_FRUSTUM, 0, stream_);
  if (rc != OXC_OK) return fail(rc);
  // --- Stage 3: cull_triangles, :337-403 (optional here: the raster fuses it)
  if (context.materialize_indices)
    if ((rc = oxc_cull_triangles(ctx_, &context.cull_camera, context.cull_flags, stream_)) != OXC_OK) return fail(rc);
  return OXC_OK;
}

// CullGeometry.cpp:10-59 — source is the depth half of the packed vis buffer
auto RendererInstance::generate_hiz(MainGeometryContext& context) -> int {
  return fail(oxc_build_hiz_packed(ctx_, context.visbuffer_attachment, context.width, context.height, stream_));
}

// DrawGeometry.cpp:104-190 — "vis encode": the HW raster of reordered_indices becomes the fused
// triangle-cull + software raster into the packed image
auto RendererInstance::draw_for_visbuffer(MainGeometryContext& context) -> int {
  return fail(oxc_raster_visbuffer(ctx_, &context.cull_camera, context.cull_flags, context.width, context.height,
                                   context.visbuffer_attachment, 0, stream_));
}

// The geometry section of RendererInstance::render (RendererInstance.cpp:768-884), enqueued on stream_, in two halves: the
// pipelined path sends the previous frame's results to the host between them (flush_pending_copy), and replays each half
// from a CUDA graph.
//   head: attachments cleared, run_geometry_pass(false) up to and including its cull          (:562-588, :842-870)
//   tail: its draw, generate_hiz, run_geometry_pass(true)                                      (:871-884)
int RendererInstance::frame_head(const OxcCullCamera& camera, const float* occluder_depth_host, void* readback, bool readback_on_device) {
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  const size_t px = (size_t)width_ * height_;
  int rc;
  OxcOutputs out;
  if ((rc = oxc_get_outputs(ctx_, &out)) != OXC_OK) return rc;
  Readback* rb = static_cast<Readback*>(readback);
  // attachments: depth cleared to 0, vis buffer to ~0 (RendererInstance.cpp:562-571,629-680), Hi-Z cleared every frame (:579-588)
  if (occluder_depth_host) {
    if (cudaMemcpyAsync(d_occluder_, occluder_depth_host, px * 4, cudaMemcpyHostToDevice, s) != cudaSuccess) return OXC_E_CUDA;
    has_external_depth_ = true;
  }
  if (has_external_depth_) rc = oxc_clear_visbuffer_with_depth(ctx_, d_vis64_, d_occluder_, width_, height_, s); // clear + merge, one pass
  else rc = oxc_clear_visbuffer(ctx_, d_vis64_, width_, height_, s);
  if (rc != OXC_OK) return rc;
  if ((rc = oxc_clear_hiz(ctx_, s)) != OXC_OK) return rc;
  g_trace.mark(s);
  if (readback_on_device) {
    if (cudaMemsetAsync(rb->draw_index_count, 0, sizeof rb->draw_index_count, s) != cudaSuccess) return OXC_E_CUDA;
  } else {
    rb->draw_index_count[0] = rb->draw_index_count[1] = 0;
  }
  // RendererInstance.cpp:796-800: hoisted so the early pass's visibility / dispatch buffers persist into the late pass
  CullGeometryContext cull_geometry_context;
  cull_geometry_context.use_hiz = true;
  cull_geometry_context.init_cull_meshes = true;
  cull_geometry_context.cull_camera = camera;
  cull_geometry_context.materialize_indices = out.reordered_indices != nullptr;
  if ((rc = cull_geometry(cull_geometry_context)) != OXC_OK) return rc; // run_geometry_pass(false), cull half
  g_trace.mark(s);
  return OXC_OK;
}

int RendererInstance::frame_tail(const OxcCullCamera& camera, void* readback) {
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  int rc;
  OxcOutputs out;
  if ((rc = oxc_get_outputs(ctx_, &out)) != OXC_OK) return rc;
  Readback* rb = static_cast<Readback*>(readback);
  const bool materialize = out.reordered_indices != nullptr;
  MainGeometryContext main_geometry_context;
  main_geometry_context.visbuffer_attachment = d_vis64_;
  main_geometry_context.width = width_;
  main_geometry_context.height = height_;
  main_geometry_context.cull_camera = camera;
  // run_geometry_pass(false), draw half (:871-881)
  if (materialize && cudaMemcpyAsync(&rb->draw_index_count[0], &out.draw_cmd->index_count, 4, cudaMemcpyDefault, s) != cudaSuccess) return OXC_E_CUDA;
  main_geometry_context.cull_flags = OXC_CULL_TEST_ALL;
  if ((rc = draw_for_visbuffer(main_geometry_context)) != OXC_OK) return rc;
  if (terrain_.set && (rc = terrain_pass(camera, false)) != OXC_OK) return rc; // :864-880, after the meshlets
  g_trace.mark(s);
  if ((rc = generate_hiz(main_geometry_context)) != OXC_OK) return rc; // :883
  g_trace.mark(s);
  // run_geometry_pass(true) (:884): cull_flags |= LatePass, init_cull_meshes = false
  CullGeometryContext cull_geometry_context;
  cull_geometry_context.use_hiz = true;
  cull_geometry_context.init_cull_meshes = false;
  cull_geometry_context.cull_flags = OXC_CULL_TEST_ALL | OXC_CULL_LATE_PASS;
  cull_geometry_context.cull_camera = camera;
  cull_geometry_context.materialize_indices = materialize;
  if ((rc = cull_geometry(cull_geometry_context)) != OXC_OK) return rc;
  g_trace.mark(s);
  if (materialize && cudaMemcpyAsync(&rb->draw_index_count[1], &out.draw_cmd->index_count, 4, cudaMemcpyDefault, s) != cudaSuccess) return OXC_E_CUDA;
  main_geometry_context.cull_flags = cull_geometry_context.cull_flags;
  if ((rc = draw_for_visbuffer(main_geometry_context)) != OXC_OK) return rc;
  if (terrain_.set && (rc = terrain_pass(camera, true)) != OXC_OK) return rc;
  g_trace.mark(s);
  return OXC_OK;
}

int RendererInstance::run_frame(const OxcCullCamera& camera, const float* occluder_depth_host, void* readback, bool readback_on_device) {
  int rc;
  if ((rc = frame_head(camera, occluder_depth_host, readback, readback_on_device)) != OXC_OK) return rc;
  if (pending_.active && (rc = flush_pending_copy(true)) != OXC_OK) return rc; // previous frame's results go out now
  return frame_tail(camera, readback);
}

// results of the frame -> the slot's device staging (drained by wait() of the slot's previous ticket)
int RendererInstance::stage_results(int slot, bool want_vis32, bool want_depth, uint32_t n_ids) {
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  Slot& sl = slots_[slot];
  int rc;
  OxcOutputs out;
  if ((rc = oxc_get_outputs(ctx_, &out)) != OXC_OK) return rc;
  Readback* dc = static_cast<Readback*>(sl.d_counters);
  if (want_vis32 || want_depth)
    if ((rc = oxc_resolve_visbuffer(ctx_, d_vis64_, width_, height_, want_vis32 ? sl.d_vis32 : nullptr, want_depth ? sl.d_depth : nullptr, s)) != OXC_OK)
      return rc;
  if (n_ids && cudaMemcpyAsync(sl.d_ids, out.visible_meshlet_instances_indices, (size_t)n_ids * 4, cudaMemcpyDeviceToDevice, s) != cudaSuccess)
    return OXC_E_CUDA;
  if (cudaMemcpyAsync(&dc->visibility, out.visibility, sizeof dc->visibility, cudaMemcpyDeviceToDevice, s) != cudaSuccess) return OXC_E_CUDA;
  if (cudaMemcpyAsync(&dc->raster_triangles, out.raster_triangle_count, 8, cudaMemcpyDeviceToDevice, s) != cudaSuccess) return OXC_E_CUDA;
  return OXC_OK;
}

void RendererInstance::drop_graphs() {
  for (auto& g : graphs_) {
    if (g.head) cudaGraphExecDestroy(static_cast<cudaGraphExec_t>(g.head));
    if (g.tail) cudaGraphExecDestroy(static_cast<cudaGraphExec_t>(g.tail));
    g = FrameGraph();
  }
}

// Captures one half of the frame into an executable graph.  `body` enqueues on stream_.  On any failure the capture is ended,
// graphs are switched off for this renderer and the caller falls back to eager launches.
template <typename Body>
int RendererInstance::capture(void** exec_out, Body body) {
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  *exec_out = nullptr;
  if (cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); return OXC_E_CUDA; }
  const int rc = body();
  cudaGraph_t graph = nullptr;
  const cudaError_t e = cudaStreamEndCapture(s, &graph);
  if (rc != OXC_OK || e != cudaSuccess || !graph) {
    if (graph) cudaGraphDestroy(graph);
    cudaGetLastError();
    return rc != OXC_OK ? rc : OXC_E_CUDA;
  }
  cudaGraphExec_t exec = nullptr;
  const cudaError_t ei = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ei != cudaSuccess) { cudaGetLastError(); return OXC_E_CUDA; }
  *exec_out = exec;
  return OXC_OK;
}

auto RendererInstance::render(const OxcCullCamera& camera, const float* occluder_depth_host, uint32_t* vis32_host,
                              float* depth_host, uint32_t* visible_indices_host, uint32_t visible_indices_capacity,
                              OxrFrameResult* result) -> int {
  if (!ctx_ || !error_.empty()) return OXC_E_STATE;
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  const size_t px = (size_t)width_ * height_;
  int rc;
  OxcOutputs out;
  if ((rc = oxc_get_outputs(ctx_, &out)) != OXC_OK) return fail(rc);
  Readback* rb = static_cast<Readback*>(h_pinned_);
  if ((rc = oxc_bind_camera_buffer(ctx_, nullptr)) != OXC_OK) return fail(rc); // the graph path may have left a device camera bound
  if ((rc = run_frame(camera, occluder_depth_host, rb, false)) != OXC_OK) return fail(rc);

  // results back to the host (the engine would hand the attachments to decode_visbuffer, :923-925)
  if (vis32_host || depth_host) {
    if ((rc = oxc_resolve_visbuffer(ctx_, d_vis64_, width_, height_, vis32_host ? d_vis32_ : nullptr,
                                    depth_host ? d_depth_ : nullptr, s)) != OXC_OK) return fail(rc);
    if (vis32_host && cudaMemcpyAsync(vis32_host, d_vis32_, px * 4, cudaMemcpyDeviceToHost, s) != cudaSuccess) return fail(OXC_E_CUDA);
    if (depth_host && cudaMemcpyAsync(depth_host, d_depth_, px * 4, cudaMemcpyDeviceToHost, s) != cudaSuccess) return fail(OXC_E_CUDA);
  }
  if (cudaMemcpyAsync(&rb->visibility, out.visibility, sizeof rb->visibility, cudaMemcpyDeviceToHost, s) != cudaSuccess) return fail(OXC_E_CUDA);
  if (cudaMemcpyAsync(&rb->raster_triangles, out.raster_triangle_count, 8, cudaMemcpyDeviceToHost, s) != cudaSuccess) return fail(OXC_E_CUDA);
  if (cudaStreamSynchronize(s) != cudaSuccess) {
    error_ = cudaGetErrorString(cudaGetLastError());
    return OXC_E_CUDA;
  }
  if (visible_indices_host) {
    uint32_t n = rb->visibility.early_visible_meshlet_instances + rb->visibility.late_visible_meshlet_instances;
    if (n > visible_indices_capacity) n = visible_indices_capacity;
    if (n && cudaMemcpy(visible_indices_host, out.visible_meshlet_instances_indices, (size_t)n * 4, cudaMemcpyDeviceToHost) != cudaSuccess)
      return fail(OXC_E_CUDA);
  }
  if (result) {
    result->visibility = rb->visibility;
    result->draw_index_count_early = rb->draw_index_count[0];
    result->draw_index_count_late = rb->draw_index_count[1];
    result->raster_triangles = rb->raster_triangles;
  }
  return OXC_OK;
}

auto RendererInstance::submit(const OxcCullCamera& camera, uint32_t* vis32_host, float* depth_host,
                              uint32_t* visible_indices_host, uint32_t visible_indices_capacity, int* ticket) -> int {
  if (!ctx_ || !error_.empty() || !ticket) return OXC_E_STATE;
  const int slot = (int)(frame_ & 1);
  Slot& sl = slots_[slot];
  if (sl.in_flight) {
    error_ = "oxr_submit: the previous frame of this slot has not been waited";
    return OXC_E_STATE;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  int rc;
  OxcOutputs out;
  if ((rc = oxc_get_outputs(ctx_, &out)) != OXC_OK) return fail(rc);
  // The compute stream carries no device->host copy: counters are staged device-side like the images and every D2H
  // goes out on the copy stream (flush_pending_copy).
  Readback* dc = static_cast<Readback*>(sl.d_counters);
  if (g_trace.on) {
    if (!g_trace.ev[slot][0])
      for (int k = 0; k < 4; k++) cudaEventCreate(&g_trace.ev[slot][k]);
    if (!g_trace.have_base) { cudaEventCreate(&g_trace.base); cudaEventRecord(g_trace.base, s); g_trace.have_base = true; }
    cudaEventRecord(g_trace.ev[slot][0], s);
    g_trace.cur_slot = slot;
    g_trace.n_stage = 0;
  }
  const bool want_vis32 = vis32_host != nullptr, want_depth = depth_host != nullptr;
  const uint32_t n_ids = visible_indices_host ? (visible_indices_capacity < ids_capacity_ ? visible_indices_capacity : ids_capacity_) : 0;
  // Steady state: both halves of the frame replay from CUDA graphs (one pair per slot).  The camera reaches the kernels through
  // a device buffer (oxc_bind_camera_buffer) that the head graph fills from this slot's pinned copy, so a replay only needs the
  // new camera written there.  Everything else a graph bakes in is part of its key; a mismatch re-captures.
  bool done = false;
  // The terrain cull and draw take the camera by value (they never read the bound device camera), so a frame with a terrain is
  // enqueued eagerly: a replayed graph would draw the terrain from the camera it was captured with.
  if (use_graphs_ && !g_trace.on && !terrain_.set && out.reordered_indices == nullptr && d_cam_[slot] && h_cam_[slot]) {
    FrameGraph& g = graphs_[slot];
    const uint32_t key = (has_external_depth_ ? 1u : 0u) | (want_vis32 ? 2u : 0u) | (want_depth ? 4u : 0u);
    *static_cast<OxcCullCamera*>(h_cam_[slot]) = camera;
    if ((rc = oxc_bind_camera_buffer(ctx_, static_cast<const OxcCullCamera*>(d_cam_[slot]))) != OXC_OK) return fail(rc);
    if (!g.head || !g.tail || g.key != key || g.n_ids != n_ids || g.mesh_instance_count != camera.mesh_instance_count) {
      if (g.head) cudaGraphExecDestroy(static_cast<cudaGraphExec_t>(g.head));
      if (g.tail) cudaGraphExecDestroy(static_cast<cudaGraphExec_t>(g.tail));
      g = FrameGraph();
      int rc_a = capture(&g.head, [&]() -> int {
        const int r = oxc_load_camera(ctx_, static_cast<OxcCullCamera*>(d_cam_[slot]), static_cast<const OxcCullCamera*>(h_cam_[slot]), s);
        return r != OXC_OK ? r : frame_head(camera, nullptr, dc, true);
      });
      int rc_b = rc_a == OXC_OK ? capture(&g.tail, [&]() -> int {
        const int r = frame_tail(camera, dc);
        return r != OXC_OK ? r : stage_results(slot, want_vis32, want_depth, n_ids);
      }) : rc_a;
      if (rc_a != OXC_OK || rc_b != OXC_OK) { // capture is not available here: eager launches from now on
        drop_graphs();
        use_graphs_ = false;
      } else {
        g.key = key; g.n_ids = n_ids; g.mesh_instance_count = camera.mesh_instance_count;
      }
    }
    if (use_graphs_) {
      if (cudaGraphLaunch(static_cast<cudaGraphExec_t>(g.head), s) != cudaSuccess) return fail(OXC_E_CUDA);
      if (pending_.active && (rc = flush_pending_copy(true)) != OXC_OK) return fail(rc);
      if (cudaGraphLaunch(static_cast<cudaGraphExec_t>(g.tail), s) != cudaSuccess) return fail(OXC_E_CUDA);
      done = true;
    }
  }
  if (!done) {
    if ((rc = oxc_bind_camera_buffer(ctx_, nullptr)) != OXC_OK) return fail(rc);
    if ((rc = run_frame(camera, nullptr, dc, true)) != OXC_OK) return fail(rc);
    if ((rc = stage_results(slot, want_vis32, want_depth, n_ids)) != OXC_OK) return fail(rc);
  }
  if (cudaEventRecord(static_cast<cudaEvent_t>(sl.ev_compute), s) != cudaSuccess) return fail(OXC_E_CUDA);
  // the device -> host copies are issued later, from inside the next frame (or by wait()): see PendingCopy
  if (g_trace.on) cudaEventRecord(g_trace.ev[slot][1], s);
  pending_.active = true;
  pending_.slot = slot;
  pending_.vis32_host = vis32_host;
  pending_.depth_host = depth_host;
  pending_.ids_host = visible_indices_host;
  pending_.n_ids = n_ids;
  sl.in_flight = true;
  *ticket = slot;
  frame_++;
  return OXC_OK;
}

// Enqueues the device->host copies of the pending frame on the copy stream.  behind_window: called from inside the next
// frame after its early cull was launched — the copies then also wait for that point of the compute stream.
int RendererInstance::flush_pending_copy(bool behind_window) {
  if (!pending_.active) return OXC_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream_), cs = static_cast<cudaStream_t>(copy_stream_);
  Slot& sl = slots_[pending_.slot];
  const size_t px = (size_t)width_ * height_;
  const int slot = pending_.slot;
  pending_.active = false;
  if (behind_window) {
    if (cudaEventRecord(static_cast<cudaEvent_t>(ev_window_), s) != cudaSuccess) return OXC_E_CUDA;
    if (cudaStreamWaitEvent(cs, static_cast<cudaEvent_t>(ev_window_), 0) != cudaSuccess) return OXC_E_CUDA;
  }
  if (cudaStreamWaitEvent(cs, static_cast<cudaEvent_t>(sl.ev_compute), 0) != cudaSuccess) return OXC_E_CUDA;
  if (g_trace.on) cudaEventRecord(g_trace.ev[slot][2], cs);
  if (cudaMemcpyAsync(sl.h_readback, sl.d_counters, sizeof(Readback), cudaMemcpyDeviceToHost, cs) != cudaSuccess) return OXC_E_CUDA;
  if (pending_.vis32_host && cudaMemcpyAsync(pending_.vis32_host, sl.d_vis32, px * 4, cudaMemcpyDeviceToHost, cs) != cudaSuccess) return OXC_E_CUDA;
  if (pending_.depth_host && cudaMemcpyAsync(pending_.depth_host, sl.d_depth, px * 4, cudaMemcpyDeviceToHost, cs) != cudaSuccess) return OXC_E_CUDA;
  if (pending_.n_ids && cudaMemcpyAsync(pending_.ids_host, sl.d_ids, (size_t)pending_.n_ids * 4, cudaMemcpyDeviceToHost, cs) != cudaSuccess)
    return OXC_E_CUDA;
  if (g_trace.on) cudaEventRecord(g_trace.ev[slot][3], cs);
  if (cudaEventRecord(static_cast<cudaEvent_t>(sl.ev_copy), cs) != cudaSuccess) return OXC_E_CUDA;
  return OXC_OK;
}

auto RendererInstance::wait(int ticket, OxrFrameResult* result) -> int {
  if (ticket < 0 || ticket > 1) return OXC_E_INVALID;
  Slot& sl = slots_[ticket];
  if (!sl.in_flight) return OXC_E_STATE;
  if (pending_.active && pending_.slot == ticket) { // nobody submitted a frame after this one: send its results now
    const int rc = flush_pending_copy(false);
    if (rc != OXC_OK) return fail(rc);
  }
  if (cudaEventSynchronize(static_cast<cudaEvent_t>(sl.ev_copy)) != cudaSuccess) {
    error_ = cudaGetErrorString(cudaGetLastError());
    return OXC_E_CUDA;
  }
  sl.in_flight = false;
  if (g_trace.on && g_trace.ev[ticket][0]) {
    float t[4];
    for (int k = 0; k < 4; k++) cudaEventElapsedTime(&t[k], g_trace.base, g_trace.ev[ticket][k]);
    std::fprintf(stderr, "[oxr trace] slot %d: start %.3f  compute_end %.3f  copy_start %.3f  copy_end %.3f ms | stages us:", ticket, t[0], t[1], t[2], t[3]);
    float prev_t = t[0];
    for (int k = 0; k < 8 && g_trace.stage[ticket][k]; k++) {
      float st;
      if (cudaEventElapsedTime(&st, g_trace.base, g_trace.stage[ticket][k]) != cudaSuccess) break;
      std::fprintf(stderr, " %.0f", (st - prev_t) * 1e3f);
      prev_t = st;
    }
    std::fprintf(stderr, " | tail %.0f\n", (t[1] - prev_t) * 1e3f);
  }
  if (result) {
    const Readback* rb = static_cast<const Readback*>(sl.h_readback);
    result->visibility = rb->visibility;
    result->draw_index_count_early = rb->draw_index_count[0];
    result->draw_index_count_late = rb->draw_index_count[1];
    result->raster_triangles = rb->raster_triangles;
  }
  return OXC_OK;
}

} // namespace ox

// ---- C exports ----
struct OxrRenderer {
  ox::RendererInstance impl;
  OxrRenderer(int device, const OxcCreateInfo& info, uint32_t w, uint32_t h) : impl(device, info, w, h) {}
};

extern "C" {

int oxr_create(int device, const OxcCreateInfo* info, uint32_t width, uint32_t height, OxrRenderer** out) {
  if (!info || !out || !width || !height) return OXC_E_INVALID;
  *out = nullptr;
  OxrRenderer* r = new (std::nothrow) OxrRenderer(device, *info, width, height);
  if (!r) return OXC_E_INVALID;
  if (!r->impl.ok()) {
    const int rc = r->impl.context() ? OXC_E_CUDA : OXC_E_NO_DEVICE;
    delete r;
    return rc;
  }
  *out = r;
  return OXC_OK;
}

void oxr_destroy(OxrRenderer* r) { delete r; }

OxcContext* oxr_context(OxrRenderer* r) { return r ? r->impl.context() : nullptr; }

int oxr_update(OxrRenderer* r, const OxcSceneDesc* scene) {
  if (!r || !scene) return OXC_E_INVALID;
  ox::RendererInstanceUpdateInfo info;
  info.mesh_instance_count = scene->mesh_instance_count;
  info.scene = *scene;
  int rc = r->impl.update(info);
  if (rc == OXC_OK && cudaStreamSynchronize(static_cast<cudaStream_t>(r->impl.stream())) != cudaSuccess) rc = OXC_E_CUDA;
  return rc;
}

int oxr_update_transforms(OxrRenderer* r, const OxcTransformWorld* transforms, uint32_t first, uint32_t count) {
  if (!r || !transforms) return OXC_E_INVALID;
  return r->impl.update_transforms(transforms, first, count);
}

int oxr_overdraw(OxrRenderer* r, const OxcCullCamera* camera, uint32_t* overdraw_host) {
  if (!r || !camera) return OXC_E_INVALID;
  return r->impl.overdraw(*camera, overdraw_host);
}

int oxr_set_materials(OxrRenderer* r, const OxcMaterialTable* table) {
  if (!r) return OXC_E_INVALID;
  return r->impl.set_materials(table);
}

int oxr_set_terrain(OxrRenderer* r, const uint16_t* heightmap_host, uint32_t res_x, uint32_t res_y, const float* patch_minmax_host,
                    const OxcTerrainDrawSettings* settings) {
  if (!r) return OXC_E_INVALID;
  return r->impl.set_terrain(heightmap_host, res_x, res_y, patch_minmax_host, settings);
}

int oxr_set_external_depth(OxrRenderer* r, const float* depth_host) {
  if (!r) return OXC_E_INVALID;
  return r->impl.set_external_depth(depth_host);
}

int oxr_submit(OxrRenderer* r, const OxcCullCamera* camera, uint32_t* vis32_host, float* depth_host,
               uint32_t* visible_indices_host, uint32_t visible_indices_capacity, int* ticket) {
  if (!r || !camera || !ticket) return OXC_E_INVALID;
  return r->impl.submit(*camera, vis32_host, depth_host, visible_indices_host, visible_indices_capacity, ticket);
}

int oxr_wait(OxrRenderer* r, int ticket, OxrFrameResult* result) {
  if (!r) return OXC_E_INVALID;
  return r->impl.wait(ticket, result);
}

int oxr_vsm_update_pages(OxrRenderer* r, const OxrVsmPageContext* context) {
  if (!r || !context) return OXC_E_INVALID;
  ox::VsmPageContext c = *context;
  return r->impl.update_virtual_shadow_pages(c);
}

int oxr_vsm_pages(OxrRenderer* r, OxrVsmPages* out) {
  if (!r) return OXC_E_INVALID;
  return r->impl.virtual_shadow_pages(out);
}

int oxr_vsm_draw_shadows(OxrRenderer* r, const OxcCullCamera* coarse) {
  if (!r || !coarse) return OXC_E_INVALID;
  return r->impl.draw_virtual_shadows(*coarse);
}

int oxr_vsm_resolve_shadows(OxrRenderer* r, const OxcCullCamera* camera, float* shadow_host) {
  if (!r || !camera) return OXC_E_INVALID;
  return r->impl.resolve_shadowmap(*camera, shadow_host);
}

int oxr_decode_gbuffer(OxrRenderer* r, const OxcCullCamera* camera, float* albedo_host, float* normal_host, float* emissive_host,
                       float* metallic_roughness_occlusion_host) {
  if (!r || !camera) return OXC_E_INVALID;
  return r->impl.decode_visbuffer(*camera, albedo_host, normal_host, emissive_host, metallic_roughness_occlusion_host);
}

int oxr_generate_ambient_occlusion(OxrRenderer* r, const OxcCullCamera* camera, const OxcGtaoCamera* gtao_camera, const OxcGtaoSettings* settings,
                                   float* ao_host) {
  if (!r || !camera || !gtao_camera || !settings) return OXC_E_INVALID;
  return r->impl.generate_ambient_occlusion(*camera, *gtao_camera, *settings, ao_host);
}

int oxr_apply_pbr(OxrRenderer* r, const OxcCullCamera* camera, const OxcPbrCamera* pbr_camera, const OxcPbrSettings* settings,
                  const OxcLight* lights_host, int cast_shadows, const OxcGtaoCamera* gtao_camera, const OxcGtaoSettings* gtao_settings,
                  float* rgba_host) {
  if (!r || !camera || !pbr_camera || !settings) return OXC_E_INVALID;
  // HasContactShadows needs the contact-shadow pass's camera and settings: oxr_apply_pbr_with_contact_shadows takes them
  if (settings->scene_flags & OXC_SCENE_HAS_CONTACT_SHADOWS) return OXC_E_INVALID;
  return r->impl.apply_pbr(*camera, *pbr_camera, *settings, lights_host, cast_shadows != 0, gtao_camera, gtao_settings, rgba_host);
}

int oxr_apply_pbr_atmosphere(OxrRenderer* r, const OxcCullCamera* camera, const OxcPbrCamera* pbr_camera, const OxcPbrSettings* settings,
                             const OxcAtmosphere* atmosphere, const OxcLight* lights_host, int cast_shadows, const OxcGtaoCamera* gtao_camera,
                             const OxcGtaoSettings* gtao_settings, const OxcContactShadowCamera* contact_camera,
                             const OxcContactShadowSettings* contact_settings, float* rgba_host) {
  if (!r || !camera || !pbr_camera || !settings || !atmosphere) return OXC_E_INVALID;
  return r->impl.apply_pbr(*camera, *pbr_camera, *settings, lights_host, cast_shadows != 0, gtao_camera, gtao_settings, rgba_host, contact_camera,
                           contact_settings, atmosphere);
}

int oxr_atmosphere_luts(OxrRenderer* r, const OxcAtmosphere* atmosphere, const OxcPbrCamera* camera, const float sun_direction[3],
                        float sun_intensity, uint16_t* transmittance_host, uint16_t* sky_view_host, uint16_t* aerial_perspective_host) {
  if (!r || !atmosphere || !camera || !sun_direction) return OXC_E_INVALID;
  return r->impl.atmosphere_luts(*atmosphere, *camera, sun_direction, sun_intensity, transmittance_host, sky_view_host, aerial_perspective_host);
}

int oxr_atmosphere_sky_ibl(OxrRenderer* r, const OxcAtmosphere* atmosphere, const OxcPbrCamera* camera, const float sun_direction[3],
                           float sun_intensity, uint16_t* cube_host) {
  if (!r || !atmosphere || !camera || !sun_direction) return OXC_E_INVALID;
  return r->impl.atmosphere_sky_ibl(*atmosphere, *camera, sun_direction, sun_intensity, cube_host);
}

int oxr_eye_adaptation(OxrRenderer* r, const OxcEyeAdaptationSettings* settings, float delta_time, OxcExposure* exposure_host) {
  if (!r || !settings) return OXC_E_INVALID;
  return r->impl.eye_adaptation(*settings, delta_time, exposure_host);
}

int oxr_bloom(OxrRenderer* r, const OxcBloomSettings* settings, float* bloom_host) {
  if (!r || !settings) return OXC_E_INVALID;
  return r->impl.bloom(*settings, bloom_host);
}

int oxr_tonemap(OxrRenderer* r, const OxcTonemapSettings* settings, float* rgba_host) {
  if (!r || !settings) return OXC_E_INVALID;
  return r->impl.tonemap(*settings, rgba_host);
}

int oxr_fxaa(OxrRenderer* r, float* rgba_host) {
  if (!r) return OXC_E_INVALID;
  return r->impl.fxaa(rgba_host);
}

int oxr_contact_shadows(OxrRenderer* r, const OxcContactShadowCamera* contact_camera, const OxcContactShadowSettings* settings,
                        float* contact_host) {
  if (!r || !contact_camera || !settings) return OXC_E_INVALID;
  return r->impl.contact_shadows(*contact_camera, *settings, contact_host);
}

int oxr_apply_pbr_with_contact_shadows(OxrRenderer* r, const OxcCullCamera* camera, const OxcPbrCamera* pbr_camera, const OxcPbrSettings* settings,
                                       const OxcLight* lights_host, int cast_shadows, const OxcGtaoCamera* gtao_camera,
                                       const OxcGtaoSettings* gtao_settings, const OxcContactShadowCamera* contact_camera,
                                       const OxcContactShadowSettings* contact_settings, float* rgba_host) {
  if (!r || !camera || !pbr_camera || !settings) return OXC_E_INVALID;
  return r->impl.apply_pbr(*camera, *pbr_camera, *settings, lights_host, cast_shadows != 0, gtao_camera, gtao_settings, rgba_host, contact_camera,
                           contact_settings);
}

int oxr_render(OxrRenderer* r, const OxcCullCamera* camera, const float* occluder_depth_host, uint32_t* vis32_host,
               float* depth_host, uint32_t* visible_indices_host, uint32_t visible_indices_capacity, OxrFrameResult* result) {
  if (!r || !camera) return OXC_E_INVALID;
  return r->impl.render(*camera, occluder_depth_host, vis32_host, depth_host, visible_indices_host, visible_indices_capacity, result);
}

} // extern "C"
