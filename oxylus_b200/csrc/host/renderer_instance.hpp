// renderer_instance.hpp — host-side mirror of the reference's frame builder for the visibility path.
//
// Mirrors (same names, argument meaning and sequencing):
//   ox::RendererInstance::update              Oxylus/src/Render/RendererInstance.cpp:1333-1788
//   ox::RendererInstance::cull_geometry       Oxylus/src/Render/Passes/CullGeometry.cpp:61-404
//   ox::RendererInstance::generate_hiz        Oxylus/src/Render/Passes/CullGeometry.cpp:10-59
//   ox::RendererInstance::draw_for_visbuffer  Oxylus/src/Render/Passes/DrawGeometry.cpp:104-190
//   the geometry section of ::render          Oxylus/src/Render/RendererInstance.cpp:768-926
// The vuk::Value<Buffer|ImageAttachment> futures of the reference's context structs become plain device
// pointers owned by this object; "recording a pass" becomes enqueuing liboxcull kernels on one stream.
#pragma once
#include <cstdint>
#include <initializer_list>
#include <string>
#include <vector>

#include "../../../include/oxcull.h"

namespace ox {

// RendererInstance.hpp:171-196
struct CullGeometryContext {
  bool use_hiz = false;
  bool use_hpb = false;          // VSM page-bitmap path: out of scope (SURVEY §8f.4); multi-view cull instead
  bool init_cull_meshes = false; // run cull_meshes (allocates / zeroes visibility + dispatch buffers)
  uint32_t cull_flags = OXC_CULL_TEST_ALL;
  OxcCullCamera cull_camera = {};
  bool materialize_indices = false; // also run cull_triangles -> reordered_indices + draw cmd (reference stage 3)
};

// RendererInstance.hpp:198-216 (attachments this path touches)
struct MainGeometryContext {
  uint32_t cull_flags = OXC_CULL_TEST_ALL;
  OxcCullCamera cull_camera = {};
  uint64_t* visbuffer_attachment = nullptr; // packed depth|data image (device), width x height
  uint32_t width = 0, height = 0;
};

// RMVSMContext's per-frame inputs (RendererInstance.hpp:259-280 with the clipmaps calculate_virtual_shadow_matrices produced,
// Shadowmaps.cpp:9-63, and the frame's dirty mesh instances, RendererInstance.cpp:1704-1716)
using VsmPageContext = OxrVsmPageContext;

// Scene.cpp:1280-1290 RendererInstanceUpdateInfo (the fields this path consumes)
struct RendererInstanceUpdateInfo {
  uint32_t mesh_instance_count = 0;
  uint32_t max_meshlet_instance_count = 0;
  OxcSceneDesc scene = {};
};

class RendererInstance {
public:
  RendererInstance(int device, const OxcCreateInfo& info, uint32_t width, uint32_t height);
  ~RendererInstance();
  RendererInstance(const RendererInstance&) = delete;
  RendererInstance& operator=(const RendererInstance&) = delete;

  bool ok() const { return ctx_ != nullptr && error_.empty(); }
  const std::string& error() const { return error_; }
  OxcContext* context() const { return ctx_; }
  void* stream() const { return stream_; }

  auto update(const RendererInstanceUpdateInfo& info) -> int;
  // dirty-range transform upload (RendererInstance.cpp:16-109,1590-1599); async on the renderer's stream
  auto update_transforms(const OxcTransformWorld* transforms, uint32_t first, uint32_t count) -> int;
  // depth laid down by passes outside this path (terrain): kept on the device until replaced; nullptr clears it
  auto set_materials(const OxcMaterialTable* table) -> int; // nullptr: plain encode
  auto overdraw(const OxcCullCamera& camera, uint32_t* overdraw_host) -> int; // fragment counter of the last rendered frame
  auto set_external_depth(const float* depth_host) -> int;
  // the terrain of RendererInstance::render (Passes/Terrain.cpp:159-277): uploads the R16 heightmap (res_x x res_y), the patch min / max
  // (float2 per patch) and the settings, and owns the visible-patch list, the draw command and the persistent patch mask; with a
  // terrain set, both geometry passes run the terrain cull and draw after the meshlet raster.  heightmap_host == nullptr removes it.
  auto set_terrain(const uint16_t* heightmap_host, uint32_t res_x, uint32_t res_y, const float* patch_minmax_host,
                   const OxcTerrainDrawSettings* settings) -> int;
  auto cull_geometry(CullGeometryContext& context) -> int;
  auto generate_hiz(MainGeometryContext& context) -> int;
  auto draw_for_visbuffer(MainGeometryContext& context) -> int;
  // draw_virtual_shadowmap's page loop (Shadowmaps.cpp:100-430) up to the shadow raster, from the depth of the last frame
  auto update_virtual_shadow_pages(VsmPageContext& context) -> int;
  auto virtual_shadow_pages(OxrVsmPages* out) const -> int;
  // draw_virtual_shadowmap's last step (Shadowmaps.cpp:433-754): cull_geometry with use_hpb for the coarse camera, then the shadow
  // casters into the dirty pages of the atlas, from the clipmaps, flags and table of the last update_virtual_shadow_pages.  Runs on
  // a context of its own, so the camera frame's survivors, counters and mask are never touched.
  auto draw_virtual_shadows(const OxcCullCamera& coarse) -> int;
  // resolve_shadowmap (Shadowmaps.cpp:756-822): decode the last frame's normals, then the PCSS shadow factor per pixel from the pages,
  // clipmaps and atlas of the last update_virtual_shadow_pages; width x height floats to the host
  auto resolve_shadowmap(const OxcCullCamera& camera, float* shadow_host) -> int;
  // the vis decode pass (visbuffer_decode.slang:88-183) on the last rendered frame: albedo, normal, emissive and metallic / roughness /
  // occlusion planes (float4 per pixel; any host pointer may be null) with the table of the last set_materials
  auto decode_visbuffer(const OxcCullCamera& camera, float* albedo_host, float* normal_host, float* emissive_host, float* mro_host) -> int;
  // generate_ambient_occlusion (PBR.cpp:143-311) on the last rendered frame: decode its normals into the plane resolve_shadowmap uses,
  // then the three GTAO passes on its depth; width x height floats to the host
  auto generate_ambient_occlusion(const OxcCullCamera& camera, const OxcGtaoCamera& gtao_camera, const OxcGtaoSettings& settings, float* ao_host)
      -> int;
  // apply_pbr (PBR.cpp:435-531, no atmosphere) on the last rendered frame, with the G-buffer decode, the shadow resolve (cast_shadows)
  // and the GTAO (HasGTAO) before it, all from the G-buffer's normal plane, and the contact shadows (HasContactShadows, both contact
  // arguments required then) between the resolve and the GTAO, as the reference orders them; width x height float4 to the host
  auto apply_pbr(const OxcCullCamera& camera, const OxcPbrCamera& pbr_camera, const OxcPbrSettings& settings, const OxcLight* lights_host,
                 bool cast_shadows, const OxcGtaoCamera* gtao_camera, const OxcGtaoSettings* gtao_settings, float* rgba_host,
                 const OxcContactShadowCamera* contact_camera = nullptr, const OxcContactShadowSettings* contact_settings = nullptr,
                 const OxcAtmosphere* atmosphere = nullptr) -> int;
  // with a record (apply_pbr_atmosphere, PBR.cpp:312-432): the settings must carry HasAtmosphere and HasDirectionalLight; the per-frame
  // LUTs and the cube update run first (RendererInstance.cpp:1022, as atmosphere_sky_ibl), then the chain above, then the atmospheric pass
  // the contact_shadows pass (RendererInstance.cpp:990-1020) on the last rendered frame's depth; width x height floats to the host
  auto contact_shadows(const OxcContactShadowCamera& contact_camera, const OxcContactShadowSettings& settings, float* contact_host) -> int;
  // the atmosphere's LUTs (RendererInstance.cpp:203-226 bake with the default record, once; PBR.cpp:11-50 and :96-140 per call with
  // the caller's record at the renderer's extents); each non-null host pointer receives its binary16 RGBA plane
  auto atmosphere_luts(const OxcAtmosphere& atmosphere, const OxcPbrCamera& camera, const float sun_direction[3], float sun_intensity,
                       uint16_t* transmittance_host, uint16_t* sky_view_host, uint16_t* aerial_perspective_host) -> int;
  // the per-frame LUTs as atmosphere_luts makes them, then the sky IBL cube (PBR.cpp:52-94) into the renderer's persistent cube with
  // sun_ambient_strength 0.15 and frame_index = the number of earlier calls; the cube (binary16 RGBA, 48 KiB) to the host when non-null
  auto atmosphere_sky_ibl(const OxcAtmosphere& atmosphere, const OxcPbrCamera& camera, const float sun_direction[3], float sun_intensity,
                          uint16_t* cube_host) -> int;
  // eye adaptation (PostProcess.cpp:7-77) on the post chain's source (post_source_), into the renderer's persistent exposure
  // record ((1, 1) at allocation, as the reference's vuk::fill); the record to the host when non-null
  auto eye_adaptation(const OxcEyeAdaptationSettings& settings, float delta_time, OxcExposure* exposure_host) -> int;
  // bloom (PostProcess.cpp:79-203) of the post chain's source into the renderer's two chains, reading the record under HasEyeAdaptation;
  // upsampled level 0 ((width / 2) x (height / 2) float4) to the host when non-null
  auto bloom(const OxcBloomSettings& settings, float* bloom_host) -> int;
  // the tonemap (PostProcess.cpp:205-247) of the post chain's source into the renderer's tonemap plane, reading the record under
  // HasEyeAdaptation and upsampled level 0 of the bloom chain under HasBloom; width x height float4 to the host when non-null
  auto tonemap(const OxcTonemapSettings& settings, float* rgba_host) -> int;
  // FXAA (RendererInstance.cpp:1225-1255) of the lit plane of the last successful apply_pbr into the renderer's FXAA plane, which
  // becomes the post chain's source; width x height float4 to the host when non-null
  auto fxaa(float* rgba_host) -> int;

  // RendererInstance::render geometry section: run_geometry_pass(false) -> generate_hiz -> run_geometry_pass(true)
  auto render(const OxcCullCamera& camera, const float* occluder_depth_host, uint32_t* vis32_host, float* depth_host,
              uint32_t* visible_indices_host, uint32_t visible_indices_capacity, OxrFrameResult* result) -> int;

  // Pipelined variant: submit() enqueues the frame and the device->host copies of its results (on a copy stream,
  // from double-buffered staging) and returns a ticket without waiting; wait(ticket) blocks until that frame's
  // outputs are in the caller's host buffers.  At most two frames in flight; a ticket must be waited before
  // its slot is reused (submit returns OXC_E_STATE otherwise).  Survivor ids: the full capacity is copied
  // (the count is only known on the device when the copy is enqueued).
  auto submit(const OxcCullCamera& camera, uint32_t* vis32_host, float* depth_host, uint32_t* visible_indices_host,
              uint32_t visible_indices_capacity, int* ticket) -> int;
  auto wait(int ticket, OxrFrameResult* result) -> int;

private:
  int fail(int rc);
  // allocates `bytes` at *p unless *p is set.  The passes' planes are optional parts: without room for one the camera path stays
  // usable, so a failed allocation clears the CUDA error, leaves *p null and returns OXC_E_CAPACITY without setting the sticky error
  template <typename T> int optional_plane(T** p, size_t bytes);
  // the copies whose host pointer is set, device to host on stream_, then the end of the stream: OXC_OK, else the sticky OXC_E_CUDA
  struct HostCopy { void* host; const void* dev; size_t bytes; };
  int copy_to_host(std::initializer_list<HostCopy> copies);
  int run_frame(const OxcCullCamera& camera, const float* occluder_depth_host, void* readback_draw_counts, bool readback_on_device);
  int frame_head(const OxcCullCamera& camera, const float* occluder_depth_host, void* readback_draw_counts, bool readback_on_device);
  int frame_tail(const OxcCullCamera& camera, void* readback_draw_counts);
  int stage_results(int slot, bool want_vis32, bool want_depth, uint32_t n_ids);
  template <typename Body> int capture(void** exec_out, Body body);
  void drop_graphs();
  int flush_pending_copy(bool behind_window);
  // submit(): the two halves of a frame as executable CUDA graphs, one pair per slot (OXR_NO_GRAPH=1 disables)
  struct FrameGraph {
    void* head = nullptr;
    void* tail = nullptr;
    uint32_t key = 0, n_ids = 0, mesh_instance_count = 0;
  } graphs_[2];
  void* d_cam_[2] = {nullptr, nullptr}; // device camera the graph's kernels read (oxc_bind_camera_buffer)
  void* h_cam_[2] = {nullptr, nullptr}; // pinned source of the head graph's camera upload
  bool use_graphs_ = true;
  struct Slot {
    uint32_t* d_vis32 = nullptr;
    float* d_depth = nullptr;
    uint32_t* d_ids = nullptr;
    void* d_counters = nullptr;  // device staging of the frame's counters (Readback layout)
    void* h_readback = nullptr; // pinned
    void* ev_compute = nullptr;
    void* ev_copy = nullptr;
    bool in_flight = false;
  } slots_[2];
  // Device->host copies of the last submitted frame, not yet enqueued.  They are issued from inside the NEXT frame,
  // right after its early cull has been launched (or by wait(), whichever comes first): a copy-engine transfer running
  // while the many short kernels at the head of a frame are being launched lengthens their latency, whereas it is free next
  // to the one long early-raster kernel (OXR_TRACE=1 shows the timeline).
  struct PendingCopy {
    bool active = false;
    int slot = 0;
    uint32_t* vis32_host = nullptr;
    float* depth_host = nullptr;
    uint32_t* ids_host = nullptr;
    uint32_t n_ids = 0;
  } pending_;
  void* ev_window_ = nullptr;
  void* copy_stream_ = nullptr;
  uint64_t frame_ = 0;
  uint32_t ids_capacity_ = 0;
  OxcContext* ctx_ = nullptr;
  void* stream_ = nullptr;
  uint32_t width_ = 0, height_ = 0;
  uint64_t* d_vis64_ = nullptr;
  uint32_t* d_vis32_ = nullptr;
  float* d_depth_ = nullptr;
  float* d_occluder_ = nullptr;
  uint32_t* d_overdraw_ = nullptr; // allocated by the first overdraw()
  float* d_gbuffer_ = nullptr;      // four float4 planes of decode_visbuffer, allocated by its first call
  float* d_uv_normal_ = nullptr;    // uv_normal plane (float4 per pixel) the shadow resolve and the GTAO decode into, allocated by the
                                    // first of them; kept for the renderer's lifetime
  void* d_gtao_ = nullptr;          // generate_ambient_occlusion's planes (mips, edges, noisy and final occlusion), allocated by its first call
  size_t gtao_mip_texels() const;   // texels of the five depth mips at the renderer's extent
  // the device parts of decode_visbuffer, resolve_shadowmap and generate_ambient_occlusion, enqueued on stream_ without a copy; the
  // two last read the given normal plane (oct(world normal) in .zw)
  int decode_gbuffer_device(const OxcCullCamera& camera, const OxcGBufferTargets& targets);
  int resolve_shadowmap_device(const float* normals);
  int generate_ambient_occlusion_device(const OxcGtaoCamera& gtao_camera, const OxcGtaoSettings& settings, const float* normals,
                                        OxcGtaoTargets* targets);
  float* d_pbr_ = nullptr;          // apply_pbr's output plane (float4 per pixel), allocated by its first call
  float* d_contact_ = nullptr;      // the contact-shadow plane (f32 per pixel), allocated by the first call that runs the pass
  // the frame's depth, then the contact-shadow pass into d_contact_, enqueued on stream_ without a copy
  int contact_shadows_device(const OxcContactShadowCamera& contact_camera, const OxcContactShadowSettings& settings);
  // the atmosphere's LUTs at the reference's extents in one block (renderer_instance.cpp: lut_planes), allocated by the first
  // atmosphere_luts; the transmittance LUT is baked once, with the default record
  uint16_t* d_atmosphere_ = nullptr;
  bool transmittance_baked_ = false;
  // the bake when missing and the per-frame LUTs on stream_, without a copy
  int atmosphere_luts_device(const OxcAtmosphere& atmosphere, const OxcPbrCamera& camera, const float sun_direction[3], float sun_intensity);
  uint16_t* d_sky_ibl_cube_ = nullptr; // the sky IBL cube, allocated and zeroed by the first atmosphere_sky_ibl
  uint32_t sky_ibl_calls_ = 0;         // atmosphere_sky_ibl calls so far: the frame_index of the next one
  // the plane eye_adaptation, bloom and tonemap read: d_pbr_ after a successful apply_pbr, d_fxaa_ after a successful fxaa (the
  // reference's final_attachment); null before the first successful apply_pbr
  const float* post_source_ = nullptr;
  uint32_t* d_post_ = nullptr;         // the eye-adaptation histogram (256 u32), then the exposure record, from the first eye_adaptation
  float* d_bloom_ = nullptr;           // bloom's downsampled chain, then its upsampled chain, from the first bloom
  bool bloomed_ = false;               // d_bloom_ holds the chains of a successful bloom
  float* d_tonemap_ = nullptr;         // the tonemap's output plane (float4 per pixel), from the first tonemap
  float* d_fxaa_ = nullptr;            // FXAA's output plane (float4 per pixel), from the first fxaa
  int sky_ibl_device(const OxcAtmosphere& atmosphere, const OxcPbrCamera& camera, const float sun_direction[3], float sun_intensity);
  OxcLight* d_lights_ = nullptr;    // apply_pbr's lights buffer (OXC_MAX_LIGHTS records), allocated with d_pbr_
  bool has_external_depth_ = false;
  // the terrain of set_terrain (device copies and the cull's buffers); the frame runs terrain_pass when `set`
  struct Terrain {
    bool set = false;
    uint16_t* d_heightmap = nullptr;
    uint32_t res_x = 0, res_y = 0;
    float* d_minmax = nullptr;
    uint32_t* d_visible = nullptr;
    uint32_t* d_mask = nullptr;
    OxcDrawIndirectCommand* d_cmd = nullptr;
    OxcTerrainDrawSettings settings{};
  } terrain_;
  void terrain_release();
  // run_geometry_pass's terrain half (RendererInstance.cpp:864-880): cull with TestFrustum | TestOcclusion (| LatePass), then draw
  int terrain_pass(const OxcCullCamera& camera, bool late);
  // transforms as the host last uploaded them, and on the device the values before the upload that last changed each of them
  // (TransformPrevious::previous_world, RendererInstance.cpp:1600-1609)
  std::vector<OxcTransformWorld> transforms_;
  OxcTransformWorld* d_transforms_previous_ = nullptr;
  uint32_t transforms_previous_capacity_ = 0;
  // virtual shadow map state (RendererInstance.hpp:259-280 vsm_* attachments, Shadowmaps.cpp:100-128 transient buffers)
  struct Vsm {
    OxrVsmPages pages{};
    OxcVsmContext shape{};
    uint32_t* d_dirty_instances = nullptr;
    uint32_t dirty_capacity = 0;
    bool updated = false;                // update_virtual_shadow_pages has run with this shape
    OxcVirtualClipmap clipmaps[10] = {}; // of the last update
    float inv_projection_view[16] = {};  // of the last update
    float resolution[2] = {};
    float* d_shadow = nullptr;           // the resolve's output, allocated by its first call
  } vsm_;
  // the shadow draw's own context (same scene, transforms and materials as ctx_; max_views >= 10 for the clipmap cull)
  OxcContext* shadow_ctx_ = nullptr;
  void drop_shadow_context();
  int vsm_allocate(const OxcVsmContext& vsm, uint32_t hpb_levels);
  void vsm_release();
  void* h_pinned_ = nullptr; // staging for small readbacks
  std::string error_;
};

} // namespace ox
