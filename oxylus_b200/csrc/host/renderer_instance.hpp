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
  auto cull_geometry(CullGeometryContext& context) -> int;
  auto generate_hiz(MainGeometryContext& context) -> int;
  auto draw_for_visbuffer(MainGeometryContext& context) -> int;

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
  bool has_external_depth_ = false;
  void* h_pinned_ = nullptr; // staging for small readbacks
  std::string error_;
};

} // namespace ox
