// oxcull.cu — liboxcull.so: context management and the C ABI of include/oxcull.h.
// Every entry point enqueues hand-written sm_90a kernels (kernels_*.cuh) on the caller's stream.
// There is no CPU fallback: without a CUDA device oxc_create fails with OXC_E_NO_DEVICE.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include <dlfcn.h>
#include <nccl.h> // types only: the library is dlopen'ed by oxc_mgpu_init (single-GPU hosts never need it)

#include "kernels_cull.cuh"
#include "kernels_decode.cuh"
#include "kernels_hiz.cuh"
#include "kernels_mgpu.cuh"
#include "kernels_tri.cuh"
#include "kernels_alpha.cuh"
#include "kernels_vsm.cuh"
#include "kernels_vsm_draw.cuh"
#include "kernels_vsm_resolve.cuh"
#include "kernels_gtao.cuh"
#include "kernels_pbr.cuh"
#include "kernels_contact_shadows.cuh"

using namespace oxc;

namespace {

thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof g_err, fmt, ap);
  va_end(ap);
  return code;
}

#define CK(expr)                                                                                      \
  do {                                                                                                \
    cudaError_t e_ = (expr);                                                                          \
    if (e_ != cudaSuccess) return fail(OXC_E_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

#define LAUNCHED()                                                                                    \
  do {                                                                                                \
    g_launches.fetch_add(1, std::memory_order_relaxed);                                               \
    cudaError_t e_ = cudaGetLastError();                                                              \
    if (e_ != cudaSuccess) return fail(OXC_E_CUDA, "kernel launch: %s (%s:%d)", cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

__global__ void k_rebase_meshes(OxcMesh* meshes, uint32_t n, uint64_t base) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  OxcMesh m = meshes[i];
  m.vertex_positions += base;
  if (m.vertex_normals) m.vertex_normals += base;  // 0 = the mesh has none (Mesh::vertex_normals == nullptr)
  if (m.texture_coords) m.texture_coords += base;  // 0 = none (scene.slang:354-356,390-392)
  m.lods += base;
  OxcMeshLOD* lods = reinterpret_cast<OxcMeshLOD*>(m.lods);
  for (uint32_t l = 0; l < m.lod_count && l < OXC_MESH_MAX_LODS; l++) {
    OxcMeshLOD d = lods[l];
    d.indices += base;
    d.meshlets += base;
    d.meshlet_bounds += base;
    d.local_triangle_indices += base;
    d.indirect_vertex_indices += base;
    lods[l] = d;
  }
  meshes[i] = m;
}

__global__ void k_set_cmd3(OxcDispatchIndirectCommand* c, uint32_t x, uint32_t y, uint32_t z) { c->x = x; c->y = y; c->z = z; }
__global__ void k_reset_draw_cmd(OxcDrawIndexedIndirectCommand* c) {
  c->index_count = 0; c->instance_count = 1; c->first_index = 0; c->vertex_offset = 0; c->first_instance = 0;
}
__global__ void k_reset_visibility(OxcMeshletInstanceVisibility* v, OxcDispatchIndirectCommand* c) {
  v->total_visible_meshlet_instances = 0; v->early_visible_meshlet_instances = 0; v->late_visible_meshlet_instances = 0;
  c->x = 0; c->y = 1; c->z = 1;
}

// debug: both half decoders over all 65536 inputs (tests/test_gpu_parity.py::test_dequantize_half_all_inputs)
__global__ void k_debug_dequantize(float* canonical, float* hw) {
  const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h < 65536u) { canonical[h] = dequantize_half(h); hw[h] = dequantize_half_hw(h); }
}

uint32_t ilog2(uint32_t v) { uint32_t r = 0; while ((1u << r) < v) r++; return r; }
bool is_pow2(uint32_t v) { return v && !(v & (v - 1)); }

} // namespace

struct OxcContext {
  int device = 0;
  int sm_count = 0;
  OxcCreateInfo info{};
  // scene tables (device)
  OxcMesh* d_meshes = nullptr;
  OxcMeshInstance* d_mesh_instances = nullptr;
  OxcTransformWorld* d_transforms = nullptr;
  uint8_t* d_blob = nullptr;
  uint32_t mesh_count = 0, mesh_instance_count = 0, transform_count = 0;
  uint32_t mesh_cap = 0, transform_cap = 0;
  uint64_t blob_cap = 0;
  bool scene_set = false;
  // per-instance caches
  InstCull* d_inst = nullptr;
  InstGeom* d_geom = nullptr;
  uint32_t* d_counts = nullptr;
  uint32_t* d_block_sums = nullptr;
  float* d_lod_aabb = nullptr; // [mesh_cap][OXC_MESH_MAX_LODS][6]
  // frame buffers
  OxcMeshletInstance* d_meshlet_instances = nullptr;
  uint2* d_slabs = nullptr; // (mesh instance, meshlet) of every 32nd meshlet instance
  uint32_t* d_visible = nullptr;
  uint32_t* d_mask = nullptr;
  uint32_t mask_words = 0;
  OxcMeshletInstanceVisibility* d_vis = nullptr;
  OxcDispatchIndirectCommand* d_cull_meshlets_cmd = nullptr;
  OxcDispatchIndirectCommand* d_cull_triangles_cmd = nullptr;
  OxcDrawIndexedIndirectCommand* d_draw_cmd = nullptr;
  uint32_t* d_reordered = nullptr;
  unsigned long long* d_tri_counter = nullptr;
  uint32_t* d_raster_work = nullptr;
  uint4* d_big_queue = nullptr;      // deferred large triangles of the raster (kernels_tri.cuh)
  uint32_t* d_big_counters = nullptr;
  uint32_t big_capacity = 0;
  uint32_t* d_clip_queue = nullptr;  // triangles the plain raster rules drop (clipped by k_raster_clip_queue)
  uint32_t* d_clip_counter = nullptr;
  uint32_t clip_capacity = 1u << 20;
  // hiz
  float* d_hiz = nullptr;
  HizDesc hiz{};
  uint32_t hiz_total = 0;
  // camera the InstCull cache was built for
  OxcCullCamera cached_cam{};
  bool cache_valid = false;
  // shard
  uint32_t shard_first = 0, shard_count = 0xFFFFFFFFu;
  const uint32_t* id_base = nullptr;
  uint32_t* d_id_base_auto = nullptr; // id base computed locally by oxc_cull_meshes (oxc_set_shard_auto)
  bool id_base_auto = false;
  // multiview
  InstPlanes* d_view_planes = nullptr;
  uint32_t* d_view_bits = nullptr;
  uint32_t* d_view_counts = nullptr;
  InstView* d_inst_views = nullptr; // shadow-clipmap cull: [max_views][max_mesh_instances]
  // launch shapes
  int occ_cull[2][2][2] = {};
  bool hiz_zero = true; // the pyramid holds the cleared (all-zero) image: lets the early pass skip the Hi-Z fetches
  int occ_tri = 1, occ_raster = 1, occ_mv = 1;
  bool hpb_smem_opt_in = false;
  // multi-GPU (oxc_mgpu_*)
  struct Mgpu {
    bool active = false, own_comm = false, peer_hiz = false;
    uint32_t rank = 0, world = 1, capacity = 0;
    ncclComm_t comm = nullptr;
    uint32_t* xbuf = nullptr;         // [2][hw*hh] exchange texels + [2][MGPU_MAX_RANKS] flags (one cudaMalloc: one IPC handle)
    size_t xbuf_words = 0;
    void* peer_base[MGPU_MAX_RANKS] = {};
    MgpuPeers peers{};
    uint32_t* d_seq = nullptr;
    unsigned long long timeout_ns = 30000000000ull; // how long a rank waits for its peers' Hi-Z flags (OXC_MGPU_TIMEOUT_MS)
    uint32_t* cnt_stage[2] = {nullptr, nullptr};
    uint32_t* ids_stage[2] = {nullptr, nullptr};
    uint32_t* cnt_all[2] = {nullptr, nullptr};
    uint32_t* ids_all[2] = {nullptr, nullptr};
  } mg;
  const OxcCullCamera* cam_dev = nullptr; // oxc_bind_camera_buffer
  uint32_t* d_status = nullptr;   // sticky OXC_STATUS_* bits raised by kernels
  std::vector<uint64_t> id_prefix; // [I + 1] prefix sums of the largest-LOD meshlet count per mesh instance (host side)
  uint64_t scene_id_bound = 0;    // upper bound of the GLOBAL meshlet-instance id range (sum over all mesh instances of the largest LOD)
  uint32_t prim_bits = OXC_VIS_PRIMITIVE_BITS; // triangle bits of the vis-buffer word (8 = reference, 6 = wide_ids)
  // alpha-tested discard (oxc_set_materials): device material table, the two survivor lists of a raster pass and their counters
  AlphaMaterial* d_alpha_materials = nullptr;
  uint32_t alpha_material_count = 0;
  bool alpha_active = false;           // at least one material has an albedo image
  uint32_t* d_alpha_lists = nullptr;   // [2][max_meshlet_instances]: opaque, alpha-tested
  uint8_t* d_alpha_cmd = nullptr;      // 64 B: opaque cmd @0, alpha-tested cmd @16, an all-zero visibility record @32
  // the G-buffer decode's table from the same oxc_set_materials: GBufMaterial[count], then GBufImage[count][GB_SLOTS]
  uint8_t* d_gbuf_table = nullptr;
  size_t gbuf_table_bytes = 0;
  uint32_t gbuf_material_count = 0;    // 0: no table set
  std::string gbuf_error;              // the first image or sampler of the table the decode cannot read (oxc_decode_gbuffer refuses)
  // VSM shadow draw (oxc_vsm_draw_pages): page bitmap, first pixel per page, work queue, counters; allocated by the first call
  uint32_t* d_vsm_bitmap = nullptr;
  int* d_vsm_first_px = nullptr;
  uint4* d_vsm_queue = nullptr;
  uint32_t* d_vsm_counters = nullptr;
  size_t vsm_bitmap_words = 0, vsm_first_px_cap = 0;
  uint32_t vsm_queue_capacity = VSM_DRAW_QUEUE; // work items; beyond it the lane that finds an item draws it
};

namespace {

void mgpu_release(OxcContext* c); // defined with the oxc_mgpu_* entry points

template <typename T>
int dalloc(T** p, size_t n) {
  *p = nullptr;
  if (n == 0) n = 1;
  CK(cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)));
  return OXC_OK;
}

// Grid of a persistent kernel: blocks_per_sm CTAs per SM (one when the occupancy query found none), but no more CTAs than
// max_meshlet_instances / items_per_block, and at least one.
uint32_t persistent_grid(const OxcContext* c, uint32_t items_per_block, int blocks_per_sm) {
  const uint32_t tiles = (c->info.max_meshlet_instances + items_per_block - 1) / items_per_block;
  const uint32_t grid = std::min((uint32_t)(c->sm_count * (blocks_per_sm > 0 ? blocks_per_sm : 1)), tiles);
  return grid ? grid : 1u;
}

// Grid of a 256-thread grid-stride kernel over n items: one CTA per 256 items, at most 8 per SM, at least one.
uint32_t capped_grid(const OxcContext* c, size_t n) {
  const size_t grid = std::min((n + 255) / 256, (size_t)c->sm_count * 8);
  return grid ? (uint32_t)grid : 1u;
}

int check_vis_id_bits(const OxcContext* c) {
  if (c->scene_id_bound > (1ull << (32u - c->prim_bits)))
    return fail(OXC_E_CAPACITY, "the scene can emit %llu meshlet instances: ids overflow the %u id bits of the vis-buffer word (visbuffer.slang:9-10)%s",
                (unsigned long long)c->scene_id_bound, 32u - c->prim_bits, c->info.wide_ids ? "" : "; create the context with wide_ids = 1 (26 + 6 bit packing)");
  return OXC_OK;
}

void shard_range(const OxcContext* c, uint32_t cam_count, uint32_t* first, uint32_t* count) {
  uint32_t n = cam_count < c->mesh_instance_count ? cam_count : c->mesh_instance_count; // cull_meshes.slang:28
  uint32_t lo = c->shard_first < n ? c->shard_first : n;
  uint32_t hi = n;
  if (c->shard_count != 0xFFFFFFFFu && (uint64_t)c->shard_first + c->shard_count < hi) hi = c->shard_first + c->shard_count;
  if (hi < lo) hi = lo;
  *first = lo;
  *count = hi - lo;
}

// meshlet instances the mesh instances [first, first + count) can emit at most (count 0xFFFFFFFF = to the end)
uint64_t shard_need(const std::vector<uint64_t>& prefix, uint32_t first, uint32_t count) {
  if (prefix.empty()) return 0;
  const uint64_t n = prefix.size() - 1;
  const uint64_t lo = first < n ? first : n;
  uint64_t hi = n;
  if (count != 0xFFFFFFFFu && (uint64_t)first + count < hi) hi = (uint64_t)first + count;
  if (hi < lo) hi = lo;
  return prefix[hi] - prefix[lo];
}

// oxc_set_shard / oxc_set_shard_auto (automatic: oxc_cull_meshes computes the id base into d_id_base_auto; id_base is ignored)
int set_shard(OxcContext* c, uint32_t first, uint32_t count, const uint32_t* id_base, bool automatic) {
  if (!c) return fail(OXC_E_INVALID, "null context");
  if (c->scene_set && shard_need(c->id_prefix, first, count) > c->info.max_meshlet_instances)
    return fail(OXC_E_CAPACITY, "mesh instances [%u, +%u) can emit %llu meshlet instances > max_meshlet_instances %u", first, count,
                (unsigned long long)shard_need(c->id_prefix, first, count), c->info.max_meshlet_instances);
  c->shard_first = first; c->shard_count = count; c->id_base = automatic ? c->d_id_base_auto : id_base; c->id_base_auto = automatic;
  c->cache_valid = false;
  return OXC_OK;
}

bool same_camera(const OxcCullCamera& a, const OxcCullCamera& b) {
  return memcmp(a.projection_view, b.projection_view, sizeof a.projection_view) == 0 &&
         memcmp(a.position, b.position, sizeof a.position) == 0;
}

// (re)build InstCull for `cam` without touching LOD selection / counts.  bound_camera: the kernel reads a camera bound with
// oxc_bind_camera_buffer instead of `cam` (the main view's passes); the shadow-clipmap cull passes false, since its coarse view
// is never the bound frame camera
int refresh_inst_cache(OxcContext* c, const OxcCullCamera* cam, cudaStream_t s, bool bound_camera = true) {
  if (c->cache_valid && same_camera(c->cached_cam, *cam)) return OXC_OK;
  if (!c->cache_valid) return fail(OXC_E_STATE, "oxc_cull_meshes must run before the meshlet/triangle passes");
  MeshesParams p{};
  p.meshes = c->d_meshes; p.mesh_instances = c->d_mesh_instances; p.transforms = c->d_transforms;
  p.inst = c->d_inst; p.geom = c->d_geom; p.counts = c->d_counts; p.block_sums = c->d_block_sums; p.lod_aabb = c->d_lod_aabb;
  shard_range(c, c->cached_cam.mesh_instance_count, &p.first, &p.count);
  p.flags = 0; p.select = 0; p.cam = *cam; p.cam_dev = bound_camera ? c->cam_dev : nullptr;
  if (p.count) {
    k_cull_meshes<<<(p.count + CULL_MESHES_THREADS - 1) / CULL_MESHES_THREADS, CULL_MESHES_THREADS, 0, s>>>(p);
    LAUNCHED();
  }
  const uint32_t keep = c->cached_cam.mesh_instance_count;
  c->cached_cam = *cam;
  c->cached_cam.mesh_instance_count = keep;
  return OXC_OK;
}

} // namespace

extern "C" {

const char* oxc_last_error(void) { return g_err; }
uint64_t oxc_kernel_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
const char* oxc_version(void) { return "oxcull 0.1 (sm_90a)"; }

int oxc_create(int device, const OxcCreateInfo* info, OxcContext** out_ctx) {
  if (!info || !out_ctx) return fail(OXC_E_INVALID, "null argument");
  *out_ctx = nullptr;
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
    cudaGetLastError();
    return fail(OXC_E_NO_DEVICE, "no CUDA device: liboxcull has no CPU fallback");
  }
  if (device < 0 || device >= n_dev) return fail(OXC_E_INVALID, "device %d out of range (%d devices)", device, n_dev);
  if (!is_pow2(info->hiz_width) || !is_pow2(info->hiz_height))
    return fail(OXC_E_INVALID, "hiz extent must be a power of two per axis (RendererInstance.cpp:573-577)");
  if (info->max_views > OXC_MAX_VIEWS) return fail(OXC_E_INVALID, "max_views > %d", OXC_MAX_VIEWS);
  CK(cudaSetDevice(device));
  OxcContext* c = new (std::nothrow) OxcContext();
  if (!c) return fail(OXC_E_INVALID, "out of host memory");
  c->device = device;
  c->info = *info;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  c->sm_count = prop.multiProcessorCount;
  const uint32_t I = info->max_mesh_instances ? info->max_mesh_instances : 1;
  const uint32_t N = info->max_meshlet_instances ? info->max_meshlet_instances : 1;
  int rc;
#define TRY(x) if ((rc = (x)) != OXC_OK) { oxc_destroy(c); return rc; }
  TRY(dalloc(&c->d_mesh_instances, (size_t)I));
  TRY(dalloc(&c->d_inst, (size_t)I));
  TRY(dalloc(&c->d_geom, (size_t)I));
  TRY(dalloc(&c->d_counts, (size_t)I));
  TRY(dalloc(&c->d_block_sums, (size_t)(I + CULL_MESHES_THREADS - 1) / CULL_MESHES_THREADS + 1));
  TRY(dalloc(&c->d_meshlet_instances, (size_t)N + CULL_TILE)); // + one tile: slack kept from a removed bulk copy of the last tile
  TRY(dalloc(&c->d_slabs, (size_t)N / 32 + 2));
  TRY(dalloc(&c->d_visible, (size_t)N));
  c->mask_words = ((info->max_mask_bits > N ? info->max_mask_bits : N) + 31) / 32; // RendererInstance.cpp:1651
  TRY(dalloc(&c->d_mask, (size_t)c->mask_words));
  TRY(dalloc(&c->d_vis, 1));
  TRY(dalloc(&c->d_cull_meshlets_cmd, 1));
  TRY(dalloc(&c->d_cull_triangles_cmd, 1));
  TRY(dalloc(&c->d_draw_cmd, 1));
  TRY(dalloc(&c->d_tri_counter, 1));
  TRY(dalloc(&c->d_raster_work, 4)); // work counter | chunk-queue counters (2) | clip-queue counter: one 16-byte memset per raster call
  c->big_capacity = 1u << 18; // 262144 chunks x 64 B = 16 MB; overflow falls back to inline rasterisation
  if (const char* e = getenv("OXC_BIG_CAPACITY")) { // test hook: force the overflow paths
    const long v = atol(e);
    if (v >= 1 && v <= (1l << 24)) c->big_capacity = (uint32_t)v;
  }
#ifdef OXC_RASTER_STATS
  TRY(dalloc(&c->d_big_queue, (size_t)c->big_capacity * 4 + 64 + (1u << 16))); // + statistics slots + per-warp timeline records
#else
  TRY(dalloc(&c->d_big_queue, (size_t)c->big_capacity * 4 + 64 /* 128 u64 statistics slots of the OXC_RASTER_STATS build */));
#endif
  CK(cudaMemset(c->d_big_queue + (size_t)c->big_capacity * 4, 0, 1024));
  c->d_big_counters = c->d_raster_work + 1;
  if (const char* e = getenv("OXC_CLIP_CAPACITY")) { // test hook: force the overflow path
    const long v = atol(e);
    if (v >= 1 && v <= (1l << 24)) c->clip_capacity = (uint32_t)v;
  }
  TRY(dalloc(&c->d_clip_queue, (size_t)c->clip_capacity));
  if (const char* e = getenv("OXC_VSM_DRAW_CAPACITY")) { // test hook: force the VSM draw's inline path
    const long v = atol(e);
    if (v >= 1 && v <= (1l << 24)) c->vsm_queue_capacity = (uint32_t)v;
  }
  c->d_clip_counter = c->d_raster_work + 3;
  TRY(dalloc(&c->d_id_base_auto, 1));
  TRY(dalloc(&c->d_status, 1));
  c->prim_bits = info->wide_ids ? OXC_VIS_WIDE_PRIMITIVE_BITS : OXC_VIS_PRIMITIVE_BITS;
  if (info->alloc_reordered_indices) TRY(dalloc(&c->d_reordered, (size_t)N * OXC_MESHLET_MAX_PRIMITIVES * 3));
  if (info->max_views > 1) {
    TRY(dalloc(&c->d_view_planes, (size_t)I * info->max_views));
    TRY(dalloc(&c->d_view_bits, (size_t)N));
    TRY(dalloc(&c->d_view_counts, (size_t)OXC_MAX_VIEWS));
    TRY(dalloc(&c->d_inst_views, (size_t)I * info->max_views));
  }
  // Hi-Z pyramid: levels = min(floor(log2(max(w,h))) + 1, 13)  (Texture.hpp:144-146, RendererInstance.cpp:583-586)
  {
    uint32_t m = info->hiz_width > info->hiz_height ? info->hiz_width : info->hiz_height, levels = 0;
    while (m) { levels++; m >>= 1; }
    levels = levels < OXC_HIZ_MAX_LEVELS ? levels : OXC_HIZ_MAX_LEVELS;
    uint32_t off = 0;
    for (uint32_t l = 0; l < OXC_HIZ_MAX_LEVELS; l++) {
      c->hiz.level_offset[l] = off;
      if (l < levels) {
        uint32_t mw = info->hiz_width >> l, mh = info->hiz_height >> l;
        off += (mw < 1 ? 1 : mw) * (mh < 1 ? 1 : mh);
      }
    }
    c->hiz.width = info->hiz_width; c->hiz.height = info->hiz_height; c->hiz.levels = levels;
    c->hiz_total = off;
    TRY(dalloc(&c->d_hiz, (size_t)off));
    c->hiz.data = c->d_hiz;
  }
#undef TRY
  CK(cudaMemset(c->d_mask, 0, (size_t)c->mask_words * 4));
  CK(cudaMemset(c->d_hiz, 0, (size_t)c->hiz_total * 4));
  CK(cudaMemset(c->d_vis, 0, sizeof(OxcMeshletInstanceVisibility)));
  CK(cudaMemset(c->d_tri_counter, 0, 8));
  CK(cudaMemset(c->d_status, 0, 4));
  OxcDispatchIndirectCommand one{0, 1, 1};
  CK(cudaMemcpy(c->d_cull_meshlets_cmd, &one, sizeof one, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(c->d_cull_triangles_cmd, &one, sizeof one, cudaMemcpyHostToDevice));
  OxcDrawIndexedIndirectCommand dc{0, 1, 0, 0, 0};
  CK(cudaMemcpy(c->d_draw_cmd, &dc, sizeof dc, cudaMemcpyHostToDevice));
#define OCC(dst, kern, threads) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&(dst), kern, threads, 0))
#define OCCC(dst, H, O, L)                                                                                                        \
  CK(cudaFuncSetAttribute(k_cull_meshlets<H, O, L, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CullShared<O && !L>)));  \
  CK(cudaFuncSetAttribute(k_cull_meshlets<H, O, L, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CullShared<O && !L>)));   \
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&(dst), (k_cull_meshlets<H, O, L, false>), CULL_THREADS, sizeof(CullShared<O && !L>)))
  OCCC(c->occ_cull[0][0][0], false, false, false);
  OCCC(c->occ_cull[1][0][0], true, false, false);
  OCCC(c->occ_cull[1][0][1], true, false, true);
  OCCC(c->occ_cull[1][1][0], true, true, false);
  OCCC(c->occ_cull[1][1][1], true, true, true);
#undef OCCC
  c->occ_cull[0][0][1] = c->occ_cull[0][1][0] = c->occ_cull[0][1][1] = c->occ_cull[0][0][0];
  OCC(c->occ_tri, k_cull_triangles, TRI_THREADS);
  OCC(c->occ_raster, k_raster_visbuffer<false>, TRI_THREADS);
  OCC(c->occ_mv, k_cull_meshlets_multiview, CULL_THREADS);
#undef OCC
  *out_ctx = c;
  return OXC_OK;
}

void oxc_destroy(OxcContext* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->mg.active) { cudaDeviceSynchronize(); mgpu_release(c); }
  cudaFree(c->d_meshes); cudaFree(c->d_mesh_instances); cudaFree(c->d_transforms); cudaFree(c->d_blob);
  cudaFree(c->d_lod_aabb); cudaFree(c->d_inst); cudaFree(c->d_geom); cudaFree(c->d_counts); cudaFree(c->d_block_sums);
  cudaFree(c->d_meshlet_instances); cudaFree(c->d_slabs); cudaFree(c->d_visible); cudaFree(c->d_mask); cudaFree(c->d_vis);
  cudaFree(c->d_cull_meshlets_cmd); cudaFree(c->d_cull_triangles_cmd); cudaFree(c->d_draw_cmd);
  cudaFree(c->d_reordered); cudaFree(c->d_tri_counter); cudaFree(c->d_raster_work); cudaFree(c->d_big_queue); cudaFree(c->d_clip_queue); cudaFree(c->d_id_base_auto); cudaFree(c->d_status); cudaFree(c->d_hiz);
  cudaFree(c->d_view_planes); cudaFree(c->d_view_bits); cudaFree(c->d_view_counts); cudaFree(c->d_inst_views);
  cudaFree(c->d_alpha_materials); cudaFree(c->d_alpha_lists); cudaFree(c->d_alpha_cmd); cudaFree(c->d_gbuf_table);
  cudaFree(c->d_vsm_bitmap); cudaFree(c->d_vsm_first_px); cudaFree(c->d_vsm_queue); cudaFree(c->d_vsm_counters);
  delete c;
}

int oxc_set_scene(OxcContext* c, const OxcSceneDesc* sc, void* stream) {
  if (!c || !sc) return fail(OXC_E_INVALID, "null argument");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  if (sc->mesh_instance_count > c->info.max_mesh_instances)
    return fail(OXC_E_CAPACITY, "mesh_instance_count %u > max_mesh_instances %u", sc->mesh_instance_count, c->info.max_mesh_instances);
  if (sc->mesh_count == 0 || !sc->meshes || !sc->blob || !sc->transforms || (sc->mesh_instance_count && !sc->mesh_instances))
    return fail(OXC_E_INVALID, "scene tables missing");
  // Layout checks on the host tables (the kernels use 128-bit loads of Meshlet / MeshletBounds records and 64-bit
  // loads of vertex positions; a misaligned or out-of-range offset must be an error here, not a device fault later).
  // The reference's own builder aligns the meshlet / bounds tables to 8 bytes only (blob_append(..., 8),
  // AssetManager_GLTF.cpp:749-750): such tables are accepted and moved to a 16-byte aligned tail of the DEVICE copy of
  // the blob (relocated below); the caller's blob is not modified.
  struct Reloc { uint64_t lod_record, src, size; int field; };
  std::vector<Reloc> relocs;
  uint64_t reloc_bytes = 0;
  for (uint32_t m = 0; m < sc->mesh_count; m++) {
    const OxcMesh& me = sc->meshes[m];
    if (me.lod_count == 0 || me.lod_count > OXC_MESH_MAX_LODS) return fail(OXC_E_INVALID, "mesh %u: lod_count %u not in 1..%d", m, me.lod_count, OXC_MESH_MAX_LODS);
    if ((me.vertex_positions & 7u) || (me.vertex_normals & 3u) || (me.texture_coords & 3u) || (me.lods & 7u))
      return fail(OXC_E_INVALID, "mesh %u: vertex_positions / lods need 8-byte, normals / texcoords 4-byte aligned blob offsets", m);
    if (me.lods + (uint64_t)me.lod_count * sizeof(OxcMeshLOD) > sc->blob_size || me.vertex_positions + (uint64_t)me.vertex_count * 8u > sc->blob_size)
      return fail(OXC_E_INVALID, "mesh %u: offsets outside the blob", m);
    // vertex records a vertex index may address: the kernels read vertex_positions[vi] and, with a material table,
    // texture_coords[vi] without a bound.  An index >= Mesh::vertex_count whose records lie inside the blob is accepted: the
    // reference's decode pass defines its result (status 2, visbuffer_decode.slang:115-117) and the other passes read blob bytes.
    uint64_t vertex_records = (sc->blob_size - me.vertex_positions) / 8u;
    if (me.texture_coords) vertex_records = std::min(vertex_records, me.texture_coords < sc->blob_size ? (sc->blob_size - me.texture_coords) / 4u : 0);
    const OxcMeshLOD* lods = reinterpret_cast<const OxcMeshLOD*>(sc->blob + me.lods);
    for (uint32_t l = 0; l < me.lod_count; l++) {
      OxcMeshLOD d;
      memcpy(&d, &lods[l], sizeof d);
      if ((d.meshlets & 7u) || (d.meshlet_bounds & 7u) || (d.local_triangle_indices & 3u) || (d.indirect_vertex_indices & 3u))
        return fail(OXC_E_INVALID, "mesh %u lod %u: meshlets / meshlet_bounds need 8-byte, index arrays 4-byte aligned blob offsets", m, l);
      if (d.meshlets + (uint64_t)d.meshlet_count * sizeof(OxcMeshlet) > sc->blob_size ||
          d.meshlet_bounds + (uint64_t)d.meshlet_count * sizeof(OxcMeshletBounds) > sc->blob_size ||
          d.local_triangle_indices + (uint64_t)d.local_triangle_indices_count > sc->blob_size ||
          d.indirect_vertex_indices + (uint64_t)d.indirect_vertex_indices_count * 4u > sc->blob_size)
        return fail(OXC_E_INVALID, "mesh %u lod %u: arrays outside the blob", m, l);
      // Every meshlet's runs: the kernels read the vertex records of every vertex index of the (clamped) vertex run without a
      // bound, so a run outside its array or a vertex index past the blob must be an error here, not a device fault.  Micro
      // indices >= the meshlet's clamped vertex count are refused too: the kernels would skip such a triangle, but no builder
      // writes one.
      for (uint32_t k = 0; k < d.meshlet_count; k++) {
        OxcMeshlet ml;
        memcpy(&ml, sc->blob + d.meshlets + (uint64_t)k * sizeof(OxcMeshlet), sizeof ml);
        const uint32_t nv = std::min(ml.vertex_count, (uint32_t)OXC_MESHLET_MAX_VERTICES);
        const uint32_t nt = std::min(ml.triangle_count, (uint32_t)OXC_MESHLET_MAX_PRIMITIVES);
        if ((uint64_t)ml.indirect_vertex_index_offset + nv > d.indirect_vertex_indices_count)
          return fail(OXC_E_INVALID, "mesh %u lod %u meshlet %u: vertex run [%u, +%u) outside indirect_vertex_indices (%u)", m, l, k,
                      ml.indirect_vertex_index_offset, nv, d.indirect_vertex_indices_count);
        if ((uint64_t)ml.local_triangle_index_offset + 3u * nt > d.local_triangle_indices_count)
          return fail(OXC_E_INVALID, "mesh %u lod %u meshlet %u: triangle run [%u, +%u) outside local_triangle_indices (%u)", m, l, k,
                      ml.local_triangle_index_offset, 3u * nt, d.local_triangle_indices_count);
        const uint8_t* vidx = sc->blob + d.indirect_vertex_indices + (uint64_t)ml.indirect_vertex_index_offset * 4u;
        for (uint32_t v = 0; v < nv; v++) {
          uint32_t vi;
          memcpy(&vi, vidx + (uint64_t)v * 4u, 4);
          if (vi >= vertex_records)
            return fail(OXC_E_INVALID, "mesh %u lod %u meshlet %u: vertex index %u outside the blob (its vertex records hold %llu vertices)", m, l,
                        k, vi, (unsigned long long)vertex_records);
        }
        const uint8_t* micro = sc->blob + d.local_triangle_indices + ml.local_triangle_index_offset;
        for (uint32_t b = 0; b < 3u * nt; b++)
          if (micro[b] >= nv)
            return fail(OXC_E_INVALID, "mesh %u lod %u meshlet %u: micro index %u >= the meshlet's vertex count %u", m, l, k, micro[b], nv);
      }
      const uint64_t rec = me.lods + (uint64_t)l * sizeof(OxcMeshLOD);
      if (d.meshlets & 15u) { relocs.push_back({rec, d.meshlets, (uint64_t)d.meshlet_count * sizeof(OxcMeshlet), 0}); reloc_bytes += (relocs.back().size + 15u) & ~15ull; }
      if (d.meshlet_bounds & 15u) { relocs.push_back({rec, d.meshlet_bounds, (uint64_t)d.meshlet_count * sizeof(OxcMeshletBounds), 1}); reloc_bytes += (relocs.back().size + 15u) & ~15ull; }
    }
  }
  // Instance table (ADVICE r1): every index in range, and the meshlet instances / mask bits the scene can ever need fit the
  // create-time capacities — whatever LOD the mesh-level cull selects.  The reference sizes these buffers from the scene itself
  // (RendererInstance.cpp:1651-1665,1717-1732); here they are create-time capacities, so an oversized scene is an error, not a
  // device fault.  (The kernels additionally clamp and raise OXC_STATUS_MESHLET_OVERFLOW, see k_scan_block_sums.)
  uint64_t id_bound = 0;
  std::vector<uint64_t> id_prefix((size_t)sc->mesh_instance_count + 1, 0);
  {
    std::vector<uint32_t> max_lod_count(sc->mesh_count, 0);
    for (uint32_t m = 0; m < sc->mesh_count; m++) {
      const OxcMeshLOD* lods = reinterpret_cast<const OxcMeshLOD*>(sc->blob + sc->meshes[m].lods);
      for (uint32_t l = 0; l < sc->meshes[m].lod_count; l++) {
        OxcMeshLOD d;
        memcpy(&d, &lods[l], sizeof d);
        if (d.meshlet_count > max_lod_count[m]) max_lod_count[m] = d.meshlet_count;
      }
    }
    const uint64_t mask_bits = (uint64_t)c->mask_words * 32u;
    for (uint32_t i = 0; i < sc->mesh_instance_count; i++) {
      const OxcMeshInstance& mi = sc->mesh_instances[i];
      if (mi.mesh_index >= sc->mesh_count) return fail(OXC_E_INVALID, "mesh instance %u: mesh_index %u >= mesh_count %u", i, mi.mesh_index, sc->mesh_count);
      if (mi.transform_index >= sc->transform_count)
        return fail(OXC_E_INVALID, "mesh instance %u: transform_index %u >= transform_count %u", i, mi.transform_index, sc->transform_count);
      if (mi.lod_index >= sc->meshes[mi.mesh_index].lod_count)
        return fail(OXC_E_INVALID, "mesh instance %u: lod_index %u >= lod_count %u", i, mi.lod_index, sc->meshes[mi.mesh_index].lod_count);
      const uint32_t n = max_lod_count[mi.mesh_index];
      if ((uint64_t)mi.meshlet_instance_visibility_offset + n > mask_bits)
        return fail(OXC_E_CAPACITY, "mesh instance %u: visibility offset %u + %u meshlets exceeds the %llu mask bits of max_meshlet_instances %u", i,
                    mi.meshlet_instance_visibility_offset, n, (unsigned long long)mask_bits, c->info.max_meshlet_instances);
      id_bound += n;
      id_prefix[i + 1] = id_bound;
    }
    // the whole scene need not fit one context — a shard only expands its own range —, but the context's range must
    const uint64_t need = shard_need(id_prefix, c->shard_first, c->shard_count);
    if (need > c->info.max_meshlet_instances)
      return fail(OXC_E_CAPACITY, "mesh instances [%u, +%u) can emit %llu meshlet instances > max_meshlet_instances %u", c->shard_first,
                  c->shard_count, (unsigned long long)need, c->info.max_meshlet_instances);
  }
  // device copy of the blob: the caller's bytes, or (8-byte aligned tables present) a patched copy with those tables
  // appended at 16-byte aligned offsets and the MeshLOD records pointing at the copies
  const uint8_t* upload = sc->blob;
  uint64_t upload_size = sc->blob_size;
  std::vector<uint8_t> patched;
  if (!relocs.empty()) {
    uint64_t cursor = (sc->blob_size + 15u) & ~15ull;
    patched.resize((size_t)(cursor + reloc_bytes));
    memcpy(patched.data(), sc->blob, (size_t)sc->blob_size);
    for (const Reloc& r : relocs) {
      memcpy(patched.data() + cursor, sc->blob + r.src, (size_t)r.size);
      OxcMeshLOD d;
      memcpy(&d, patched.data() + r.lod_record, sizeof d);
      (r.field == 0 ? d.meshlets : d.meshlet_bounds) = cursor;
      memcpy(patched.data() + r.lod_record, &d, sizeof d);
      cursor += (r.size + 15u) & ~15ull;
    }
    upload = patched.data();
    upload_size = patched.size();
  }
  if (sc->mesh_count > c->mesh_cap) {
    CK(cudaFree(c->d_meshes)); c->d_meshes = nullptr;
    CK(cudaMalloc(&c->d_meshes, (size_t)sc->mesh_count * sizeof(OxcMesh)));
    CK(cudaFree(c->d_lod_aabb)); c->d_lod_aabb = nullptr;
    CK(cudaMalloc(&c->d_lod_aabb, (size_t)sc->mesh_count * OXC_MESH_MAX_LODS * 6 * sizeof(float)));
    c->mesh_cap = sc->mesh_count;
  }
  if (sc->transform_count > c->transform_cap) {
    CK(cudaFree(c->d_transforms)); c->d_transforms = nullptr;
    CK(cudaMalloc(&c->d_transforms, (size_t)sc->transform_count * sizeof(OxcTransformWorld)));
    c->transform_cap = sc->transform_count;
  }
  if (upload_size > c->blob_cap) {
    CK(cudaFree(c->d_blob)); c->d_blob = nullptr;
    CK(cudaMalloc(&c->d_blob, (size_t)upload_size + 64)); // + slack: the raster stages micro-index runs in whole words, so a run
    c->blob_cap = upload_size;                            //   that ends at the blob's last byte is read up to 3 bytes past it
  }
  CK(cudaMemcpyAsync(c->d_meshes, sc->meshes, (size_t)sc->mesh_count * sizeof(OxcMesh), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(c->d_mesh_instances, sc->mesh_instances, (size_t)sc->mesh_instance_count * sizeof(OxcMeshInstance), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(c->d_transforms, sc->transforms, (size_t)sc->transform_count * sizeof(OxcTransformWorld), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(c->d_blob, upload, (size_t)upload_size, cudaMemcpyHostToDevice, s));
  if (!patched.empty()) CK(cudaStreamSynchronize(s)); // the patched copy dies with this call
  // upload_gltf_mesh (AssetManager_GLTF.cpp:778-800): blob offsets -> device addresses
  k_rebase_meshes<<<(sc->mesh_count + 127) / 128, 128, 0, s>>>(c->d_meshes, sc->mesh_count, reinterpret_cast<uint64_t>(c->d_blob));
  LAUNCHED();
  {
    const uint32_t warps = sc->mesh_count * OXC_MESH_MAX_LODS;
    k_lod_union_aabb<<<(warps * 32 + 255) / 256, 256, 0, s>>>(c->d_meshes, sc->mesh_count, c->d_lod_aabb);
    LAUNCHED();
  }
  c->mesh_count = sc->mesh_count; c->mesh_instance_count = sc->mesh_instance_count; c->transform_count = sc->transform_count;
  c->scene_id_bound = id_bound;
  c->id_prefix.swap(id_prefix);
  c->scene_set = true;
  c->cache_valid = false;
  // instance table changed => zero_fill_pass on the mask (RendererInstance.cpp:1651-1665)
  CK(cudaMemsetAsync(c->d_mask, 0, (size_t)c->mask_words * 4, s));
  return OXC_OK;
}

int oxc_update_transforms(OxcContext* c, const OxcTransformWorld* t, uint32_t first, uint32_t count, void* stream) {
  if (!c || !t) return fail(OXC_E_INVALID, "null argument");
  if (!c->scene_set) return fail(OXC_E_STATE, "oxc_set_scene first");
  if ((uint64_t)first + count > c->transform_count) return fail(OXC_E_CAPACITY, "transform range out of bounds");
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(c->d_transforms + first, t, (size_t)count * sizeof(OxcTransformWorld), cudaMemcpyHostToDevice,
                     static_cast<cudaStream_t>(stream)));
  c->cache_valid = false;
  return OXC_OK;
}

int oxc_reset_visibility_mask(OxcContext* c, void* stream) {
  if (!c) return fail(OXC_E_INVALID, "null context");
  CK(cudaSetDevice(c->device));
  CK(cudaMemsetAsync(c->d_mask, 0, (size_t)c->mask_words * 4, static_cast<cudaStream_t>(stream)));
  return OXC_OK;
}

int oxc_clear_hiz(OxcContext* c, void* stream) {
  if (!c) return fail(OXC_E_INVALID, "null context");
  CK(cudaSetDevice(c->device));
  CK(cudaMemsetAsync(c->d_hiz, 0, (size_t)c->hiz_total * 4, static_cast<cudaStream_t>(stream)));
  c->hiz_zero = true;
  return OXC_OK;
}

int oxc_set_shard(OxcContext* c, uint32_t first, uint32_t count, const uint32_t* id_base_dev) { return set_shard(c, first, count, id_base_dev, false); }
int oxc_set_shard_auto(OxcContext* c, uint32_t first, uint32_t count) { return set_shard(c, first, count, nullptr, true); }

int oxc_cull_meshes(OxcContext* c, const OxcCullCamera* cam, uint32_t flags, void* stream) {
  if (!c || !cam) return fail(OXC_E_INVALID, "null argument");
  if (!c->scene_set) return fail(OXC_E_STATE, "oxc_set_scene first");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  MeshesParams p{};
  p.meshes = c->d_meshes; p.mesh_instances = c->d_mesh_instances; p.transforms = c->d_transforms;
  p.inst = c->d_inst; p.geom = c->d_geom; p.counts = c->d_counts; p.block_sums = c->d_block_sums; p.lod_aabb = c->d_lod_aabb;
  shard_range(c, cam->mesh_instance_count, &p.first, &p.count);
  p.flags = flags; p.select = 1; p.cam = *cam; p.cam_dev = c->cam_dev;
  if (c->id_base_auto) { // global id base of this shard = meshlets emitted by the mesh instances below it (no communication)
    CK(cudaMemsetAsync(c->d_id_base_auto, 0, 4, s));
    if (p.first) {
      k_count_prefix_meshlets<<<(p.first + CULL_MESHES_THREADS - 1) / CULL_MESHES_THREADS, CULL_MESHES_THREADS, 0, s>>>(p, c->d_id_base_auto);
      LAUNCHED();
    }
  }
  const uint32_t n_blocks = (p.count + CULL_MESHES_THREADS - 1) / CULL_MESHES_THREADS;
  if (n_blocks == 0) {
    k_reset_visibility<<<1, 1, 0, s>>>(c->d_vis, c->d_cull_meshlets_cmd);
    LAUNCHED();
  } else {
    k_cull_meshes<<<n_blocks, CULL_MESHES_THREADS, 0, s>>>(p);
    LAUNCHED();
    k_scan_block_sums<<<1, 1024, 0, s>>>(c->d_block_sums, n_blocks, c->d_vis, c->d_cull_meshlets_cmd, c->info.max_meshlet_instances, c->d_status);
    LAUNCHED();
    k_expand_meshlet_instances<<<n_blocks * EXPAND_SPLIT, CULL_MESHES_THREADS, 0, s>>>(c->d_counts, c->d_block_sums, p.first, p.count,
                                                                      c->d_meshlet_instances, c->info.max_meshlet_instances, c->d_slabs);
    LAUNCHED();
  }
  c->cached_cam = *cam;
  c->cache_valid = true;
  return OXC_OK;
}

int oxc_cull_meshlets(OxcContext* c, const OxcCullCamera* cam, uint32_t flags, int use_hiz, void* stream) {
  if (!c || !cam) return fail(OXC_E_INVALID, "null argument");
  if (!c->scene_set) return fail(OXC_E_STATE, "oxc_set_scene first");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  int rc = refresh_inst_cache(c, cam, s);
  if (rc != OXC_OK) return rc;
  CK(cudaMemsetAsync(&c->d_cull_triangles_cmd->x, 0, 4, s)); // CullGeometry.cpp:125-127 ({0, 1, 1}: y and z are never modified)
  CullParams p{};
  p.slabs = c->d_slabs;
  p.meshlet_instances = c->d_meshlet_instances; p.inst = c->d_inst; p.vis = c->d_vis; p.visible_indices = c->d_visible;
  p.mask = c->d_mask; p.tri_cmd = c->d_cull_triangles_cmd; p.id_base = c->id_base; p.hiz = c->hiz;
  p.cam_pos[0] = cam->position[0]; p.cam_pos[1] = cam->position[1]; p.cam_pos[2] = cam->position[2];
  p.near_clip = cam->near_clip;
  p.cam_dev = c->cam_dev;
  // the plain variant is dispatched with TestFrustum only (CullGeometry.cpp:275,298) and has no mask / late logic
  const bool hizp = use_hiz != 0;
  const bool occ = hizp && (flags & OXC_CULL_TEST_OCCLUSION) != 0;
  const bool late = hizp && (flags & OXC_CULL_LATE_PASS) != 0;
  const uint32_t grid = persistent_grid(c, CULL_THREADS, c->occ_cull[hizp][occ][late]);
#define GO(H, O, L, Z) k_cull_meshlets<H, O, L, Z><<<grid, CULL_THREADS, sizeof(CullShared<O && !L>), s>>>(p)
  const bool zero = hizp && c->hiz_zero;
  if (hizp) {
    if (occ) {
      if (late) { if (zero) GO(true, true, true, true); else GO(true, true, true, false); }
      else { if (zero) GO(true, true, false, true); else GO(true, true, false, false); }
    } else {
      if (late) { if (zero) GO(true, false, true, true); else GO(true, false, true, false); }
      else { if (zero) GO(true, false, false, true); else GO(true, false, false, false); }
    }
  } else {
    GO(false, false, false, false);
  }
#undef GO
  LAUNCHED();
  return OXC_OK;
}

static int build_hiz_impl(OxcContext* c, const float* depth_dev, uint32_t stride, uint32_t offset, uint32_t width,
                          uint32_t height, void* stream, uint32_t mode = 0) {
  if (!c || (!depth_dev && mode != 2) || ((!width || !height) && mode != 2)) return fail(OXC_E_INVALID, "bad argument");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  HizBuildParams p{};
  p.depth = depth_dev; p.elem_stride = stride; p.elem_offset = offset; p.width = width; p.height = height; p.hiz = c->d_hiz;
  p.hw = c->hiz.width; p.hh = c->hiz.height; p.levels = c->hiz.levels;
  p.hw_shift = ilog2(p.hw); p.hh_shift = ilog2(p.hh);
  p.mode = mode;
  memcpy(p.level_offset, c->hiz.level_offset, sizeof p.level_offset);
  if (p.hw % 64 == 0 && p.hh % 64 == 0) {
    k_hiz_tiles<<<dim3(p.hw / 64, p.hh / 64), 256, 0, s>>>(p);
    LAUNCHED();
    if (p.levels > 7 && mode != 1) { k_hiz_tail<<<1, 1024, 0, s>>>(p, 7); LAUNCHED(); }
  } else {
    const uint32_t n = p.hw * p.hh;
    if (mode != 2) { k_hiz_mip0_generic<<<(n + 255) / 256, 256, 0, s>>>(p); LAUNCHED(); }
    if (p.levels > 1 && mode != 1) { k_hiz_tail<<<1, 1024, 0, s>>>(p, 1); LAUNCHED(); }
  }
  c->hiz_zero = false;
  return OXC_OK;
}

int oxc_build_hiz(OxcContext* c, const float* depth_dev, uint32_t width, uint32_t height, void* stream) {
  return build_hiz_impl(c, depth_dev, 1, 0, width, height, stream);
}

// same pyramid straight from the packed 64-bit vis buffer (depth = high 32 bits, little endian): saves the
// resolve pass between the early raster and generate_hiz
int oxc_build_hiz_packed(OxcContext* c, const uint64_t* vis_dev, uint32_t width, uint32_t height, void* stream) {
  return build_hiz_impl(c, reinterpret_cast<const float*>(vis_dev), 2, 1, width, height, stream);
}

// Multi-GPU split of generate_hiz: mip 0 is a point sample, and max over ranks commutes with sampling, so ranks
// exchange only mip 0 (hw*hh floats, e.g. 4 MB at 1080p instead of the 16.6 MB packed image):
//   oxc_build_hiz_mip0_packed -> all_reduce(MAX) on the mip-0 texels -> oxc_build_hiz_from_mip0
int oxc_build_hiz_mip0_packed(OxcContext* c, const uint64_t* vis_dev, uint32_t width, uint32_t height, void* stream) {
  return build_hiz_impl(c, reinterpret_cast<const float*>(vis_dev), 2, 1, width, height, stream, 1);
}
int oxc_build_hiz_from_mip0(OxcContext* c, void* stream) { return build_hiz_impl(c, nullptr, 1, 0, 0, 0, stream, 2); }

static int tri_common(OxcContext* c, const OxcCullCamera* cam, uint32_t flags, cudaStream_t s, TriParams* p) {
  if (!c->scene_set) return fail(OXC_E_STATE, "oxc_set_scene first");
  int rc = refresh_inst_cache(c, cam, s);
  if (rc != OXC_OK) return rc;
  p->meshlet_instances = c->d_meshlet_instances; p->inst = c->d_inst; p->geom = c->d_geom; p->vis = c->d_vis;
  p->visible_indices = c->d_visible; p->tri_cmd = c->d_cull_triangles_cmd; p->id_base = c->id_base; p->late = (flags & OXC_CULL_LATE_PASS) ? 1u : 0u;
  p->reordered_indices = c->d_reordered; p->draw_cmd = c->d_draw_cmd; p->tri_counter = c->d_tri_counter;
  p->prim_bits = c->prim_bits; p->status = c->d_status; p->small_primitive_cull = 0;
  return OXC_OK;
}

// the packed image a raster pass writes, and the chunk queue its large triangles go to (k_raster_big)
static void raster_target(const OxcContext* c, uint64_t* vis, uint32_t w, uint32_t h, TriParams* p) {
  p->visbuf = reinterpret_cast<unsigned long long*>(vis); p->width = w; p->height = h; p->f_width = (float)w; p->f_height = (float)h;
  p->big_queue = c->d_big_queue; p->big_counters = c->d_big_counters; p->big_capacity = c->big_capacity;
}

// the material table of the alpha test (none when oxc_set_materials holds no alpha-tested material)
static AlphaParams alpha_materials(const OxcContext* c) {
  AlphaParams ap{};
  ap.mesh_instances = c->d_mesh_instances;
  if (c->alpha_active) { ap.materials = c->d_alpha_materials; ap.material_count = c->alpha_material_count; }
  return ap;
}

// visbuffer_encode.slang:54-66: splits the pass's survivors by material (kernels_alpha.cuh) and points *pm, what the plain
// raster walks, at the opaque part
static int split_alpha(OxcContext* c, const TriParams& p, cudaStream_t s, TriParams* pm, AlphaParams* ap) {
  *ap = alpha_materials(c);
  ap->opaque_list = c->d_alpha_lists; ap->masked_list = c->d_alpha_lists + c->info.max_meshlet_instances;
  ap->opaque_cmd = reinterpret_cast<OxcDispatchIndirectCommand*>(c->d_alpha_cmd);
  ap->masked_cmd = reinterpret_cast<OxcDispatchIndirectCommand*>(c->d_alpha_cmd + 16);
  CK(cudaMemsetAsync(c->d_alpha_cmd, 0, 64, s));
  k_partition_alpha<<<c->sm_count * 4, 256, 0, s>>>(p, *ap);
  LAUNCHED();
  pm->visible_indices = ap->opaque_list; pm->tri_cmd = ap->opaque_cmd;
  pm->vis = reinterpret_cast<const OxcMeshletInstanceVisibility*>(c->d_alpha_cmd + 32); // the list starts at 0 in either pass
  return OXC_OK;
}

static int cull_triangles_impl(OxcContext* c, const OxcCullCamera* cam, uint32_t flags, uint32_t spc, uint32_t w, uint32_t h, void* stream);

int oxc_cull_triangles(OxcContext* c, const OxcCullCamera* cam, uint32_t flags, void* stream) {
  return cull_triangles_impl(c, cam, flags, 0, 0, 0, stream);
}

int oxc_cull_triangles_small_primitive(OxcContext* c, const OxcCullCamera* cam, uint32_t flags, uint32_t width, uint32_t height, void* stream) {
  if (!width || !height) return fail(OXC_E_INVALID, "the small-primitive cull needs the raster extent");
  return cull_triangles_impl(c, cam, flags, 1, width, height, stream);
}

static int cull_triangles_impl(OxcContext* c, const OxcCullCamera* cam, uint32_t flags, uint32_t spc, uint32_t w, uint32_t h, void* stream) {
  if (!c || !cam) return fail(OXC_E_INVALID, "null argument");
  if (!c->d_reordered) return fail(OXC_E_STATE, "context created without alloc_reordered_indices");
  if (c->scene_id_bound > (1ull << (32u - OXC_VIS_PRIMITIVE_BITS)))
    return fail(OXC_E_CAPACITY, "the scene can emit %llu meshlet instances: ids overflow the %u id bits of the vis-buffer word (visbuffer.slang:9-10)%s",
                (unsigned long long)c->scene_id_bound, 24u, " (the reordered index buffer always uses the reference packing)");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  TriParams p{};
  int rc = tri_common(c, cam, flags, s, &p);
  if (rc != OXC_OK) return rc;
  p.small_primitive_cull = spc; p.width = w; p.height = h; p.f_width = (float)w; p.f_height = (float)h;
  k_reset_draw_cmd<<<1, 1, 0, s>>>(c->d_draw_cmd); // CullGeometry.cpp:380-382
  LAUNCHED();
  k_cull_triangles<<<persistent_grid(c, TRI_WARPS, c->occ_tri), TRI_THREADS, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_clear_visbuffer(OxcContext* c, uint64_t* vis, uint32_t w, uint32_t h, void* stream) {
  if (!c || !vis) return fail(OXC_E_INVALID, "null argument");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  const size_t n = (size_t)w * h;
  k_clear_visbuffer<<<c->sm_count * 8, 256, 0, s>>>(reinterpret_cast<unsigned long long*>(vis), n);
  LAUNCHED();
  CK(cudaMemsetAsync(c->d_tri_counter, 0, 8, s));
  return OXC_OK;
}

int oxc_raster_visbuffer(OxcContext* c, const OxcCullCamera* cam, uint32_t flags, uint32_t w, uint32_t h, uint64_t* vis,
                         int small_primitive_cull, void* stream) {
  if (!c || !cam || !vis) return fail(OXC_E_INVALID, "null argument");
  int rc = check_vis_id_bits(c);
  if (rc != OXC_OK) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  TriParams p{};
  rc = tri_common(c, cam, flags, s, &p);
  if (rc != OXC_OK) return rc;
  raster_target(c, vis, w, h, &p);
  p.small_primitive_cull = small_primitive_cull ? 1u : 0u;
  p.work_counter = c->d_raster_work;
  CK(cudaMemsetAsync(c->d_raster_work, 0, 16, s)); // work counter, chunk-queue counters, clip-queue counter
  const uint32_t grid = persistent_grid(c, TRI_WARPS, c->occ_raster);
  p.clip_queue = c->d_clip_queue; p.clip_counter = c->d_clip_counter; p.clip_capacity = c->clip_capacity;
  TriParams pm = p; // what the plain raster kernel walks: the pass's survivors, or their opaque part
  AlphaParams ap{};
  if (c->alpha_active) {
    rc = split_alpha(c, p, s, &pm, &ap);
    if (rc != OXC_OK) return rc;
  }
  if (p.late) k_raster_visbuffer<true><<<grid, TRI_THREADS, 0, s>>>(pm);
  else k_raster_visbuffer<false><<<grid, TRI_THREADS, 0, s>>>(pm);
  LAUNCHED();
  k_raster_clip_queue<<<c->sm_count, 128, 0, s>>>(p); // the triangles the plain rules drop (usually none: exits at once)
  LAUNCHED();
  if (c->alpha_active) {
    k_raster_alpha<false><<<c->sm_count * 8, ALPHA_THREADS, 0, s>>>(p, ap); // the alpha-tested meshlets, one warp each
    LAUNCHED();
  }
  k_raster_big<<<c->sm_count * 8, 256, 0, s>>>(p); // the deferred large triangles, one warp per <= 64x32-pixel chunk
  LAUNCHED();
  return OXC_OK;
}

// RENDER_OVERDRAW of the encode pass (visbuffer_encode.slang:15,68-70; MainGeometryContext::draw_overdraw): a separate launch of the
// general per-meshlet raster with the fragment counter as its sink — the tuned raster kernels know nothing about it
int oxc_raster_overdraw(OxcContext* c, const OxcCullCamera* cam, uint32_t flags, uint32_t w, uint32_t h, uint32_t* overdraw, int after_frame,
                        void* stream) {
  if (!c || !cam || !overdraw) return fail(OXC_E_INVALID, "null argument");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  TriParams p{};
  int rc = tri_common(c, cam, flags, s, &p);
  if (rc != OXC_OK) return rc;
  p.width = w; p.height = h; p.f_width = (float)w; p.f_height = (float)h;
  AlphaParams ap = alpha_materials(c);
  ap.overdraw = overdraw; ap.count_from_visibility = after_frame ? 1u : 0u;
  k_raster_alpha<true><<<c->sm_count * 8, ALPHA_THREADS, 0, s>>>(p, ap);
  LAUNCHED();
  return OXC_OK;
}

int oxc_clear_overdraw(OxcContext* c, uint32_t* overdraw, uint32_t w, uint32_t h, void* stream) {
  if (!c || !overdraw) return fail(OXC_E_INVALID, "null argument");
  CK(cudaSetDevice(c->device));
  CK(cudaMemsetAsync(overdraw, 0, (size_t)w * h * 4, static_cast<cudaStream_t>(stream)));
  return OXC_OK;
}

int oxc_set_materials(OxcContext* c, const OxcMaterialTable* t, void* stream) {
  if (!c) return fail(OXC_E_INVALID, "null context");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  if (!t || t->material_count == 0) { // back to the plain encode
    c->alpha_active = false;
    c->alpha_material_count = 0;
    c->gbuf_material_count = 0;
    return OXC_OK;
  }
  if (!t->materials || (t->image_count && !t->images) || (t->sampler_count && !t->samplers)) return fail(OXC_E_INVALID, "material table: null array");
  std::vector<AlphaMaterial> ms(t->material_count);
  bool any = false;
  for (uint32_t i = 0; i < t->material_count; i++) {
    const OxcMaterial& m = t->materials[i];
    AlphaMaterial& d = ms[i];
    memset(&d, 0, sizeof d);
    if (!(m.flags & OXC_MATERIAL_HAS_ALBEDO_IMAGE)) continue; // visbuffer_encode.slang:55: no image, no test
    if (m.albedo_image_index >= t->image_count)
      return fail(OXC_E_INVALID, "material %u: albedo_image_index %u outside the image table (%u)", i, m.albedo_image_index, t->image_count);
    const OxcAlphaImage& im = t->images[m.albedo_image_index];
    if (!im.texels_dev || im.width == 0 || im.height == 0 || im.width > (1u << 16) || im.height > (1u << 16) ||
        (im.format != OXC_IMAGE_RGBA8_UNORM && im.format != OXC_IMAGE_R8_UNORM && im.format != OXC_IMAGE_RGBA8_SRGB))
      return fail(OXC_E_INVALID, "image %u: null texels, extent outside 1..65536 or unknown format", m.albedo_image_index);
    uint32_t full_chain = 1;
    for (uint32_t e = im.width > im.height ? im.width : im.height; e > 1; e >>= 1) full_chain++;
    if (im.level_count > full_chain) return fail(OXC_E_INVALID, "image %u: level_count %u > %u levels of a %u x %u image", m.albedo_image_index, im.level_count, full_chain, im.width, im.height);
    d.texels = static_cast<const uint8_t*>(im.texels_dev); d.width = im.width; d.height = im.height; d.format = im.format;
    d.levels = im.level_count ? im.level_count : 1u;
    d.mag_filter = OXC_FILTER_LINEAR; d.min_filter = OXC_FILTER_LINEAR; d.mipmap_mode = OXC_MIPMAP_LINEAR; // Texture.hpp:38-45 defaults
    d.address_u = OXC_ADDRESS_REPEAT; d.address_v = OXC_ADDRESS_REPEAT;
    if (t->samplers && m.sampler_index < t->sampler_count) {
      const OxcSamplerDesc& sd = t->samplers[m.sampler_index];
      if (sd.mag_filter > OXC_FILTER_NEAREST || sd.min_filter > OXC_FILTER_NEAREST || sd.mipmap_mode > OXC_MIPMAP_NEAREST ||
          sd.address_u > OXC_ADDRESS_MIRRORED_REPEAT || sd.address_v > OXC_ADDRESS_MIRRORED_REPEAT)
        return fail(OXC_E_INVALID, "sampler %u: unknown filter / mipmap / address mode", m.sampler_index);
      d.mag_filter = sd.mag_filter; d.min_filter = sd.min_filter; d.mipmap_mode = sd.mipmap_mode;
      d.address_u = sd.address_u; d.address_v = sd.address_v;
    }
    d.albedo_a = host_dequantize_half(m.albedo_color[3]);
    const float cut = host_dequantize_half(m.alpha_cutoff);
    d.cutoff = !(cut == cut) ? cut : (cut < 0.001f ? 0.001f : (cut > 1.0f ? 1.0f : cut)); // clamp(.., 0.001, 1.0); NaN keeps everything
    any = true;
  }
  if (t->material_count > c->alpha_material_count || !c->d_alpha_materials) {
    c->alpha_active = false;
    CK(cudaStreamSynchronize(s)); // a raster in flight may still read the old table
    cudaFree(c->d_alpha_materials);
    c->d_alpha_materials = nullptr;
    if (dalloc(&c->d_alpha_materials, (size_t)t->material_count) != OXC_OK) return OXC_E_CUDA;
  }
  if (!c->d_alpha_lists) {
    if (dalloc(&c->d_alpha_lists, (size_t)c->info.max_meshlet_instances * 2) != OXC_OK) return OXC_E_CUDA;
    if (dalloc(&c->d_alpha_cmd, (size_t)64) != OXC_OK) return OXC_E_CUDA;
  }
  std::string gbuf_error;
  const std::vector<uint8_t> gb = gbuffer_table(t, &gbuf_error);
  if (gb.size() > c->gbuf_table_bytes) {
    c->gbuf_material_count = 0;
    CK(cudaStreamSynchronize(s)); // a decode in flight may still read the old table
    cudaFree(c->d_gbuf_table);
    c->d_gbuf_table = nullptr;
    c->gbuf_table_bytes = 0;
    if (dalloc(&c->d_gbuf_table, gb.size()) != OXC_OK) return OXC_E_CUDA;
    c->gbuf_table_bytes = gb.size();
  }
  CK(cudaMemcpyAsync(c->d_alpha_materials, ms.data(), ms.size() * sizeof(AlphaMaterial), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(c->d_gbuf_table, gb.data(), gb.size(), cudaMemcpyHostToDevice, s));
  CK(cudaStreamSynchronize(s)); // ms and gb are stack-owned staging copies
  c->alpha_material_count = t->material_count;
  c->alpha_active = any;
  c->gbuf_material_count = t->material_count;
  c->gbuf_error = gbuf_error;
  return OXC_OK;
}

int oxc_raster_visbuffer_clip_pass(OxcContext* c, const OxcCullCamera* cam, uint32_t flags, uint32_t w, uint32_t h, uint64_t* vis,
                                   void* stream) {
  if (!c || !cam || !vis) return fail(OXC_E_INVALID, "null argument");
  int rc = check_vis_id_bits(c);
  if (rc != OXC_OK) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  TriParams p{};
  rc = tri_common(c, cam, flags, s, &p);
  if (rc != OXC_OK) return rc;
  raster_target(c, vis, w, h, &p);
  CK(cudaMemsetAsync(c->d_big_counters, 0, 8, s));
  TriParams pm = p;
  if (c->alpha_active) { // alpha-tested meshlets clip in place (k_raster_alpha) and never depend on the queue: walk the others only
    AlphaParams ap;
    rc = split_alpha(c, p, s, &pm, &ap);
    if (rc != OXC_OK) return rc;
  }
  k_raster_clip_pass<<<persistent_grid(c, TRI_WARPS, 4), TRI_THREADS, 0, s>>>(pm);
  LAUNCHED();
  k_raster_big<<<c->sm_count * 8, 256, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_resolve_visbuffer(OxcContext* c, const uint64_t* vis, uint32_t w, uint32_t h, uint32_t* vis32, float* depth, void* stream) {
  if (!c || !vis) return fail(OXC_E_INVALID, "null argument");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  k_resolve_visbuffer<<<c->sm_count * 8, 256, 0, s>>>(reinterpret_cast<const unsigned long long*>(vis), vis32, depth, (size_t)w * h);
  LAUNCHED();
  return OXC_OK;
}

int oxc_clear_visbuffer_with_depth(OxcContext* c, uint64_t* vis, const float* depth_dev, uint32_t w, uint32_t h, void* stream) {
  if (!c || !vis || !depth_dev) return fail(OXC_E_INVALID, "null argument");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  k_clear_visbuffer_depth<<<c->sm_count * 8, 256, 0, s>>>(reinterpret_cast<unsigned long long*>(vis), depth_dev, (size_t)w * h);
  LAUNCHED();
  CK(cudaMemsetAsync(c->d_tri_counter, 0, 8, s));
  return OXC_OK;
}

// internal helper exported for the host mirror: vis = max(vis, depth<<32 | ~0u)
int oxc_merge_depth(OxcContext* c, uint64_t* vis, const float* depth_dev, uint32_t w, uint32_t h, void* stream) {
  if (!c || !vis || !depth_dev) return fail(OXC_E_INVALID, "null argument");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  k_merge_depth<<<c->sm_count * 8, 256, 0, s>>>(reinterpret_cast<unsigned long long*>(vis), depth_dev, (size_t)w * h);
  LAUNCHED();
  return OXC_OK;
}

int oxc_cull_meshlets_multiview(OxcContext* c, const OxcCullCamera* views, uint32_t n_views, int directional, void* stream) {
  if (!c || !views || n_views == 0) return fail(OXC_E_INVALID, "bad argument");
  if (n_views > c->info.max_views || !c->d_view_planes) return fail(OXC_E_CAPACITY, "n_views %u > max_views %u", n_views, c->info.max_views);
  if (!c->scene_set || !c->cache_valid) return fail(OXC_E_STATE, "oxc_cull_meshes must run first");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  ViewMatrices vm{};
  for (uint32_t v = 0; v < n_views; v++) memcpy(vm.m[v], views[v].projection_view, sizeof vm.m[v]);
  CK(cudaMemsetAsync(c->d_view_counts, 0, OXC_MAX_VIEWS * 4, s));
  uint32_t first, count;
  shard_range(c, c->cached_cam.mesh_instance_count, &first, &count);
  const uint32_t stride = c->info.max_mesh_instances;
  if (count) {
    k_prepare_view_planes<<<(count + 127) / 128, 128, 0, s>>>(c->d_mesh_instances, c->d_transforms, vm, n_views, first,
                                                             count, stride, c->d_view_planes);
    LAUNCHED();
  }
  MultiViewParams p{};
  p.meshlet_instances = c->d_meshlet_instances; p.inst = c->d_inst; p.view_planes = c->d_view_planes; p.vis = c->d_vis;
  p.view_bits = c->d_view_bits; p.view_counts = c->d_view_counts; p.n_views = n_views; p.inst_stride = stride;
  p.directional = directional;
  for (uint32_t v = 0; v < n_views; v++) {
    p.view_pos[v][0] = views[v].position[0]; p.view_pos[v][1] = views[v].position[1]; p.view_pos[v][2] = views[v].position[2];
    p.view_pos[v][3] = 0.f;
  }
  k_cull_meshlets_multiview<<<persistent_grid(c, CULL_THREADS, c->occ_mv), CULL_THREADS, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_debug_dequantize_half(OxcContext* c, float* canonical_dev, float* hw_dev, void* stream) {
  if (!c || !canonical_dev || !hw_dev) return fail(OXC_E_INVALID, "null argument");
  CK(cudaSetDevice(c->device));
  k_debug_dequantize<<<256, 256, 0, static_cast<cudaStream_t>(stream)>>>(canonical_dev, hw_dev);
  LAUNCHED();
  return OXC_OK;
}

// plumbing helpers for hosts without their own CUDA bindings (ctypes tests, bench)
int oxc_copy(OxcContext* c, void* dst, const void* src, uint64_t bytes, int kind, void* stream) {
  if (!c || (!dst && bytes) || (!src && bytes)) return fail(OXC_E_INVALID, "null argument");
  CK(cudaSetDevice(c->device));
  const cudaMemcpyKind k = kind == 0 ? cudaMemcpyHostToDevice : kind == 1 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  if (bytes) CK(cudaMemcpyAsync(dst, src, (size_t)bytes, k, static_cast<cudaStream_t>(stream)));
  return OXC_OK;
}
int oxc_sync(OxcContext* c, void* stream) {
  if (!c) return fail(OXC_E_INVALID, "null context");
  CK(cudaSetDevice(c->device));
  CK(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  return OXC_OK;
}
int oxc_device_alloc(OxcContext* c, uint64_t bytes, void** out) {
  if (!c || !out) return fail(OXC_E_INVALID, "null argument");
  CK(cudaSetDevice(c->device));
  CK(cudaMalloc(out, (size_t)(bytes ? bytes : 1)));
  return OXC_OK;
}
int oxc_device_free(OxcContext* c, void* p) {
  if (!c) return fail(OXC_E_INVALID, "null context");
  CK(cudaSetDevice(c->device));
  CK(cudaFree(p));
  return OXC_OK;
}

} // extern "C"

namespace {
// oxc_cull_meshlets_hpb (dirty flags on the host) and oxc_cull_meshlets_hpb_dirty_dev (on the device): exactly one is non-null
int cull_meshlets_hpb(OxcContext* c, const OxcCullCamera* cam, const OxcVirtualClipmap* clipmaps, const uint32_t* dirty,
                      const uint32_t* dirty_dev, uint32_t n, const uint8_t* hpb_dev, uint32_t hpb_size, uint32_t hpb_levels, void* stream) {
  if (!c || !cam || !clipmaps || !(dirty || dirty_dev) || !hpb_dev || n == 0 || hpb_size == 0) return fail(OXC_E_INVALID, "bad argument");
  if (hpb_levels == 0 || hpb_levels > 16) return fail(OXC_E_INVALID, "hpb_levels %u outside 1..16 (oxc_build_hpb's range)", hpb_levels);
  if (n > c->info.max_views || !c->d_inst_views) return fail(OXC_E_CAPACITY, "clipmap_count %u > max_views %u", n, c->info.max_views);
  if (!c->scene_set) return fail(OXC_E_STATE, "oxc_set_scene first");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  int rc = refresh_inst_cache(c, cam, s, false); // InstCull for the coarse view, from the argument even while a camera is bound
  if (rc != OXC_OK) return rc;
  ViewMatrices vm{};
  HpbParams p{};
  for (uint32_t v = 0; v < n; v++) {
    memcpy(vm.m[v], clipmaps[v].projection_view_mat, sizeof vm.m[v]);
    p.z_near[v] = clipmaps[v].z_near;
    p.page_offset[v][0] = clipmaps[v].page_offset[0]; p.page_offset[v][1] = clipmaps[v].page_offset[1];
    if (dirty && dirty[v]) p.dirty_mask |= 1u << v;
  }
  uint32_t first, count;
  shard_range(c, c->cached_cam.mesh_instance_count, &first, &count);
  const uint32_t stride = c->info.max_mesh_instances;
  if (count) {
    k_prepare_inst_views<<<(count + 127) / 128, 128, 0, s>>>(c->d_mesh_instances, c->d_transforms, vm, n, first, count, stride, c->d_inst_views);
    LAUNCHED();
  }
  k_set_cmd3<<<1, 1, 0, s>>>(c->d_cull_triangles_cmd, 0, 1, 1); // CullGeometry.cpp:125-127
  LAUNCHED();
  p.meshlet_instances = c->d_meshlet_instances; p.inst = c->d_inst; p.views = c->d_inst_views; p.vis = c->d_vis;
  p.visible_indices = c->d_visible; p.tri_cmd = c->d_cull_triangles_cmd; p.id_base = c->id_base; p.hpb = hpb_dev;
  p.hpb_size = hpb_size; p.hpb_levels = hpb_levels; p.clipmap_count = n; p.inst_stride = stride;
  p.view_dir[0] = cam->position[0]; p.view_dir[1] = cam->position[1]; p.view_dir[2] = cam->position[2];
  const uint32_t grid = persistent_grid(c, CULL_THREADS, 4);
  p.dirty_dev = dirty_dev;
  if (dirty_dev) k_cull_meshlets_hpb<true><<<grid, CULL_THREADS, 0, s>>>(p);
  else k_cull_meshlets_hpb<false><<<grid, CULL_THREADS, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}
} // namespace

extern "C" {

int oxc_cull_meshlets_hpb(OxcContext* c, const OxcCullCamera* cam, const OxcVirtualClipmap* clipmaps, const uint32_t* dirty,
                          uint32_t n, const uint8_t* hpb_dev, uint32_t hpb_size, uint32_t hpb_levels, void* stream) {
  if (!dirty) return fail(OXC_E_INVALID, "bad argument");
  return cull_meshlets_hpb(c, cam, clipmaps, dirty, nullptr, n, hpb_dev, hpb_size, hpb_levels, stream);
}

int oxc_cull_meshlets_hpb_dirty_dev(OxcContext* c, const OxcCullCamera* cam, const OxcVirtualClipmap* clipmaps, const uint32_t* dirty_dev,
                                    uint32_t n, const uint8_t* hpb_dev, uint32_t hpb_size, uint32_t hpb_levels, void* stream) {
  if (!dirty_dev) return fail(OXC_E_INVALID, "null clipmap_dirty_flags_dev");
  return cull_meshlets_hpb(c, cam, clipmaps, nullptr, dirty_dev, n, hpb_dev, hpb_size, hpb_levels, stream);
}

int oxc_cull_terrain(OxcContext* c, const OxcTerrainData* terrain, const float* patch_minmax_dev, const OxcCullCamera* cam,
                     uint32_t flags, uint32_t* visible_patches_dev, uint32_t* mask_dev, OxcDrawIndirectCommand* draw_cmd_dev, void* stream) {
  if (!c || !terrain || !patch_minmax_dev || !cam || !visible_patches_dev || !mask_dev || !draw_cmd_dev) return fail(OXC_E_INVALID, "null argument");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  TerrainParams p{};
  p.terrain = *terrain; p.patch_minmax = reinterpret_cast<const float2*>(patch_minmax_dev); p.visible_patches = visible_patches_dev;
  p.mask = mask_dev; p.draw_cmd = draw_cmd_dev; p.hiz = c->hiz; p.cam = *cam; p.flags = flags;
  k_reset_terrain_cmd<<<1, 1, 0, s>>>(draw_cmd_dev); // Terrain.cpp:168-170
  LAUNCHED();
  const uint32_t n = terrain->patch_count[0] * terrain->patch_count[1];
  if (n) { k_cull_terrain<<<(n + 255) / 256, 256, 0, s>>>(p); LAUNCHED(); }
  return OXC_OK;
}

// the geometry inputs of both decode kernels (targets left null)
static void decode_params(const OxcContext* c, const OxcCullCamera* cam, const uint64_t* vis64_dev, const uint32_t* vis32_dev, uint32_t w,
                          uint32_t h, DecodeParams* p) {
  p->vis64 = reinterpret_cast<const unsigned long long*>(vis64_dev); p->vis32 = vis32_dev;
  p->meshlet_instances = c->d_meshlet_instances; p->vis = c->d_vis; p->inst = c->d_inst; p->geom = c->d_geom; p->id_base = c->id_base;
  const float* m = cam->projection_view; // column-major: row i = (m[i], m[4+i], m[8+i], m[12+i])
  for (int i = 0; i < 4; i++) p->pv_row[i] = make_float4(m[i], m[4 + i], m[8 + i], m[12 + i]);
  p->res_x = cam->resolution[0]; p->res_y = cam->resolution[1];
  p->width = w; p->height = h; p->prim_bits = c->prim_bits;
}

int oxc_decode_visbuffer(OxcContext* c, const OxcCullCamera* cam, const uint64_t* vis64_dev, const uint32_t* vis32_dev,
                         uint32_t w, uint32_t h, const OxcDecodeTargets* t, void* stream) {
  if (!c || !cam || !t) return fail(OXC_E_INVALID, "null argument");
  if ((vis64_dev == nullptr) == (vis32_dev == nullptr)) return fail(OXC_E_INVALID, "exactly one of vis64_dev / vis32_dev");
  if (!c->scene_set) return fail(OXC_E_STATE, "oxc_set_scene first");
  int rc = check_vis_id_bits(c);
  if (rc != OXC_OK) return rc;
  if (w == 0 || h == 0) return OXC_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  rc = refresh_inst_cache(c, cam, s); // world rows / normal-matrix rows of the frame's mesh instances
  if (rc != OXC_OK) return rc;
  DecodeParams p{};
  decode_params(c, cam, vis64_dev, vis32_dev, w, h, &p);
  p.lambda = reinterpret_cast<float4*>(t->lambda); p.ddx = reinterpret_cast<float4*>(t->ddx); p.ddy = reinterpret_cast<float4*>(t->ddy);
  p.uv_normal = reinterpret_cast<float4*>(t->uv_normal); p.uv_grad = reinterpret_cast<float4*>(t->uv_grad);
  const dim3 grid((w + DECODE_TX - 1) / DECODE_TX, (h + DECODE_TY - 1) / DECODE_TY);
  k_decode_visbuffer<<<grid, dim3(DECODE_TX, DECODE_TY), 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_decode_gbuffer(OxcContext* c, const OxcCullCamera* cam, const uint64_t* vis64_dev, const uint32_t* vis32_dev, uint32_t w, uint32_t h,
                       const OxcGBufferTargets* t, void* stream) {
  if (!c || !cam || !t) return fail(OXC_E_INVALID, "null argument");
  if ((vis64_dev == nullptr) == (vis32_dev == nullptr)) return fail(OXC_E_INVALID, "exactly one of vis64_dev / vis32_dev");
  if (w == 0 || h == 0) return fail(OXC_E_INVALID, "empty extent %u x %u", w, h);
  float* const planes[4] = {t->albedo, t->normal, t->emissive, t->metallic_roughness_occlusion};
  static const char* const plane_name[4] = {"albedo", "normal", "emissive", "metallic_roughness_occlusion"};
  for (int k = 0; k < 4; k++)
    if (reinterpret_cast<uintptr_t>(planes[k]) & 15u) return fail(OXC_E_INVALID, "target %s is not 16-byte aligned (float4 per pixel)", plane_name[k]);
  if (!c->scene_set) return fail(OXC_E_STATE, "oxc_set_scene first");
  if (c->gbuf_material_count == 0) return fail(OXC_E_STATE, "oxc_set_materials first: the decode reads the material table");
  if (!c->gbuf_error.empty()) return fail(OXC_E_INVALID, "material table: %s", c->gbuf_error.c_str());
  int rc = check_vis_id_bits(c);
  if (rc != OXC_OK) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  rc = refresh_inst_cache(c, cam, s); // world rows / normal-matrix rows of the frame's mesh instances
  if (rc != OXC_OK) return rc;
  GBufferParams p{};
  decode_params(c, cam, vis64_dev, vis32_dev, w, h, &p.d);
  p.mesh_instances = c->d_mesh_instances;
  p.materials = reinterpret_cast<const GBufMaterial*>(c->d_gbuf_table);
  p.images = reinterpret_cast<const GBufImage*>(c->d_gbuf_table + (size_t)c->gbuf_material_count * sizeof(GBufMaterial));
  p.material_count = c->gbuf_material_count;
  for (int k = 0; k < 4; k++) p.want |= planes[k] ? 1u << k : 0u;
  for (int k = 0; k < 3; k++) p.cam[k] = cam->position[k];
  p.albedo = reinterpret_cast<float4*>(t->albedo); p.normal = reinterpret_cast<float4*>(t->normal);
  p.emissive = reinterpret_cast<float4*>(t->emissive); p.mro = reinterpret_cast<float4*>(t->metallic_roughness_occlusion);
  p.status = c->d_status;
  const dim3 grid((w + DECODE_TX - 1) / DECODE_TX, (h + DECODE_TY - 1) / DECODE_TY);
  k_decode_gbuffer<<<grid, dim3(DECODE_TX, DECODE_TY), 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_mark_visible_pages(OxcContext* c, const float inv_pv[16], const float resolution[2], const OxcVirtualClipmap* clipmaps,
                           const OxcVsmContext* vsm, const float* depth_dev, uint32_t* page_tables_dev, uint32_t* page_occupancy_dev,
                           uint32_t* request_count_dev, int32_t* requests_dev, uint32_t request_capacity, void* stream) {
  if (!c || !inv_pv || !resolution || !clipmaps || !vsm || !depth_dev || !page_tables_dev || !page_occupancy_dev || !request_count_dev || !requests_dev)
    return fail(OXC_E_INVALID, "null argument");
  if (vsm->clipmap_count < 1 || vsm->clipmap_count > 10 || vsm->page_table_size < 1 || vsm->depth_extent[0] < 1 || vsm->depth_extent[1] < 1)
    return fail(OXC_E_INVALID, "bad VSMContext (clipmap_count 1..10, page_table_size >= 1)");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  VsmMarkParams p{};
  vsm_fill_view(p, inv_pv, resolution, clipmaps, *vsm);
  p.depth = depth_dev; p.page_tables = page_tables_dev; p.page_occupancy = page_occupancy_dev; p.request_count = request_count_dev;
  p.requests = requests_dev; p.request_capacity = request_capacity;
  p.width = vsm->depth_extent[0]; p.height = vsm->depth_extent[1]; p.size = vsm->page_table_size; p.clipmap_count = vsm->clipmap_count;
  const dim3 grid((p.width + 31) / 32, (p.height + 7) / 8);
  k_vsm_mark_visible_pages<<<grid, 256, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_build_hpb(OxcContext* c, const uint32_t* page_table_dev, uint32_t size, uint32_t layers, uint8_t* hpb_dev, uint32_t levels,
                  void* stream) {
  if (!c || !page_table_dev || !hpb_dev) return fail(OXC_E_INVALID, "null argument");
  if (size == 0 || layers == 0 || levels == 0 || levels > 16) return fail(OXC_E_INVALID, "bad hpb shape");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  const size_t smem = (size_t)size * size + (size_t)(size / 2 + 1) * (size / 2 + 1);
  if (size <= 256) {
    if (!c->hpb_smem_opt_in && smem > 48 * 1024) { // per context == per device
      CK(cudaFuncSetAttribute(k_hpb_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
      c->hpb_smem_opt_in = true;
    }
    HpbBuildParams p{page_table_dev, hpb_dev, size, layers, levels};
    k_hpb_fused<<<layers, 1024, smem, s>>>(p);
    LAUNCHED();
    return OXC_OK;
  }
  size_t src_off = 0, dst_off = 0;
  for (uint32_t l = 0; l < levels; l++) { // Shadowmaps.cpp:338-360
    const uint32_t sl = (size >> l) ? (size >> l) : 1u, ps = l ? ((size >> (l - 1)) ? (size >> (l - 1)) : 1u) : size;
    const size_t n = (size_t)layers * sl * sl;
    k_hpb_level<<<capped_grid(c, n), 256, 0, s>>>(page_table_dev, hpb_dev + src_off, hpb_dev + dst_off, ps, sl, layers, l == 0);
    LAUNCHED();
    src_off = dst_off;
    dst_off += n;
  }
  return OXC_OK;
}

} // extern "C"

namespace {
// the OxcVsmContext checks every VSM entry point shares (include/oxcull.h); physical_page_count == UINT32_MAX: not an argument
int check_vsm(const OxcVsmContext* vsm, uint32_t physical_page_count) {
  if (vsm->clipmap_count < 1 || vsm->clipmap_count > VSM_MAX_CLIPMAPS)
    return fail(OXC_E_INVALID, "clipmap_count %d outside 1..%d (shared_clipmaps[10], rmvsm_mark_visible_pages.slang:17)", vsm->clipmap_count, VSM_MAX_CLIPMAPS);
  if (vsm->page_table_size < 1) return fail(OXC_E_INVALID, "page_table_size %d < 1", vsm->page_table_size);
  if (vsm->page_size < 1 || vsm->physical_page_table_size < 1 || vsm->physical_page_table_size % vsm->page_size != 0)
    return fail(OXC_E_INVALID, "page_size %d does not divide physical_page_table_size %d", vsm->page_size, vsm->physical_page_table_size);
  const uint64_t per_row = (uint64_t)(vsm->physical_page_table_size / vsm->page_size);
  if (per_row * per_row > 65536u)
    return fail(OXC_E_INVALID, "%llu physical pages: more than the 16-bit physical address holds (65536, rmvsm.slang:33-34)",
                (unsigned long long)(per_row * per_row));
  if ((uint64_t)vsm->clipmap_count * vsm->page_table_size * vsm->page_table_size > (1ull << 30))
    return fail(OXC_E_INVALID, "page table of %d x %d x %d entries is too large", vsm->clipmap_count, vsm->page_table_size, vsm->page_table_size);
  if (physical_page_count != 0xFFFFFFFFu && physical_page_count != per_row * per_row)
    return fail(OXC_E_INVALID, "physical_page_count %u != (physical_page_table_size / page_size)^2 = %llu", physical_page_count,
                (unsigned long long)(per_row * per_row));
  return OXC_OK;
}

uint32_t vsm_entries(const OxcVsmContext* vsm) { return (uint32_t)vsm->clipmap_count * vsm->page_table_size * vsm->page_table_size; }
} // namespace

extern "C" {

int oxc_vsm_begin_frame(OxcContext* c, const OxcVsmContext* vsm, int sun_moved, uint32_t* page_tables_dev, uint32_t* occupancy_dev,
                        uint32_t physical_page_count, uint32_t* request_count_dev, void* stream) {
  if (!c || !vsm || !page_tables_dev || !occupancy_dev || !request_count_dev) return fail(OXC_E_INVALID, "null argument");
  int rc = check_vsm(vsm, physical_page_count);
  if (rc != OXC_OK) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  const uint32_t n = std::max(vsm_entries(vsm), physical_page_count);
  k_vsm_begin_frame<<<(n + 255) / 256, 256, 0, s>>>(page_tables_dev, vsm_entries(vsm), occupancy_dev, physical_page_count, request_count_dev,
                                                    sun_moved ? 1 : 0);
  LAUNCHED();
  return OXC_OK;
}

int oxc_vsm_invalidate_pages(OxcContext* c, const OxcVsmContext* vsm, const OxcVirtualClipmap* clipmaps, const uint32_t* dirty_mesh_instances_dev,
                             uint32_t dirty_count, const OxcTransformWorld* previous_transforms_dev, uint32_t* page_tables_dev, void* stream) {
  if (!c || !vsm || !clipmaps || !dirty_mesh_instances_dev || !previous_transforms_dev || !page_tables_dev) return fail(OXC_E_INVALID, "null argument");
  int rc = check_vsm(vsm, 0xFFFFFFFFu);
  if (rc != OXC_OK) return rc;
  if (!c->scene_set) return fail(OXC_E_STATE, "oxc_set_scene first");
  if (dirty_count == 0) return OXC_OK;
  if ((uint64_t)dirty_count * vsm->clipmap_count * 2u * 32u > 0xFFFFFFFFull) return fail(OXC_E_INVALID, "dirty_count %u too large", dirty_count);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  VsmInvalidateParams p{};
  for (int k = 0; k < vsm->clipmap_count; k++) {
    memcpy(p.clip_pv[k], clipmaps[k].projection_view_mat, sizeof p.clip_pv[k]);
    p.z_near[k] = clipmaps[k].z_near;
    p.page_offset[k][0] = clipmaps[k].page_offset[0]; p.page_offset[k][1] = clipmaps[k].page_offset[1];
  }
  p.mesh_instances = c->d_mesh_instances; p.meshes = c->d_meshes; p.transforms = c->d_transforms; p.previous_transforms = previous_transforms_dev;
  p.dirty = dirty_mesh_instances_dev; p.dirty_count = dirty_count;
  p.mesh_instance_count = c->mesh_instance_count; p.mesh_count = c->mesh_count; p.transform_count = c->transform_count;
  p.page_tables = page_tables_dev; p.size = vsm->page_table_size; p.clipmap_count = vsm->clipmap_count;
  const uint64_t threads = (uint64_t)dirty_count * vsm->clipmap_count * 2u * 32u;
  k_vsm_invalidate_pages<<<(uint32_t)((threads + 255) / 256), 256, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_vsm_allocate_pages(OxcContext* c, const OxcVsmContext* vsm, uint32_t* page_tables_dev, const uint32_t* occupancy_dev,
                           uint32_t physical_page_count, const int32_t* requests_dev, uint32_t request_capacity, OxcVsmAllocator* allocator_dev,
                           uint32_t* free_list_dev, uint32_t* dirty_coords_dev, uint32_t* clipmap_dirty_flags_dev, void* stream) {
  if (!c || !vsm || !page_tables_dev || !occupancy_dev || !requests_dev || !allocator_dev || !free_list_dev || !dirty_coords_dev ||
      !clipmap_dirty_flags_dev)
    return fail(OXC_E_INVALID, "null argument");
  int rc = check_vsm(vsm, physical_page_count);
  if (rc != OXC_OK) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  VsmAllocParams p{};
  p.page_tables = page_tables_dev; p.occupancy = occupancy_dev; p.requests = requests_dev; p.allocator = allocator_dev;
  p.free_list = free_list_dev; p.dirty_coords = dirty_coords_dev; p.dirty_flags = clipmap_dirty_flags_dev;
  p.entries = vsm_entries(vsm); p.physical_page_count = physical_page_count; p.request_capacity = request_capacity;
  p.phys_per_row = (uint32_t)(vsm->physical_page_table_size / vsm->page_size); p.size = vsm->page_table_size; p.clipmap_count = vsm->clipmap_count;
  k_vsm_allocate<<<1, VSM_ALLOC_THREADS, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_vsm_clear_dirty_pages(OxcContext* c, const OxcVsmContext* vsm, const OxcVsmAllocator* allocator_dev, const uint32_t* dirty_coords_dev,
                              float* physical_atlas_dev, void* stream) {
  if (!c || !vsm || !allocator_dev || !dirty_coords_dev || !physical_atlas_dev) return fail(OXC_E_INVALID, "null argument");
  int rc = check_vsm(vsm, 0xFFFFFFFFu);
  if (rc != OXC_OK) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  VsmClearParams p{};
  p.allocator = allocator_dev; p.dirty_coords = reinterpret_cast<const uint2*>(dirty_coords_dev); p.atlas = physical_atlas_dev;
  p.page_size = (uint32_t)vsm->page_size; p.atlas_size = (uint32_t)vsm->physical_page_table_size; p.phys_per_row = p.atlas_size / p.page_size;
  p.vec4 = (p.page_size % 4u == 0u && (reinterpret_cast<uintptr_t>(physical_atlas_dev) & 15u) == 0u) ? 1 : 0;
  p.row_shift = -1;
  if (p.vec4 && is_pow2(p.page_size / 4u)) p.row_shift = (int)ilog2(p.page_size / 4u);
  // up to 8 CTAs per SM, never more than there can be dirty pages: a frame with few dirty pages costs a short, mostly idle launch
  const uint32_t pages = p.phys_per_row * p.phys_per_row;
  const uint32_t grid = std::min<uint32_t>((uint32_t)c->sm_count * 8u, pages ? pages : 1u);
  k_vsm_clear_dirty_pages<<<grid, 256, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_vsm_draw_pages(OxcContext* c, const OxcVsmContext* vsm, const OxcCullCamera* coarse, const OxcVirtualClipmap* clipmaps,
                       const uint32_t* clipmap_dirty_flags_dev, const uint32_t* page_tables_dev, float* physical_atlas_dev, void* stream) {
  if (!c || !vsm || !coarse || !clipmaps || !clipmap_dirty_flags_dev || !page_tables_dev || !physical_atlas_dev) return fail(OXC_E_INVALID, "null argument");
  int rc = check_vsm(vsm, 0xFFFFFFFFu);
  if (rc != OXC_OK) return rc;
  if (vsm->physical_page_table_size > VSM_DRAW_MAX_EXTENT)
    return fail(OXC_E_INVALID, "physical_page_table_size %d > %d: pixel centres beyond the raster's 2^22 sub-pixel snap range", vsm->physical_page_table_size,
                VSM_DRAW_MAX_EXTENT);
  if (!c->scene_set) return fail(OXC_E_STATE, "oxc_set_scene first");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  rc = refresh_inst_cache(c, coarse, s, false); // the coarse camera's PV . W for the triangle test, from the argument
  if (rc != OXC_OK) return rc;
  const int size = vsm->page_table_size, wpr = (size + 31) / 32;
  const size_t words = (size_t)vsm->clipmap_count * size * wpr;
  if (words > c->vsm_bitmap_words) {
    cudaFree(c->d_vsm_bitmap);
    c->vsm_bitmap_words = 0;
    if (dalloc(&c->d_vsm_bitmap, words) != OXC_OK) return OXC_E_CUDA;
    c->vsm_bitmap_words = words;
  }
  if ((size_t)size + 1 > c->vsm_first_px_cap) {
    cudaFree(c->d_vsm_first_px);
    c->vsm_first_px_cap = 0;
    if (dalloc(&c->d_vsm_first_px, (size_t)size + 1) != OXC_OK) return OXC_E_CUDA;
    c->vsm_first_px_cap = (size_t)size + 1;
  }
  if (!c->d_vsm_queue) {
    if (dalloc(&c->d_vsm_queue, (size_t)c->vsm_queue_capacity) != OXC_OK || dalloc(&c->d_vsm_counters, (size_t)4) != OXC_OK) return OXC_E_CUDA;
    CK(cudaMemsetAsync(c->d_vsm_counters, 0, 16, s));
  }
  VsmDrawParams p{};
  p.meshlet_instances = c->d_meshlet_instances; p.inst = c->d_inst; p.geom = c->d_geom; p.mesh_instances = c->d_mesh_instances;
  p.transforms = c->d_transforms; p.visible_indices = c->d_visible; p.tri_cmd = c->d_cull_triangles_cmd; p.id_base = c->id_base;
  if (c->alpha_active) { p.materials = c->d_alpha_materials; p.material_count = c->alpha_material_count; }
  for (int k = 0; k < vsm->clipmap_count; k++) {
    const float* m = clipmaps[k].projection_view_mat;
    for (int i = 0; i < 4; i++) p.pv_row[k][i] = make_float4(m[i], m[4 + i], m[8 + i], m[12 + i]);
    p.page_offset[k][0] = clipmaps[k].page_offset[0]; p.page_offset[k][1] = clipmaps[k].page_offset[1];
  }
  p.dirty_flags = clipmap_dirty_flags_dev; p.page_tables = page_tables_dev; p.atlas = reinterpret_cast<uint32_t*>(physical_atlas_dev);
  p.bitmap = c->d_vsm_bitmap; p.first_px = c->d_vsm_first_px; p.queue = c->d_vsm_queue; p.counters = c->d_vsm_counters;
  p.queue_capacity = c->vsm_queue_capacity;
  p.size = size; p.page_size = vsm->page_size; p.P = vsm->physical_page_table_size; p.phys_per_row = vsm->physical_page_table_size / vsm->page_size;
  p.clipmap_count = vsm->clipmap_count; p.words_per_row = wpr;
  p.fP = (float)p.P; p.fsize = (float)size; p.fpage = (float)vsm->page_size;
  k_vsm_draw_prepare<<<1, 1024, 0, s>>>(p);
  LAUNCHED();
  k_vsm_draw_meshlets<<<persistent_grid(c, VSM_DRAW_WARPS, 8), VSM_DRAW_THREADS, 0, s>>>(p);
  LAUNCHED();
  k_vsm_draw_items<<<(uint32_t)c->sm_count * 8u, VSM_DRAW_THREADS, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_vsm_draw_stats(OxcContext* c, uint32_t out[2], void* stream) {
  if (!c || !out) return fail(OXC_E_INVALID, "null argument");
  if (!c->d_vsm_counters) return fail(OXC_E_STATE, "oxc_vsm_draw_pages has not run on this context");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(out, c->d_vsm_counters, 8, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return OXC_OK;
}

int oxc_vsm_resolve_shadows(OxcContext* c, const OxcVsmContext* vsm, const float inv_pv[16], const float resolution[2],
                            const OxcVirtualClipmap* clipmaps, const float* depth_dev, const float* normals_dev, const uint32_t* page_tables_dev,
                            const float* physical_atlas_dev, float* shadow_dev, void* stream) {
  if (!c || !vsm || !inv_pv || !resolution || !clipmaps || !depth_dev || !normals_dev || !page_tables_dev || !physical_atlas_dev || !shadow_dev)
    return fail(OXC_E_INVALID, "null argument");
  int rc = check_vsm(vsm, 0xFFFFFFFFu);
  if (rc != OXC_OK) return rc;
  if (vsm->depth_extent[0] < 1 || vsm->depth_extent[1] < 1)
    return fail(OXC_E_INVALID, "depth_extent %d x %d is empty", vsm->depth_extent[0], vsm->depth_extent[1]);
  if (reinterpret_cast<uintptr_t>(normals_dev) & 15u) return fail(OXC_E_INVALID, "normals_dev is not 16-byte aligned (float4 per pixel)");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  const VsmResolveParams p = vsm_resolve_make_params(*vsm, inv_pv, resolution, clipmaps, depth_dev, normals_dev, page_tables_dev,
                                                      physical_atlas_dev, shadow_dev);
  const dim3 grid((p.width + VSM_RESOLVE_TILE_X - 1) / VSM_RESOLVE_TILE_X, (p.height + VSM_RESOLVE_TILE_Y - 1) / VSM_RESOLVE_TILE_Y);
  k_vsm_resolve_shadows<<<grid, VSM_RESOLVE_THREADS, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_generate_ambient_occlusion(OxcContext* c, const OxcGtaoCamera* cam, const OxcGtaoSettings* st, const float* depth_dev,
                                   const float* normals_dev, uint32_t w, uint32_t h, const OxcGtaoTargets* t, void* stream) {
  if (!c || !cam || !st || !depth_dev || !normals_dev || !t) return fail(OXC_E_INVALID, "null argument");
  if (!t->depth_mips || !t->edges || !t->noisy_occlusion || !t->ambient_occlusion) return fail(OXC_E_INVALID, "null target");
  if (w == 0 || h == 0) return fail(OXC_E_INVALID, "empty extent %u x %u", w, h);
  if (w > 32768u || h > 32768u) return fail(OXC_E_INVALID, "extent %u x %u above 32768", w, h);
  if (st->slice_count < 1u || st->slice_count > OXC_GTAO_MAX_SLICES)
    return fail(OXC_E_INVALID, "slice_count %u outside 1..%u", st->slice_count, OXC_GTAO_MAX_SLICES);
  if (st->samples_per_slice_side < 1u || st->samples_per_slice_side > OXC_GTAO_MAX_SAMPLES_PER_SIDE)
    return fail(OXC_E_INVALID, "samples_per_slice_side %u outside 1..%u", st->samples_per_slice_side, OXC_GTAO_MAX_SAMPLES_PER_SIDE);
  if (reinterpret_cast<uintptr_t>(normals_dev) & 15u) return fail(OXC_E_INVALID, "normals_dev is not 16-byte aligned (float4 per pixel)");
  if ((reinterpret_cast<uintptr_t>(depth_dev) | reinterpret_cast<uintptr_t>(t->depth_mips) | reinterpret_cast<uintptr_t>(t->edges) |
       reinterpret_cast<uintptr_t>(t->ambient_occlusion)) & 3u)
    return fail(OXC_E_INVALID, "depth_dev, depth_mips, edges and ambient_occlusion must be 4-byte aligned");
  if (reinterpret_cast<uintptr_t>(t->noisy_occlusion) & 1u) return fail(OXC_E_INVALID, "noisy_occlusion is not 2-byte aligned");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  const GtaoParams p = gtao_make_params(*cam, *st, depth_dev, normals_dev, w, h, *t);
  const dim3 pre((w + 2 * GTAO_PREFILTER_SIDE - 1) / (2 * GTAO_PREFILTER_SIDE), (h + 2 * GTAO_PREFILTER_SIDE - 1) / (2 * GTAO_PREFILTER_SIDE));
  k_gtao_prefilter<<<pre, dim3(GTAO_PREFILTER_SIDE, GTAO_PREFILTER_SIDE), 0, s>>>(p);
  LAUNCHED();
  const dim3 grid((w + GTAO_TILE_X - 1) / GTAO_TILE_X, (h + GTAO_TILE_Y - 1) / GTAO_TILE_Y);
  k_gtao_main<<<grid, GTAO_THREADS, 0, s>>>(p);
  LAUNCHED();
  k_gtao_denoise<<<grid, GTAO_THREADS, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_apply_pbr(OxcContext* c, const OxcPbrCamera* cam, const OxcPbrSettings* st, const OxcLight* lights_dev, const OxcPbrInputs* in,
                  uint32_t w, uint32_t h, float* out_dev, void* stream) {
  if (!c || !cam || !st || !in || !out_dev) return fail(OXC_E_INVALID, "null argument");
  if (!in->depth || !in->albedo || !in->normal || !in->emissive || !in->metallic_roughness_occlusion) return fail(OXC_E_INVALID, "null input plane");
  if (st->light_count > OXC_MAX_LIGHTS) return fail(OXC_E_INVALID, "light_count %u above %u", st->light_count, OXC_MAX_LIGHTS);
  if (st->light_count > 0 && !lights_dev) return fail(OXC_E_INVALID, "null lights with light_count %u", st->light_count);
  if (st->scene_flags & OXC_SCENE_HAS_ATMOSPHERE) return fail(OXC_E_INVALID, "HasAtmosphere: the atmosphere variant is not available");
  if ((st->scene_flags & OXC_SCENE_HAS_CONTACT_SHADOWS) && !in->contact_shadow)
    return fail(OXC_E_INVALID, "null contact_shadow plane under HasContactShadows");
  if (w == 0 || h == 0) return fail(OXC_E_INVALID, "empty extent %u x %u", w, h);
  if (w > 32768u || h > 32768u) return fail(OXC_E_INVALID, "extent %u x %u above 32768", w, h);
  if ((reinterpret_cast<uintptr_t>(in->albedo) | reinterpret_cast<uintptr_t>(in->normal) | reinterpret_cast<uintptr_t>(in->emissive) |
       reinterpret_cast<uintptr_t>(in->metallic_roughness_occlusion) | reinterpret_cast<uintptr_t>(out_dev) |
       reinterpret_cast<uintptr_t>(lights_dev)) & 15u)
    return fail(OXC_E_INVALID, "float4 planes, out_dev and lights_dev must be 16-byte aligned");
  if ((reinterpret_cast<uintptr_t>(in->depth) | reinterpret_cast<uintptr_t>(in->ambient_occlusion) | reinterpret_cast<uintptr_t>(in->shadow) |
       reinterpret_cast<uintptr_t>(in->contact_shadow)) & 3u)
    return fail(OXC_E_INVALID, "depth, ambient_occlusion, shadow and contact_shadow must be 4-byte aligned");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  const PbrParams p = pbr_make_params(*cam, *st, lights_dev, *in, w, h, out_dev);
  const dim3 grid((w + PBR_TILE_X - 1) / PBR_TILE_X, (h + PBR_TILE_Y - 1) / PBR_TILE_Y);
  k_apply_pbr<<<grid, PBR_THREADS, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_contact_shadows(OxcContext* c, const OxcContactShadowCamera* cam, const OxcContactShadowSettings* st, const float* depth_dev, uint32_t w,
                        uint32_t h, float* out_dev, void* stream) {
  if (!c || !cam || !st || !depth_dev || !out_dev) return fail(OXC_E_INVALID, "null argument");
  if (w == 0 || h == 0) return fail(OXC_E_INVALID, "empty extent %u x %u", w, h);
  if (w > 32768u || h > 32768u) return fail(OXC_E_INVALID, "extent %u x %u above 32768", w, h);
  if (st->steps < 1u || st->steps > OXC_CONTACT_SHADOW_MAX_STEPS)
    return fail(OXC_E_INVALID, "steps %u outside 1..%u", st->steps, OXC_CONTACT_SHADOW_MAX_STEPS);
  if ((reinterpret_cast<uintptr_t>(depth_dev) | reinterpret_cast<uintptr_t>(out_dev)) & 3u)
    return fail(OXC_E_INVALID, "depth_dev and out_dev must be 4-byte aligned");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  const ContactShadowParams p = cs_make_params(*cam, *st, depth_dev, w, h, out_dev);
  const dim3 grid((w + CONTACT_TILE_X - 1) / CONTACT_TILE_X, (h + CONTACT_TILE_Y - 1) / CONTACT_TILE_Y);
  k_contact_shadows<<<grid, CONTACT_THREADS, 0, s>>>(p);
  LAUNCHED();
  return OXC_OK;
}

int oxc_check_status(OxcContext* c, void* stream, uint32_t* flags_out) {
  if (!c) return fail(OXC_E_INVALID, "null context");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  uint32_t f = 0;
  CK(cudaMemcpyAsync(&f, c->d_status, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (flags_out) *flags_out = f;
  if (!f) return OXC_OK;
  CK(cudaMemsetAsync(c->d_status, 0, 4, s));
  if (f & (OXC_STATUS_MESHLET_OVERFLOW | OXC_STATUS_SURVIVOR_OVERFLOW | OXC_STATUS_ID_OVERFLOW | OXC_STATUS_CLIP_OVERFLOW | OXC_STATUS_PEER_TIMEOUT))
    return fail(OXC_E_CAPACITY, "device status 0x%x:%s%s%s%s%s", f, (f & OXC_STATUS_MESHLET_OVERFLOW) ? " cull_meshes exceeded max_meshlet_instances (clamped)" : "",
                (f & OXC_STATUS_SURVIVOR_OVERFLOW) ? " a survivor list exceeded the gather capacity (truncated)" : "",
                (f & OXC_STATUS_ID_OVERFLOW) ? " a meshlet-instance id overflowed the vis-buffer id bits" : "",
                (f & OXC_STATUS_CLIP_OVERFLOW) ? " the clip queue overflowed (run oxc_raster_visbuffer_clip_pass)" : "",
                (f & OXC_STATUS_PEER_TIMEOUT) ? " a peer GPU did not signal its Hi-Z exchange in time" : "");
  if (f & OXC_STATUS_BAD_MATERIAL)
    return fail(OXC_E_INVALID, "device status 0x%x: a MeshInstance::material_index lies outside the table of oxc_set_materials (rasterised as opaque)", f);
  return fail(OXC_E_INVALID, "device status 0x%x: unknown status bit (OXC_STATUS_BAD_GEOMETRY is reserved: oxc_set_scene refuses malformed meshlets)", f);
}

// instrumentation builds (-DOXC_RASTER_STATS): device pointer of the 128 u64 statistics slots behind the chunk queue
void* oxc_debug_stats_ptr(OxcContext* c) { return c ? static_cast<void*>(c->d_big_queue + (size_t)c->big_capacity * 4) : nullptr; }

// 96 bytes from pinned (mapped) host memory into the device camera buffer by a kernel: inside a captured frame this keeps the
// copy engines out of the frame's critical path (they are busy with the previous frame's read-back)
__global__ void k_load_camera(OxcCullCamera* dst, const OxcCullCamera* src_pinned) {
  if (threadIdx.x < sizeof(OxcCullCamera) / 4)
    reinterpret_cast<uint32_t*>(dst)[threadIdx.x] = reinterpret_cast<const volatile uint32_t*>(src_pinned)[threadIdx.x];
}

int oxc_load_camera(OxcContext* c, OxcCullCamera* camera_dev, const OxcCullCamera* camera_pinned_host, void* stream) {
  if (!c || !camera_dev || !camera_pinned_host) return fail(OXC_E_INVALID, "null argument");
  CK(cudaSetDevice(c->device));
  k_load_camera<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(camera_dev, camera_pinned_host);
  LAUNCHED();
  return OXC_OK;
}

int oxc_bind_camera_buffer(OxcContext* c, const OxcCullCamera* camera_dev) {
  if (!c) return fail(OXC_E_INVALID, "null context");
  c->cam_dev = camera_dev;
  c->cache_valid = c->cache_valid && camera_dev == nullptr; // whatever InstCull holds was built for some other camera
  return OXC_OK;
}

int oxc_mark_hiz_dirty(OxcContext* c) {
  if (!c) return fail(OXC_E_INVALID, "null context");
  c->hiz_zero = false;
  return OXC_OK;
}

/* ------------------------------------------------------------------------------------------------
 * Multi-GPU exchange (SURVEY §8e).  NCCL is loaded with dlopen: a host that never calls oxc_mgpu_* needs no NCCL at all, and a
 * process that already carries one (PyTorch) shares it.
 * ---------------------------------------------------------------------------------------------- */
} // extern "C"

namespace {
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*CommCount)(const ncclComm_t, int*) = nullptr;
  ncclResult_t (*CommUserRank)(const ncclComm_t, int*) = nullptr;
} g_nccl;

int nccl_load() {
  if (g_nccl.lib) return OXC_OK;
  void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) return fail(OXC_E_INVALID, "libnccl.so.2 not found (%s): oxc_mgpu_* needs NCCL", dlerror());
#define SYM(field, name)                                                                    \
  g_nccl.field = reinterpret_cast<decltype(g_nccl.field)>(dlsym(lib, name));                \
  if (!g_nccl.field) return fail(OXC_E_INVALID, "libnccl.so.2 lacks %s", name)
  SYM(GetUniqueId, "ncclGetUniqueId"); SYM(CommInitRank, "ncclCommInitRank"); SYM(CommDestroy, "ncclCommDestroy");
  SYM(AllReduce, "ncclAllReduce"); SYM(AllGather, "ncclAllGather"); SYM(GetErrorString, "ncclGetErrorString");
  SYM(CommCount, "ncclCommCount"); SYM(CommUserRank, "ncclCommUserRank");
#undef SYM
  g_nccl.lib = lib;
  return OXC_OK;
}
#define NCK(expr)                                                                                                   \
  do {                                                                                                              \
    ncclResult_t r_ = (expr);                                                                                       \
    if (r_ != ncclSuccess) return fail(OXC_E_CUDA, "%s: %s (%s:%d)", #expr, g_nccl.GetErrorString(r_), __FILE__, __LINE__); \
  } while (0)

void mgpu_release(OxcContext* c) {
  OxcContext::Mgpu& m = c->mg;
  for (uint32_t r = 0; r < m.world && r < (uint32_t)MGPU_MAX_RANKS; r++)
    if (r != m.rank && m.peer_base[r]) cudaIpcCloseMemHandle(m.peer_base[r]);
  cudaFree(m.xbuf); cudaFree(m.d_seq);
  for (int k = 0; k < 2; k++) { cudaFree(m.cnt_stage[k]); cudaFree(m.ids_stage[k]); cudaFree(m.cnt_all[k]); cudaFree(m.ids_all[k]); }
  if (m.comm && m.own_comm && g_nccl.CommDestroy) g_nccl.CommDestroy(m.comm);
  m = OxcContext::Mgpu();
}

#define MGDBG(...) do { if (getenv("OXC_MGPU_DEBUG")) { fprintf(stderr, "[oxc_mgpu r%u] ", rank); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); fflush(stderr); } } while (0)
int mgpu_setup(OxcContext* c, ncclComm_t comm, bool own, uint32_t rank, uint32_t world, uint32_t survivor_capacity) {
  OxcContext::Mgpu& m = c->mg;
  MGDBG("setup: world %u, communicator ready", world);
  m.comm = comm; m.own_comm = own; m.rank = rank; m.world = world;
  m.capacity = survivor_capacity ? survivor_capacity : c->info.max_meshlet_instances;
  if (const char* e = getenv("OXC_MGPU_TIMEOUT_MS")) {
    const long long v = atoll(e);
    if (v > 0) m.timeout_ns = (unsigned long long)v * 1000000ull;
  }
  if (world > 1) { // ncclAllGather needs the same segment size on every rank: agree on the largest request
    uint32_t* d_cap = nullptr;
    CK(cudaMalloc(&d_cap, 4));
    CK(cudaMemcpy(d_cap, &m.capacity, 4, cudaMemcpyHostToDevice));
    NCK(g_nccl.AllReduce(d_cap, d_cap, 1, ncclUint32, ncclMax, comm, nullptr));
    CK(cudaStreamSynchronize(nullptr));
    CK(cudaMemcpy(&m.capacity, d_cap, 4, cudaMemcpyDeviceToHost));
    cudaFree(d_cap);
    MGDBG("survivor segment capacity %u", m.capacity);
  }
  const size_t texels = (size_t)c->hiz.width * c->hiz.height;
  m.xbuf_words = 2 * texels + 2 * MGPU_MAX_RANKS;
  CK(cudaMalloc(&m.xbuf, m.xbuf_words * 4));
  CK(cudaMemset(m.xbuf, 0, m.xbuf_words * 4));
  CK(cudaMalloc(&m.d_seq, 4));
  CK(cudaMemset(m.d_seq, 0, 4));
  for (int k = 0; k < 2; k++) {
    CK(cudaMalloc(&m.cnt_stage[k], 16));
    CK(cudaMalloc(&m.ids_stage[k], (size_t)m.capacity * 4));
    CK(cudaMalloc(&m.cnt_all[k], (size_t)world * 16));
    CK(cudaMalloc(&m.ids_all[k], (size_t)world * m.capacity * 4));
    CK(cudaMemset(m.cnt_all[k], 0, (size_t)world * 16));
  }
  // Exchange the CUDA-IPC handles of the Hi-Z exchange buffers through the communicator itself (64 bytes per rank), then map
  // every peer's buffer.  Any failure (no peer access between the devices, IPC disabled in the container) leaves peer_hiz false:
  // oxc_mgpu_exchange_hiz then falls back to an NCCL all-reduce of the mip-0 texels — slower, same result.
  m.peer_hiz = false;
  m.peers = MgpuPeers{};
  m.peers.rank = rank; m.peers.world = world;
  m.peers.xbuf[rank] = m.xbuf; m.peers.flags[rank] = m.xbuf + 2 * texels;
  m.peer_base[rank] = m.xbuf;
  if (world > 1) {
    cudaIpcMemHandle_t mine{};
    const bool have = cudaIpcGetMemHandle(&mine, m.xbuf) == cudaSuccess;
    if (!have) cudaGetLastError();
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    unsigned char *d_one = nullptr, *d_all = nullptr;
    CK(cudaMalloc(&d_one, 128));
    CK(cudaMalloc(&d_all, (size_t)128 * world));
    unsigned char rec[128] = {};
    memcpy(rec, &mine, 64);
    rec[64] = have ? 1 : 0;
    CK(cudaMemcpy(d_one, rec, 128, cudaMemcpyHostToDevice));
    MGDBG("ipc handle %s; allgather of the handles", have ? "ok" : "UNAVAILABLE");
    NCK(g_nccl.AllGather(d_one, d_all, 128, ncclUint8, comm, nullptr));
    CK(cudaStreamSynchronize(nullptr));
    MGDBG("handles gathered");
    std::vector<unsigned char> all((size_t)128 * world);
    CK(cudaMemcpy(all.data(), d_all, all.size(), cudaMemcpyDeviceToHost));
    cudaFree(d_one); cudaFree(d_all);
    bool ok = true;
    for (uint32_t r = 0; r < world && ok; r++) ok = all[(size_t)r * 128 + 64] == 1;
    for (uint32_t r = 0; r < world && ok; r++) {
      if (r == rank) continue;
      cudaIpcMemHandle_t h;
      memcpy(&h, &all[(size_t)r * 128], 64);
      void* base = nullptr;
      if (cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = false; break; }
      m.peer_base[r] = base;
      m.peers.xbuf[r] = static_cast<uint32_t*>(base);
      m.peers.flags[r] = static_cast<uint32_t*>(base) + 2 * texels;
    }
    MGDBG("peer buffers mapped: %s", ok ? "yes" : "NO");
    // every rank must take the same path: agree through one more tiny collective (min over ranks of "ok")
    uint32_t* d_ok = nullptr;
    CK(cudaMalloc(&d_ok, 4));
    const uint32_t okv = ok ? 1u : 0u;
    CK(cudaMemcpy(d_ok, &okv, 4, cudaMemcpyHostToDevice));
    NCK(g_nccl.AllReduce(d_ok, d_ok, 1, ncclUint32, ncclMin, comm, nullptr));
    CK(cudaStreamSynchronize(nullptr));
    uint32_t all_ok = 0;
    CK(cudaMemcpy(&all_ok, d_ok, 4, cudaMemcpyDeviceToHost));
    cudaFree(d_ok);
    m.peer_hiz = all_ok != 0;
    MGDBG("hiz exchange over %s", m.peer_hiz ? "NVLink peer memory" : "NCCL all-reduce (fallback)");
  }
  m.active = true;
  return OXC_OK;
}
} // namespace

extern "C" {

int oxc_mgpu_get_unique_id(uint8_t id[OXC_MGPU_ID_BYTES]) {
  if (!id) return fail(OXC_E_INVALID, "null argument");
  int rc = nccl_load();
  if (rc != OXC_OK) return rc;
  static_assert(sizeof(ncclUniqueId) == OXC_MGPU_ID_BYTES, "ncclUniqueId size");
  ncclUniqueId u;
  NCK(g_nccl.GetUniqueId(&u));
  memcpy(id, &u, sizeof u);
  return OXC_OK;
}

int oxc_mgpu_init(OxcContext* c, uint32_t rank, uint32_t world, const uint8_t id[OXC_MGPU_ID_BYTES], uint32_t survivor_capacity) {
  if (!c || !id) return fail(OXC_E_INVALID, "null argument");
  if (world == 0 || world > (uint32_t)MGPU_MAX_RANKS || rank >= world) return fail(OXC_E_INVALID, "rank %u / world %u (max %d ranks)", rank, world, MGPU_MAX_RANKS);
  if (c->mg.active) return fail(OXC_E_STATE, "oxc_mgpu_init called twice");
  CK(cudaSetDevice(c->device));
  int rc = nccl_load();
  if (rc != OXC_OK) return rc;
  ncclUniqueId u;
  memcpy(&u, id, sizeof u);
  ncclComm_t comm = nullptr;
  NCK(g_nccl.CommInitRank(&comm, (int)world, u, (int)rank));
  rc = mgpu_setup(c, comm, true, rank, world, survivor_capacity);
  if (rc != OXC_OK) mgpu_release(c);
  return rc;
}

int oxc_mgpu_init_with_comm(OxcContext* c, void* nccl_comm, uint32_t survivor_capacity) {
  if (!c || !nccl_comm) return fail(OXC_E_INVALID, "null argument");
  if (c->mg.active) return fail(OXC_E_STATE, "oxc_mgpu_init called twice");
  CK(cudaSetDevice(c->device));
  int rc = nccl_load();
  if (rc != OXC_OK) return rc;
  int world = 0, rank = 0;
  NCK(g_nccl.CommCount(static_cast<ncclComm_t>(nccl_comm), &world));
  NCK(g_nccl.CommUserRank(static_cast<ncclComm_t>(nccl_comm), &rank));
  if (world <= 0 || world > MGPU_MAX_RANKS) return fail(OXC_E_INVALID, "communicator of %d ranks (max %d)", world, MGPU_MAX_RANKS);
  rc = mgpu_setup(c, static_cast<ncclComm_t>(nccl_comm), false, (uint32_t)rank, (uint32_t)world, survivor_capacity);
  if (rc != OXC_OK) mgpu_release(c);
  return rc;
}

// Collective: the ranks agree on max(capacity) and reallocate the gather buffers.  For hosts that only learn how many
// survivors a frame leaves once real (exchanged) frames have run: init generously, measure, shrink.
int oxc_mgpu_set_survivor_capacity(OxcContext* c, uint32_t capacity) {
  if (!c || capacity == 0) return fail(OXC_E_INVALID, "bad argument");
  if (!c->mg.active) return fail(OXC_E_STATE, "oxc_mgpu_init first");
  CK(cudaSetDevice(c->device));
  CK(cudaDeviceSynchronize());
  OxcContext::Mgpu& m = c->mg;
  if (m.world > 1) {
    uint32_t* d_cap = nullptr;
    CK(cudaMalloc(&d_cap, 4));
    CK(cudaMemcpy(d_cap, &capacity, 4, cudaMemcpyHostToDevice));
    NCK(g_nccl.AllReduce(d_cap, d_cap, 1, ncclUint32, ncclMax, m.comm, nullptr));
    CK(cudaStreamSynchronize(nullptr));
    CK(cudaMemcpy(&capacity, d_cap, 4, cudaMemcpyDeviceToHost));
    cudaFree(d_cap);
  }
  for (int k = 0; k < 2; k++) {
    cudaFree(m.ids_stage[k]); cudaFree(m.ids_all[k]);
    m.ids_stage[k] = m.ids_all[k] = nullptr;
    CK(cudaMalloc(&m.ids_stage[k], (size_t)capacity * 4));
    CK(cudaMalloc(&m.ids_all[k], (size_t)m.world * capacity * 4));
  }
  m.capacity = capacity;
  return OXC_OK;
}

int oxc_mgpu_shutdown(OxcContext* c) {
  if (!c) return fail(OXC_E_INVALID, "null context");
  CK(cudaSetDevice(c->device));
  CK(cudaDeviceSynchronize());
  mgpu_release(c);
  return OXC_OK;
}

int oxc_mgpu_info(OxcContext* c, OxcMgpuInfo* out) {
  if (!c || !out) return fail(OXC_E_INVALID, "null argument");
  memset(out, 0, sizeof *out);
  out->active = c->mg.active; out->rank = c->mg.rank; out->world = c->mg.world; out->survivor_capacity = c->mg.capacity;
  out->hiz_over_peer_memory = c->mg.peer_hiz;
  for (int k = 0; k < 2; k++) { out->gathered_counts[k] = c->mg.cnt_all[k]; out->gathered_ids[k] = c->mg.ids_all[k]; }
  return OXC_OK;
}

// generate_hiz with the other ranks' depth: replaces oxc_build_hiz_packed between the two passes of a sharded frame
int oxc_mgpu_exchange_hiz(OxcContext* c, const uint64_t* vis, uint32_t w, uint32_t h, void* stream) {
  if (!c || !vis || !w || !h) return fail(OXC_E_INVALID, "bad argument");
  if (!c->mg.active) return fail(OXC_E_STATE, "oxc_mgpu_init first");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  OxcContext::Mgpu& m = c->mg;
  if (m.world == 1) return oxc_build_hiz_packed(c, vis, w, h, stream);
  const size_t n = (size_t)c->hiz.width * c->hiz.height;
  if (m.peer_hiz) {
    k_mgpu_hiz_push<<<capped_grid(c, n), 256, 0, s>>>(reinterpret_cast<const unsigned long long*>(vis), w, h, c->hiz.width, c->hiz.height, ilog2(c->hiz.width),
                                         ilog2(c->hiz.height), m.peers, m.d_seq);
    LAUNCHED();
    k_mgpu_signal<<<1, 32, 0, s>>>(m.peers, m.d_seq);
    LAUNCHED();
    k_mgpu_hiz_collect<<<c->sm_count * 4, 256, 0, s>>>(m.peers, m.d_seq, c->d_hiz, n, c->d_status, m.timeout_ns);
    LAUNCHED();
  } else {
    int rc = oxc_build_hiz_mip0_packed(c, vis, w, h, stream);
    if (rc != OXC_OK) return rc;
    // depths are >= +0: the unsigned order of the bits is the order of the floats
    NCK(g_nccl.AllReduce(c->d_hiz, c->d_hiz, n, ncclUint32, ncclMax, m.comm, s));
  }
  return oxc_build_hiz_from_mip0(c, stream);
}

// End of a sharded frame: per-pixel max of the packed vis buffer over the ranks (in place), and every rank's survivor list +
// counters gathered into the context's buffers of `slot` (0/1: a host that overlaps this exchange with the next frame on a
// side stream alternates the slots).
int oxc_mgpu_stage_survivors(OxcContext* c, int slot, void* stream) {
  if (!c || (slot != 0 && slot != 1)) return fail(OXC_E_INVALID, "bad argument");
  if (!c->mg.active) return fail(OXC_E_STATE, "oxc_mgpu_init first");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  OxcContext::Mgpu& m = c->mg;
  k_mgpu_stage_survivors<<<c->sm_count, 256, 0, s>>>(c->d_vis, c->d_visible, m.capacity, m.cnt_stage[slot], m.ids_stage[slot], c->d_status);
  LAUNCHED();
  return OXC_OK;
}

int oxc_mgpu_exchange_frame(OxcContext* c, uint64_t* vis, uint32_t w, uint32_t h, int slot, uint32_t flags, void* stream) {
  if (!c || (slot != 0 && slot != 1)) return fail(OXC_E_INVALID, "bad argument");
  if (!c->mg.active) return fail(OXC_E_STATE, "oxc_mgpu_init first");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  CK(cudaSetDevice(c->device));
  OxcContext::Mgpu& m = c->mg;
  if (!(flags & OXC_MGPU_ALREADY_STAGED)) {
    int rc = oxc_mgpu_stage_survivors(c, slot, stream);
    if (rc != OXC_OK) return rc;
  }
  if (m.world == 1) {
    CK(cudaMemcpyAsync(m.cnt_all[slot], m.cnt_stage[slot], 16, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(m.ids_all[slot], m.ids_stage[slot], (size_t)m.capacity * 4, cudaMemcpyDeviceToDevice, s));
    return OXC_OK;
  }
  if (vis) NCK(g_nccl.AllReduce(vis, vis, (size_t)w * h, ncclUint64, ncclMax, m.comm, s)); // reverse-Z GreaterOrEqual == max of depth|id
  NCK(g_nccl.AllGather(m.cnt_stage[slot], m.cnt_all[slot], 4, ncclUint32, m.comm, s));
  NCK(g_nccl.AllGather(m.ids_stage[slot], m.ids_all[slot], m.capacity, ncclUint32, m.comm, s));
  return OXC_OK;
}

int oxc_get_outputs(OxcContext* c, OxcOutputs* o) {
  if (!c || !o) return fail(OXC_E_INVALID, "null argument");
  memset(o, 0, sizeof *o);
  o->visibility = c->d_vis; o->cull_meshlets_cmd = c->d_cull_meshlets_cmd; o->cull_triangles_cmd = c->d_cull_triangles_cmd;
  o->draw_cmd = c->d_draw_cmd; o->meshlet_instances = c->d_meshlet_instances; o->visible_meshlet_instances_indices = c->d_visible;
  o->meshlet_instance_visibility_mask = c->d_mask; o->reordered_indices = c->d_reordered; o->mesh_instances = c->d_mesh_instances;
  o->hiz = c->d_hiz;
  memcpy(o->hiz_level_offset, c->hiz.level_offset, sizeof o->hiz_level_offset);
  o->hiz_levels = c->hiz.levels; o->hiz_width = c->hiz.width; o->hiz_height = c->hiz.height;
  o->visibility_mask_words = c->mask_words;
  o->view_visibility_bits = c->d_view_bits; o->view_visible_counts = c->d_view_counts;
  o->raster_triangle_count = reinterpret_cast<uint64_t*>(c->d_tri_counter);
  o->status_flags = c->d_status;
  o->vis_primitive_bits = c->prim_bits;
  return OXC_OK;
}

} // extern "C"
