/*
 * oxcull.h — C ABI of liboxcull.so: the H100-native meshlet visibility pipeline.
 *
 * Drop-in boundary for the ONE hot path of oxylusengine/Oxylus that SURVEY.md §8 scopes:
 *   RendererInstance::cull_geometry      Oxylus/src/Render/Passes/CullGeometry.cpp:61-404
 *   RendererInstance::generate_hiz       Oxylus/src/Render/Passes/CullGeometry.cpp:10-59
 *   RendererInstance::draw_for_visbuffer Oxylus/src/Render/Passes/DrawGeometry.cpp:104-190
 * The reference has no FFI for this path: the seam is the *buffer set and call sequence* those three
 * member functions record into the vuk render graph.  Every entry point below names the reference
 * pass it replaces (file:line).  Plain pointers and sizes only; no torch / vuk / glm types.
 *
 * Conventions (identical to the reference):
 *   - reverse-Z (near = 1, far = 0; depth cleared to 0, depth test GreaterOrEqual)
 *   - matrices are column-major in memory (glm): m[col*4 + row]; Slang M[i] = row i
 *   - scalar buffer layout; struct sizes are static_assert'ed below against SceneGPU.hpp
 *   - all work is enqueued on the caller's cudaStream_t (passed as void*); no hidden syncs
 *   - one context per device; a context is not thread-safe (the reference records on one thread)
 *   - return 0 on success, negative OXC_E_* otherwise; oxc_last_error() gives text
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails loudly.
 */
#ifndef OXCULL_H_
#define OXCULL_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__cplusplus)
#define OXC_STATIC_ASSERT(c, m) static_assert(c, m)
#else
#define OXC_STATIC_ASSERT(c, m) _Static_assert(c, m)
#endif

/* ------------------------------------------------------------------------------------------------
 * GPU data ABI — host mirrors of Oxylus/include/Scene/SceneGPU.hpp (scalar layout)
 * ---------------------------------------------------------------------------------------------- */

/* SceneGPU.hpp:20-22 TransformWorld — glm::mat4, column-major */
typedef struct OxcTransformWorld { float world[16]; } OxcTransformWorld;

/* SceneGPU.hpp:84-90 / scene.slang:401-435 MeshletBounds (16 B): half3 center, s8 cone xy,
 * half3 extent (FULL size, halved by the tests), s8 cone z, s8 cutoff */
typedef struct OxcMeshletBounds {
  uint16_t aabb_center[3];
  int8_t cone_axis_xy[2];
  uint16_t aabb_extent[3];
  int8_t cone_axis_z;
  int8_t cone_cutoff;
} OxcMeshletBounds;

/* SceneGPU.hpp:92-95 MeshBounds */
typedef struct OxcMeshBounds { float aabb_center[3]; float aabb_extent[3]; } OxcMeshBounds;

/* SceneGPU.hpp:97-104 MeshletInstanceVisibility */
typedef struct OxcMeshletInstanceVisibility {
  uint32_t total_visible_meshlet_instances; /* written by cull_meshes only */
  uint32_t early_visible_meshlet_instances;
  uint32_t late_visible_meshlet_instances;
} OxcMeshletInstanceVisibility;

/* SceneGPU.hpp:106-109 */
typedef struct OxcMeshletInstance { uint32_t mesh_instance_index; uint32_t meshlet_index; } OxcMeshletInstance;

/* SceneGPU.hpp:111-117 (20 B) */
typedef struct OxcMeshInstance {
  uint32_t mesh_index;
  uint32_t lod_index;
  uint32_t material_index;
  uint32_t transform_index;
  uint32_t meshlet_instance_visibility_offset;
} OxcMeshInstance;

/* SceneGPU.hpp:119-124 (16 B) */
typedef struct OxcMeshlet {
  uint32_t indirect_vertex_index_offset;
  uint32_t local_triangle_index_offset;
  uint32_t vertex_count;
  uint32_t triangle_count;
} OxcMeshlet;

/* SceneGPU.hpp:126-140 (64 B).  The u64 members are device addresses on the GPU (reference ABI);
 * in an OxcSceneDesc passed to oxc_set_scene they are BYTE OFFSETS into OxcSceneDesc::blob and are
 * rebased on upload, exactly like upload_gltf_mesh patches blob offsets into device addresses
 * (Oxylus/src/Asset/AssetManager_GLTF.cpp:778-800). */
typedef struct OxcMeshLOD {
  uint64_t indices;
  uint64_t meshlets;                /* OxcMeshlet[meshlet_count] */
  uint64_t meshlet_bounds;          /* OxcMeshletBounds[meshlet_bounds_count] */
  uint64_t local_triangle_indices;  /* u8 micro indices packed in u32 words */
  uint64_t indirect_vertex_indices; /* u32 */
  uint32_t indices_count;
  uint32_t meshlet_count;
  uint32_t meshlet_bounds_count;
  uint32_t local_triangle_indices_count;
  uint32_t indirect_vertex_indices_count;
  float error;
} OxcMeshLOD;

/* SceneGPU.hpp:142-152 (64 B) */
typedef struct OxcMesh {
  uint64_t vertex_positions; /* u16x4 per vertex (half3 + pad) */
  uint64_t vertex_normals;   /* u32 per vertex, 10:10:10 (scene.slang:486-489); 0 = none (read by oxc_decode_visbuffer only) */
  uint64_t texture_coords;   /* u16x2 halves per vertex (scene.slang:491-497); 0 = none (Mesh::texture_coords == nullptr) */
  uint32_t vertex_count;
  uint32_t lod_count;
  uint64_t lods; /* OxcMeshLOD[lod_count] */
  OxcMeshBounds bounds;
} OxcMesh;

/* SceneGPU.hpp:222-229 (96 B) */
typedef struct OxcCullCamera {
  float projection_view[16];
  float position[3];
  float acceptable_lod_error;
  float resolution[2];
  float near_clip;
  uint32_t mesh_instance_count;
} OxcCullCamera;

/* Shaders/gpu/base.slang:5-17 */
typedef struct OxcDispatchIndirectCommand { uint32_t x, y, z; } OxcDispatchIndirectCommand;
typedef struct OxcDrawIndexedIndirectCommand {
  uint32_t index_count;
  uint32_t instance_count;
  uint32_t first_index;
  int32_t vertex_offset;
  uint32_t first_instance;
} OxcDrawIndexedIndirectCommand;

OXC_STATIC_ASSERT(sizeof(OxcTransformWorld) == 64, "TransformWorld");
OXC_STATIC_ASSERT(sizeof(OxcMeshletBounds) == 16, "MeshletBounds");
OXC_STATIC_ASSERT(sizeof(OxcMeshBounds) == 24, "MeshBounds");
OXC_STATIC_ASSERT(sizeof(OxcMeshletInstanceVisibility) == 12, "MeshletInstanceVisibility");
OXC_STATIC_ASSERT(sizeof(OxcMeshletInstance) == 8, "MeshletInstance");
OXC_STATIC_ASSERT(sizeof(OxcMeshInstance) == 20, "MeshInstance");
OXC_STATIC_ASSERT(sizeof(OxcMeshlet) == 16, "Meshlet");
OXC_STATIC_ASSERT(sizeof(OxcMeshLOD) == 64, "MeshLOD");
OXC_STATIC_ASSERT(sizeof(OxcMesh) == 64, "Mesh");
OXC_STATIC_ASSERT(sizeof(OxcCullCamera) == 96, "CullCamera");
OXC_STATIC_ASSERT(sizeof(OxcDispatchIndirectCommand) == 12, "DispatchIndirectCommand");
OXC_STATIC_ASSERT(sizeof(OxcDrawIndexedIndirectCommand) == 20, "DrawIndexedIndirectCommand");

/* SceneGPU.hpp:345-353 CullFlag */
enum {
  OXC_CULL_NONE = 0,
  OXC_CULL_TEST_FRUSTUM = 1 << 0,
  OXC_CULL_SELECT_LOD = 1 << 1,
  OXC_CULL_TEST_OCCLUSION = 1 << 2,
  OXC_CULL_LATE_PASS = 1 << 3,
  OXC_CULL_TEST_ALL = (1 << 0) | (1 << 1) | (1 << 2)
};

/* defines.slang:1-23 */
#define OXC_MESH_MAX_LODS 8
#define OXC_MESHLET_MAX_PRIMITIVES 64
#define OXC_MESHLET_MAX_VERTICES 64
/* RendererInstance.cpp:573-588: Hi-Z has min(mips, 13) levels */
#define OXC_HIZ_MAX_LEVELS 13
/* visbuffer.slang:9-14 */
#define OXC_VIS_PRIMITIVE_BITS 8u
#define OXC_VIS_PRIMITIVE_MASK 0xFFu
#define OXC_VIS_CLEAR 0xFFFFFFFFu
/* OxcCreateInfo::wide_ids packing (no reference equivalent): 26-bit meshlet instance id, 6-bit triangle */
#define OXC_VIS_WIDE_PRIMITIVE_BITS 6u
/* oxc_cull_meshlets_multiview: upper bound on batched views */
#define OXC_MAX_VIEWS 16

/* error codes */
enum {
  OXC_OK = 0,
  OXC_E_INVALID = -1,  /* bad argument */
  OXC_E_CUDA = -2,     /* CUDA runtime error (text in oxc_last_error) */
  OXC_E_NO_DEVICE = -3,/* no CUDA device: there is no CPU fallback */
  OXC_E_CAPACITY = -4, /* a create-time capacity would be exceeded */
  OXC_E_STATE = -5     /* call sequence violated (e.g. cull before set_scene) */
};

/* ------------------------------------------------------------------------------------------------
 * Context
 * ---------------------------------------------------------------------------------------------- */
typedef struct OxcContext OxcContext;

typedef struct OxcCreateInfo {
  uint32_t max_mesh_instances;    /* capacity of mesh_instances[] */
  uint32_t max_meshlet_instances; /* == RendererInstanceUpdateInfo::max_meshlet_instance_count (Σ LOD0 meshlets),
                                     sizes meshlet_instances (8 B), visible indices (4 B), mask bits;
                                     RendererInstance.cpp:1651-1665,1717-1732 */
  uint32_t hiz_width;             /* bit_ceil((W+1)>>1), RendererInstance.cpp:573-577; power of two */
  uint32_t hiz_height;
  uint32_t alloc_reordered_indices; /* 1: allocate the 768 B x max index buffer for oxc_cull_triangles
                                       (RendererInstance.cpp:1727-1731); 0: fused raster only */
  uint32_t max_views;             /* 0/1, or up to OXC_MAX_VIEWS for oxc_cull_meshlets_multiview */
  uint32_t max_mask_bits;         /* 0: = max_meshlet_instances.  Multi-GPU shards: the persistent visibility mask is indexed by the
                                     GLOBAL meshlet_instance_visibility_offset, so a shard context keeps max_meshlet_instances at
                                     its own share (8 + 4 B each) and sets this to the whole scene's LOD0 meshlet count (1 bit each) */
  uint32_t wide_ids;              /* 0: the reference's 24 + 8 bit vis-buffer word (visbuffer.slang:9-14; <= 2^24 meshlet instances,
                                     the raster / decode entry points refuse larger scenes with OXC_E_CAPACITY);
                                     1: 26 + 6 bit word (meshlets hold <= 64 triangles, so 6 bits suffice) for scenes of up to
                                     2^26 meshlet instances (BASELINE configs[4], 50 M).  Same ordering of equal-depth winners. */
} OxcCreateInfo;

/* Host-side scene tables (what Scene::runtime_update hands to RendererInstance::update,
 * Oxylus/src/Scene/Scene.cpp:1226-1290).  Mesh/MeshLOD u64 members are byte offsets into blob. */
typedef struct OxcSceneDesc {
  const OxcMesh* meshes;
  uint32_t mesh_count;
  const OxcMeshInstance* mesh_instances;
  uint32_t mesh_instance_count;
  const OxcTransformWorld* transforms;
  uint32_t transform_count;
  const uint8_t* blob;   /* vertex / meshlet / bounds / index data of every mesh; 16-byte aligned offsets */
  uint64_t blob_size;
} OxcSceneDesc;

/* Device pointers of everything the reference keeps in prepared_frame / CullGeometryContext.
 * Valid until oxc_destroy; contents are ordered by the stream the producing call was enqueued on. */
typedef struct OxcOutputs {
  OxcMeshletInstanceVisibility* visibility;        /* CullGeometry.cpp:97 */
  OxcDispatchIndirectCommand* cull_meshlets_cmd;   /* CullGeometry.cpp:98-100 */
  OxcDispatchIndirectCommand* cull_triangles_cmd;  /* CullGeometry.cpp:125-127 (reset by every oxc_cull_meshlets) */
  OxcDrawIndexedIndirectCommand* draw_cmd;         /* CullGeometry.cpp:380-382 */
  OxcMeshletInstance* meshlet_instances;           /* RendererInstance.cpp:1717-1721 */
  uint32_t* visible_meshlet_instances_indices;     /* RendererInstance.cpp:1722-1726 */
  uint32_t* meshlet_instance_visibility_mask;      /* RendererInstance.cpp:1651-1665 */
  uint32_t* reordered_indices;                     /* RendererInstance.cpp:1727-1731 (NULL if not allocated) */
  OxcMeshInstance* mesh_instances;                 /* lod_index is written back by cull_meshes */
  float* hiz;                                      /* all mips, level l at hiz + hiz_level_offset[l] floats */
  uint32_t hiz_level_offset[OXC_HIZ_MAX_LEVELS];
  uint32_t hiz_levels;
  uint32_t hiz_width, hiz_height;
  uint32_t visibility_mask_words;
  uint32_t* view_visibility_bits;                  /* multiview: one u32 per meshlet instance, bit v = view v (NULL if max_views<=1) */
  uint32_t* view_visible_counts;                   /* multiview: u32[OXC_MAX_VIEWS] */
  uint64_t* raster_triangle_count;                 /* triangles that survived cull and were rasterised, cumulative per clear */
  uint32_t* status_flags;                          /* sticky OXC_STATUS_* bits raised by kernels (see oxc_check_status) */
  uint32_t vis_primitive_bits;                     /* 8 (reference packing) or 6 (OxcCreateInfo::wide_ids) */
} OxcOutputs;

/* Device-side error conditions.  Kernels never write out of bounds: they clamp, raise a sticky bit in
 * OxcOutputs::status_flags and carry on; oxc_check_status reads the word (synchronises `stream`), returns
 * OXC_E_CAPACITY / OXC_E_INVALID when a bit is set and clears it. */
enum {
  OXC_STATUS_MESHLET_OVERFLOW = 1 << 0, /* cull_meshes wanted to emit more than max_meshlet_instances (clamped) */
  OXC_STATUS_BAD_GEOMETRY = 1 << 1,     /* reserved, never raised: oxc_set_scene refuses a meshlet whose runs leave their arrays, whose
                                           vertex index addresses records past the blob or whose micro index is >= its vertex count */
  OXC_STATUS_SURVIVOR_OVERFLOW = 1 << 2,/* oxc_mgpu_exchange_frame: a rank's survivor list exceeded the gather capacity (truncated) */
  OXC_STATUS_ID_OVERFLOW = 1 << 3,      /* a vis-buffer id did not fit the id bits of the packing (pixel skipped) */
  OXC_STATUS_CLIP_OVERFLOW = 1 << 5,    /* a triangle across the near / guard-band planes found the raster's deferred queue (2^20 entries) full: the raster still drew it, by a slow second walk over the pass */
  OXC_STATUS_BAD_MATERIAL = 1 << 6,     /* a MeshInstance::material_index outside the table of oxc_set_materials (rasterised as opaque) */
  OXC_STATUS_PEER_TIMEOUT = 1 << 4      /* oxc_mgpu_exchange_hiz: a peer did not raise its flag within 30 s (OXC_MGPU_TIMEOUT_MS); that frame's pyramid is incomplete */
};
int oxc_check_status(OxcContext* ctx, void* stream, uint32_t* flags_out /* may be NULL */);
/* CUDA-graph support: while a DEVICE camera buffer is bound, oxc_cull_meshes / oxc_cull_meshlets (and the InstCull refresh of
 * the triangle passes and of oxc_decode_visbuffer) read projection_view / position / near_clip / resolution / acceptable_lod_error
 * from it instead of from the by-value copy of their `camera` argument, so a captured frame replays with whatever camera the host
 * copied into the buffer before the launch (the host mirror's oxr_submit does exactly that).  The `camera` argument is still
 * required: host-side decisions (mesh_instance_count, "same camera as the InstCull cache") use it; pass the same camera for every
 * main-view pass of a frame.  The passes with views of their own never read the bound buffer: oxc_cull_meshlets_hpb /
 * _hpb_dirty_dev cull against their coarse `camera` argument and oxc_cull_meshlets_multiview / oxc_cull_terrain against their
 * arguments, bound camera or not.  NULL unbinds. */
int oxc_bind_camera_buffer(OxcContext* ctx, const OxcCullCamera* camera_dev);
/* Fills a device camera buffer from PINNED host memory (cudaMallocHost / cudaHostRegister) with a kernel that reads the 96
 * bytes over the bus: capturable, re-reads the host location at every replay, and does not occupy a copy engine. */
int oxc_load_camera(OxcContext* ctx, OxcCullCamera* camera_dev, const OxcCullCamera* camera_pinned_host, void* stream);
/* The Hi-Z pyramid was written through OxcOutputs::hiz by something other than an oxc_* call (an external reduce,
 * a terrain pass): the early pass may no longer assume the per-frame cleared image. */
int oxc_mark_hiz_dirty(OxcContext* ctx);

const char* oxc_last_error(void);
/* number of CUDA kernels this library has launched in this process (bench.py "gpu_launches") */
uint64_t oxc_kernel_launch_count(void);
const char* oxc_version(void);

int oxc_create(int device, const OxcCreateInfo* info, OxcContext** out_ctx);
void oxc_destroy(OxcContext* ctx);

/* RendererInstance::update (RendererInstance.cpp:1333-1788): uploads meshes / mesh_instances /
 * transforms / geometry blob from HOST memory (async on stream; pinned memory recommended),
 * rebases blob offsets to device addresses, (re)sizes and zero-fills the visibility mask
 * (instance table changed => zero_fill_pass, :1651-1665).  Returns OXC_E_INVALID, naming the mesh, LOD and meshlet, for a
 * meshlet whose vertex or triangle run leaves its array, whose vertex index addresses a position (or, when the mesh has
 * them, texture-coordinate) record past the end of the blob, or whose micro index is >= min(vertex_count, 64); nothing is
 * uploaded then.  A vertex index >= Mesh::vertex_count inside the blob is accepted: the decode pass flags it (status 2,
 * visbuffer_decode.slang:115-117) and the other passes read the blob's bytes there. */
int oxc_set_scene(OxcContext* ctx, const OxcSceneDesc* scene, void* stream);
/* dirty-range transform upload (RendererInstance.cpp:16-109,1590-1599), HOST source */
int oxc_update_transforms(OxcContext* ctx, const OxcTransformWorld* transforms, uint32_t first, uint32_t count, void* stream);
/* zero_fill_pass on the persistent mask (RendererInstance.cpp:1582-1588,1663) */
int oxc_reset_visibility_mask(OxcContext* ctx, void* stream);
/* vuk::clear_image(hiz, DepthZero) once per frame (RendererInstance.cpp:579-588) */
int oxc_clear_hiz(OxcContext* ctx, void* stream);

/* Multi-GPU sharding (SURVEY §8e; no reference equivalent): restrict this context to mesh instances
 * [first, first+count) — cull_meshes only expands those, so meshlet_instances / survivors are this
 * rank's shard.  id_base_dev (device u32, may be NULL = 0) is added to every meshlet-instance index
 * this context emits (survivor list, vis-buffer IDs) so IDs are global across ranks. */
int oxc_set_shard(OxcContext* ctx, uint32_t first_mesh_instance, uint32_t mesh_instance_count, const uint32_t* id_base_dev);
/* Same shard, but the id base is computed by oxc_cull_meshes itself: the number of meshlet instances the mesh
 * instances below the shard emit under the same camera / flags (count-only replay of the mesh-level cull; the
 * small tables are replicated on every rank) — no inter-GPU exchange needed for global ids. */
int oxc_set_shard_auto(OxcContext* ctx, uint32_t first_mesh_instance, uint32_t mesh_instance_count);

/* cull_meshes.slang:17-85 via CullGeometry.cpp:68-117 (init_cull_meshes == true).
 * Resets visibility{0,0,0} and cull_meshlets_cmd{0,1,1} (scratch_buffer init, :97-100), then per
 * mesh instance: frustum test, LOD select, expansion into meshlet_instances (deterministic order:
 * ascending mesh instance, ascending meshlet), lod_index write-back. */
int oxc_cull_meshes(OxcContext* ctx, const OxcCullCamera* camera, uint32_t cull_flags, void* stream);

/* cull_meshlets_hiz.slang:19-88 (use_hiz != 0; CullGeometry.cpp:129-198) or
 * cull_meshlets.slang:21-73 (use_hiz == 0; CullGeometry.cpp:274-335).
 * Resets cull_triangles_cmd{0,1,1} first (CullGeometry.cpp:125-127).  Late pass = cull_flags has
 * OXC_CULL_LATE_PASS; survivors are appended after the early ones (:70-76). */
int oxc_cull_meshlets(OxcContext* ctx, const OxcCullCamera* camera, uint32_t cull_flags, int use_hiz, void* stream);

/* hiz.slang:171-267 via generate_hiz (CullGeometry.cpp:10-59): depth_dev is a device D32F image,
 * row-major width x height floats.  Fills every mip of the context's pyramid. */
int oxc_build_hiz(OxcContext* ctx, const float* depth_dev, uint32_t width, uint32_t height, void* stream);

/* Same pyramid, sampled straight from the packed 64-bit vis buffer (depth = high 32 bits): saves the
 * resolve pass between the early raster and generate_hiz.  No reference equivalent (it has a D32F image). */
int oxc_build_hiz_packed(OxcContext* ctx, const uint64_t* vis_dev, uint32_t width, uint32_t height, void* stream);

/* Multi-GPU split of generate_hiz (no reference equivalent): mip 0 is a point sample and max-over-ranks
 * commutes with sampling, so ranks exchange mip 0 only.  oxc_build_hiz_mip0_packed writes just mip 0 (texels
 * at OxcOutputs::hiz + hiz_level_offset[0]); after an all_reduce(MAX) on those texels (non-negative floats
 * order like their int32 bits) oxc_build_hiz_from_mip0 builds mips 1.. . */
int oxc_build_hiz_mip0_packed(OxcContext* ctx, const uint64_t* vis_dev, uint32_t width, uint32_t height, void* stream);
int oxc_build_hiz_from_mip0(OxcContext* ctx, void* stream);

/* cull_triangles.slang:27-90 via CullGeometry.cpp:337-403: resets draw_cmd{0,1,0,0,0}, then one
 * block per surviving meshlet of this pass (early: [0,E); late: [E,E+L)).  Requires
 * alloc_reordered_indices. */
int oxc_cull_triangles(OxcContext* ctx, const OxcCullCamera* camera, uint32_t cull_flags, void* stream);
/* Same, with north_star's small-primitive cull switched on (the reference has none, cull_triangles.slang:59-90, so this is a
 * separate opt-in entry point): a triangle that passed the near / backface test is additionally dropped when all three
 * vertices project in front of the camera and its bounding box, snapped to the 24.8 raster grid of a width x height target,
 * holds no sample centre — it cannot produce a fragment (specification: oracle/oxc_oracle.c orc_triangle_covers_no_sample).
 * The vis buffer rendered from the shorter index buffer is identical. */
int oxc_cull_triangles_small_primitive(OxcContext* ctx, const OxcCullCamera* camera, uint32_t cull_flags, uint32_t width,
                                       uint32_t height, void* stream);

/* visbuffer_clear.slang:20-28 on the packed 64-bit image (visbuffer.slang:49-79):
 * every pixel = depth 0.0 | data ~0u. */
int oxc_clear_visbuffer(OxcContext* ctx, uint64_t* vis_dev, uint32_t width, uint32_t height, void* stream);

/* Software replacement of cull_triangles + visbuffer_encode (visbuffer_encode.slang:24-74,
 * visbuffer_encode_ms.slang:110-171; DrawGeometry.cpp:104-190): per surviving meshlet of this pass,
 * per-triangle near/backface cull then rasterisation with atomicMax on asuint(depth)<<32 | data
 * (reverse-Z GreaterOrEqual == max; visbuffer.slang:72-74 packing).  Triangles with a vertex at w <= 0 or outside the
 * 2^22 snap range — geometry around the camera, which the reference's hardware rasteriser clips — are queued by the raster
 * kernel and clipped against near + the four side planes by a follow-up kernel (Sutherland-Hodgman, fan of <= 6 pieces drawn
 * with the same rules; specification + tests: oracle/oxc_oracle.c raster_triangle_clipped).  small_primitive_cull != 0
 * additionally drops triangles whose pixel bbox covers no sample centre BEFORE they are counted (north_star's
 * small-primitive cull; the reference has none, cull_triangles.slang:59-90): the image is unchanged — such a triangle
 * produces no fragment — only OxcOutputs::raster_triangle_count drops by the number culled. */
int oxc_raster_visbuffer(OxcContext* ctx, const OxcCullCamera* camera, uint32_t cull_flags, uint32_t width,
                         uint32_t height, uint64_t* vis_dev, int small_primitive_cull, void* stream);

/* ---- alpha-tested discard of the vis-buffer encode (visbuffer_encode.slang:54-66) -------------------------------------------
 * The reference's fragment shader discards a fragment of a material that has an albedo image when
 *   material.albedo_color.a * albedo_image.SampleGrad(sampler, uv).a  <  clamp(material.alpha_cutoff, 0.001, 1.0)
 * (scene.slang:51-66,92-94,115-124).  Once a material table is set, oxc_raster_visbuffer does the same: the pass's survivors
 * are split by material (one extra kernel), meshlets of materials WITHOUT an albedo image go through the unchanged raster
 * kernel, the others through k_raster_alpha, which evaluates the test per covered sample before the packed atomic max.
 * The hardware's interpolation and sampling arithmetic is not specified bit for bit, so the test is SPECIFIED here (full text:
 * oracle/oxc_oracle.c above raster_triangle; canonical binary32 order, IEEE divide):
 *   - uv at a covered sample: the raster's own integer edge functions E_a, E_b, E_c (exact, >= 0, sum = 2 * area) are the
 *     screen-space weights; perspective correction p_i = (float)E_i * (1 / w_i), l_i = p_i / ((p_a + p_b) + p_c),
 *     u = (l_a*u_a + l_b*u_b) + l_c*u_c — non-negative terms only, no cancellation for tiny or thin triangles.  Triangles that
 *     take the clip path carry uv through the Sutherland-Hodgman cuts (same t as the position).  Vertices of a mesh without
 *     texture coordinates have uv = (0, 0) (scene.slang:355-361)
 *   - filter / address / mipmap modes from the material's sampler (default: linear, linear, repeat — Texture.hpp:38-45; no
 *     anisotropy, LOD bias or clamp: the reference sets none): texel centre convention x = u * width - 0.5, weights = the f32
 *     fractions (no 8-bit weight quantisation), alpha = texel / 255
 *   - images with a mip chain (and samplers whose mag and min filters differ) select the level like SampleGrad with
 *     ddx / ddy(tex_coord) does (visbuffer_encode.slang:57-60): "fine" quad differences of the interpolated uv, the isotropic
 *     rule lambda = log2(max(|ddx(uv) * size|, |ddy(uv) * size|)) with the library's canonical log2, lambda > 0 -> min filter,
 *     else mag filter; trilinear blend of floor(lambda) and the next level, or the nearest level
 *   - NaN alpha or cutoff keeps the fragment (the comparison is false)
 * The raster_triangle_count still counts every triangle that passed the near / backface test (discard is per fragment). */
typedef struct OxcMaterial { /* SceneGPU.hpp:67-82 / scene.slang:51-66, 56 B */
  uint16_t albedo_color[4];   /* halves */
  uint16_t emissive_color[3];
  uint16_t roughness_factor;
  uint16_t metallic_factor;
  uint16_t alpha_cutoff;      /* half */
  uint32_t flags;             /* MaterialFlag, scene.slang:34-49 */
  uint32_t sampler_index;
  uint32_t albedo_image_index;
  uint32_t normal_image_index;
  uint32_t emissive_image_index;
  uint32_t metallic_roughness_image_index;
  uint32_t occlusion_image_index;
  uint16_t uv_size[2];
  uint16_t uv_offset[2];
} OxcMaterial;
#define OXC_MATERIAL_HAS_ALBEDO_IMAGE (1u << 0) /* MaterialFlag::HasAlbedoImage */
#define OXC_MATERIAL_ALPHA_MASK (1u << 8)       /* MaterialFlag::AlphaMask (informational: the encode pass tests HasAlbedoImage only) */
/* read by oxc_decode_gbuffer only */
#define OXC_MATERIAL_HAS_NORMAL_IMAGE (1u << 1)             /* MaterialFlag::HasNormalImage */
#define OXC_MATERIAL_HAS_EMISSIVE_IMAGE (1u << 2)           /* MaterialFlag::HasEmissiveImage */
#define OXC_MATERIAL_HAS_METALLIC_ROUGHNESS_IMAGE (1u << 3) /* MaterialFlag::HasMetallicRoughnessImage */
#define OXC_MATERIAL_HAS_OCCLUSION_IMAGE (1u << 4)          /* MaterialFlag::HasOcclusionImage */
#define OXC_MATERIAL_NORMAL_TWO_COMPONENT (1u << 5)         /* MaterialFlag::NormalTwoComponent */
#define OXC_MATERIAL_NORMAL_FLIP_Y (1u << 6)                /* MaterialFlag::NormalFlipY */

/* The alpha test reads byte 3 of the RGBA formats (sRGB or not: alpha is linear) and the byte of R8 as alpha.  oxc_decode_gbuffer
 * converts a texel as Vulkan does: R8 -> (r, 0, 0, 1), RG8 -> (r, g, 0, 1), sRGB rgb through the EOTF.  oxc_set_materials accepts
 * RGBA8_UNORM, RGBA8_SRGB and R8_UNORM for an albedo image; RG8_UNORM is for the decode's other images (two-component normal maps). */
enum OxcImageFormat {
  OXC_IMAGE_RGBA8_UNORM = 0,
  OXC_IMAGE_R8_UNORM = 1,
  OXC_IMAGE_RGBA8_SRGB = 2, /* glTF base colour and emissive images (AssetManager_GLTF.cpp:887) */
  OXC_IMAGE_RG8_UNORM = 3
};
typedef struct OxcAlphaImage {  /* one entry of the engine's bindless image table, the part this pass reads */
  const void* texels_dev;       /* device pointer to level 0, tightly packed rows; level l (max(1, width >> l) x max(1, height >> l)) */
  uint32_t width, height;       /*   follows level l - 1 immediately (vkCmdCopyImageToBuffer with consecutive regions).  1..65536 */
  uint32_t format;              /* OxcImageFormat */
  uint32_t level_count;         /* 0 or 1: level 0 only; at most floor(log2(max(width, height))) + 1 */
} OxcAlphaImage;
enum OxcSamplerFilter { OXC_FILTER_LINEAR = 0, OXC_FILTER_NEAREST = 1 };
enum OxcSamplerMipmapMode { OXC_MIPMAP_LINEAR = 0, OXC_MIPMAP_NEAREST = 1 };
enum OxcSamplerAddress { OXC_ADDRESS_REPEAT = 0, OXC_ADDRESS_CLAMP_TO_EDGE = 1, OXC_ADDRESS_MIRRORED_REPEAT = 2 };
typedef struct OxcSamplerDesc { /* vuk::SamplerCreateInfo subset, AssetManager_GLTF.cpp:75-120 */
  uint32_t mag_filter, min_filter; /* OxcSamplerFilter */
  uint32_t mipmap_mode;            /* OxcSamplerMipmapMode */
  uint32_t address_u, address_v;   /* OxcSamplerAddress */
} OxcSamplerDesc;
typedef struct OxcMaterialTable {
  const OxcMaterial* materials;    /* host */
  uint32_t material_count;
  const OxcAlphaImage* images;     /* host array of device images */
  uint32_t image_count;
  const OxcSamplerDesc* samplers;  /* host; may be NULL: every sampler_index then means linear, linear, repeat */
  uint32_t sampler_count;
} OxcMaterialTable;
OXC_STATIC_ASSERT(sizeof(OxcMaterial) == 56, "Material");            /* SceneGPU.hpp:67-82 */
OXC_STATIC_ASSERT(sizeof(OxcAlphaImage) == 24, "AlphaImage");
OXC_STATIC_ASSERT(sizeof(OxcSamplerDesc) == 20, "SamplerDesc");
OXC_STATIC_ASSERT(sizeof(OxcMaterialTable) == 48, "MaterialTable");
/* Copies the tables (the image texels stay where they are).  table == NULL or material_count == 0 switches the test off again.
 * OXC_E_INVALID when a material with HasAlbedoImage names an image outside the table or an image is malformed.  A mesh instance
 * whose material_index lies outside the table is rasterised as opaque and raises OXC_STATUS_BAD_MATERIAL. */
int oxc_set_materials(OxcContext* ctx, const OxcMaterialTable* table, void* stream);

/* RENDER_OVERDRAW of the encode pass (visbuffer_encode.slang:15,68-70, visbuffer_encode_ms.slang:189-191; MainGeometryContext::
 * draw_overdraw / overdraw_attachment, RendererInstance.cpp:649-679,771-776): overdraw[pixel] += 1 for every fragment of this pass's
 * survivors the fragment shader reaches its atomic with — covered sample, depth inside [0, 1], not discarded by the alpha test (table
 * of oxc_set_materials, if any).  The depth comparison plays no part (the shader's side effect and discard put it after the shader).
 * A separate launch next to oxc_raster_visbuffer (same arguments, R32UI counter image instead of the vis buffer); the image is
 * accumulated into: clear it once per frame (oxc_clear_overdraw == the reference's vis_clear_pass, which clears both images).
 * after_frame = 0: issued where the reference draws — right after the pass's oxc_raster_visbuffer, the pass's survivor count is the
 * dispatch command's.  after_frame = 1: issued once the two-pass frame has completed (the command then holds the late count): the
 * pass's range comes from the visibility record, early [0, E), late [E, E + L) (Hi-Z cull variants only: the plain
 * oxc_cull_meshlets does not maintain that record). */
int oxc_raster_overdraw(OxcContext* ctx, const OxcCullCamera* camera, uint32_t cull_flags, uint32_t width, uint32_t height,
                        uint32_t* overdraw_dev, int after_frame, void* stream);
int oxc_clear_overdraw(OxcContext* ctx, uint32_t* overdraw_dev, uint32_t width, uint32_t height, void* stream);

/* Stand-alone clip pass: walks the pass's survivors again and clips / draws exactly the triangles described above.
 * oxc_raster_visbuffer does this by itself (it queues those triangles while it rasterises, and walks the pass again when the
 * queue overflows), so a host only needs this entry point when it drives the plain raster itself; drawing a triangle twice is
 * harmless (same depth, same id). */
int oxc_raster_visbuffer_clip_pass(OxcContext* ctx, const OxcCullCamera* camera, uint32_t cull_flags, uint32_t width,
                                   uint32_t height, uint64_t* vis_dev, void* stream);

/* Splits the packed image into the reference's two attachments: R32UI vis (data, ~0u = empty) and
 * D32F depth.  Either output may be NULL. */
int oxc_resolve_visbuffer(OxcContext* ctx, const uint64_t* vis_dev, uint32_t width, uint32_t height,
                          uint32_t* vis32_dev, float* depth_dev, void* stream);

/* Depth laid down by passes outside this path (terrain, RendererInstance.cpp:862-873): vis = max(vis,
 * asuint(depth)<<32 | ~0u) per pixel. */
int oxc_merge_depth(OxcContext* ctx, uint64_t* vis_dev, const float* depth_dev, uint32_t width, uint32_t height, void* stream);
/* oxc_clear_visbuffer followed by oxc_merge_depth in one pass over the image (same result, bit for bit). */
int oxc_clear_visbuffer_with_depth(OxcContext* ctx, uint64_t* vis_dev, const float* depth_dev, uint32_t width, uint32_t height,
                                   void* stream);

/* Multi-view batched cull (the reference's analogue is cull_meshlets_hpb.slang:27-99, which loops
 * <=10 shadow clipmaps per meshlet; CullGeometry.cpp:199-273).  Reads every meshlet's bounds ONCE and
 * tests it against n_views cameras: per view  cone (directional when view_dirs != NULL,
 * cull.slang:177-179, else positional :173-175) AND frustum (:57-84).  Output: bit v of
 * view_visibility_bits[i] and view_visible_counts[v]. */
int oxc_cull_meshlets_multiview(OxcContext* ctx, const OxcCullCamera* views, uint32_t n_views, int directional,
                                void* stream);

/* Shadow-clipmap cull: passes/cull_meshlets_hpb.slang:27-99 via CullGeometry.cpp:199-273 (use_hpb).  Per meshlet:
 * directional cone test against camera->position (= -light_dir, Shadowmaps.cpp:433-463) and frustum test against the
 * coarse view `camera`; then for each clipmap whose dirty flag is set: frustum test, project_aabb with the clipmap's
 * z_near, and the hierarchical page-bitmap test test_vsm_page (cull.slang:137-166; nearest, clamped sampling of an R8UI
 * pyramid: 4 corner taps at mip = clamp(ceil(log2(box extent in pages)), 0, levels-1), visible iff any tap != 0); a
 * projection failure counts as visible; first visible clipmap wins.  Survivors are appended like the plain variant
 * (base index from cull_triangles_cmd.x, which is reset first).  Requires OxcCreateInfo::max_views >= clipmap_count and
 * hpb_levels in 1..16 (the range oxc_build_hpb accepts); OXC_E_INVALID otherwise.
 * hpb_dev layout: for level l = 0..levels-1 (side s_l = max(1, hpb_size >> l)): layers x s_l x s_l bytes, layer-major. */
typedef struct OxcVirtualClipmap { /* SceneGPU.hpp:339-343, scalar layout, 76 B */
  float projection_view_mat[16];
  int32_t page_offset[2];
  float z_near;
} OxcVirtualClipmap;
OXC_STATIC_ASSERT(sizeof(OxcVirtualClipmap) == 76, "VirtualClipmap");
int oxc_cull_meshlets_hpb(OxcContext* ctx, const OxcCullCamera* camera, const OxcVirtualClipmap* clipmaps /* host */,
                          const uint32_t* clipmap_dirty_flags /* host */, uint32_t clipmap_count, const uint8_t* hpb_dev,
                          uint32_t hpb_size, uint32_t hpb_levels, void* stream);

/* Terrain patch cull (SURVEY §8f.3): passes/terrain_cull.slang:19-83 via RendererInstance::cull_terrain
 * (Passes/Terrain.cpp:159-216).  One thread per patch: AABB from the patch grid + patch_minmax, frustum test against
 * projection_view itself, Hi-Z occlusion against the context's pyramid, own persistent visibility mask, early/late
 * semantics identical to the meshlet cull.  draw_cmd is reset to {4, 0, 0, 0} first (Terrain.cpp:168-170);
 * instance_count counts the emitted patches, visible_patches holds their indices (order unspecified). */
typedef struct OxcTerrainData { /* scene.slang:634-647, the fields the cull reads */
  float world_min[2];
  float world_size[2];
  uint32_t patch_count[2];
  float base_height;
  float height_scale;
} OxcTerrainData;
typedef struct OxcDrawIndirectCommand { uint32_t vertex_count, instance_count, first_vertex, first_instance; } OxcDrawIndirectCommand;
int oxc_cull_terrain(OxcContext* ctx, const OxcTerrainData* terrain, const float* patch_minmax_dev /* float2 per patch, row-major */,
                     const OxcCullCamera* camera, uint32_t cull_flags, uint32_t* visible_patches_dev,
                     uint32_t* patch_visibility_mask_dev, OxcDrawIndirectCommand* draw_cmd_dev, void* stream);

/* Terrain draw into the vis buffer: passes/terrain_visbuffer.slang (vs_main, hs_constants, ds_main, fs_main) via
 * RendererInstance::draw_terrain_for_visbuffer (Passes/Terrain.cpp:218-277), the consumer of oxc_cull_terrain's visible_patches and
 * draw_cmd.  The hardware tessellator leaves points open; each item states what this library commits to.  Binary32, IEEE RN, no
 * contraction, the canonical operation order (oracle/oxc_oracle_terrain_draw.c computes it; oxylus_b200/csrc/oxc_terrain.cuh is the
 * device source).
 *   1. Corners and factors.  Patch i of visible_patches is (i % patch_count.x, i / patch_count.x); corner (dx, dz) is patch_corner =
 *      world_min + (f32(patch + corner) / f32(patch_count)) * world_size, as oxc_cull_terrain forms it; p0 = (0, 0), p1 = (1, 0),
 *      p2 = (1, 1), p3 = (0, 1); its height is sampled like a domain point (item 4).  Edges as hs_constants writes them:
 *      u0 = (p0, p3), v0 = (p0, p1), u1 = (p1, p2), v1 = (p3, p2); inner[0] = max(v0, v1) (along u), inner[1] = max(u0, u1) (along v).
 *      edge_tessellation(a, b): centre = (a + b) * 0.5; radius = length(a - b) * 0.5; view_distance = max(length(centre - camera.
 *      position) - radius, camera.near_clip); projected = ((2 * radius) * projection_scale) / view_distance; factor = clamp(projected /
 *      target_edge_pixels, 1, max_tessellation), with HLSL max / min (a NaN quotient gives 1).  length(v) = sqrt((x*x + y*y) + z*z).
 *      projection_scale = (camera.resolution.y * 0.5) / (s / c), (s, c) = the library's canonical sin and cos (oxc_exact.cuh
 *      canonical_sincos) of (fov * 0x3C8EFA35) * 0.5 — fov in degrees (Camera::fov), 0x3C8EFA35 = pi / 180 in binary32 — formed
 *      once per call.
 *   2. Rounding (fractional_odd).  Each of the six factors is pinned to [1, 63] (Vulkan's maxTessellationGenerationLevel of 64, minus
 *      one for odd spacing; NaN -> 1) and rounded up to the next odd integer n = 2 * ceil((f - 1) / 2) + 1.  When all six n are 1 the
 *      patch is the two-triangle quad.  Otherwise an inner factor of 1 counts as 1 + 2^-23 and becomes 3 (Vulkan: an inner level of 1
 *      with odd spacing is rounded as if it were slightly above 1).
 *   3. Domain points and triangulation.  An edge of pinned factor f rounded to n has the points t_0 = 0 < t_1 < ... < t_n = 1: n - 2
 *      equal segments L = 1 / f and two equal shorter ones s = (f - (n - 2)) / (2 f) at its two ends (symmetric, and 0 < s <= L since
 *      n - 2 < f <= n: the fractional_odd rule of equal full segments and two symmetric fractional ones).  For 1 <= k < n / 2:
 *      t_k = s + f32(k - 1) * L; past the middle t_k = 1 - t_{n - k}, so the points are mirror images bit for bit; n = 1 gives {0, 1}.
 *      The domain (u, v) has u along p0 -> p1 and v along p0 -> p3.  The inner grid is (a_i, b_j), i = 1..N_u - 1, j = 1..N_v - 1,
 *      with a, b the points of the inner factors; its (N_u - 2)(N_v - 2) cells are split along the (a_i, b_j) - (a_i+1, b_j+1)
 *      diagonal.  Each outer edge is stitched to the inner row beside it by a merge walk over the two rows by coordinate along the edge,
 *      ties going to the outer row: from (O_0, I_0) each step adds the triangle of the next outer point when the inner row is finished
 *      or that point's coordinate is <= the next inner point's, else of the next inner point.  The four stitch strips meet on the
 *      corner diagonals (corner, inner corner), so strips and cells tile the unit square exactly: no gap, no overlap, one winding.  A
 *      patch has 2 triangles, or sum(n_edge) + 2 (N_u - 2 + N_v - 2) + 2 (N_u - 2)(N_v - 2) (7,938 at 63 everywhere).
 *   4. Heights.  sample_height(x, z) = base_height + tap * height_scale, tap = the bilinear R16Unorm tap (texel / 65535 in binary32) of
 *      the res_x x res_y heightmap at uv = ((x, z) - world_min) * inv_world_size: level 0, ClampToEdge, Vulkan's texel centres
 *      (x = u * res_x - 0.5, x0 = floor(x), weights x - x0, a + w * (b - a) per axis).  ds_main's point: e0 = lerp(p0, p1, u),
 *      e1 = lerp(p3, p2, u), (x, z) = lerp(e0, e1, v), with lerp(a, b, t) = a * (1 - t) + b * t.  That form gives b exactly at t = 1
 *      (and a at t = 0), so two neighbouring patches place bit-identical vertices along their shared edge (same factor: the same two
 *      corners in the same order; same points) and the terrain is watertight; a + (b - a) * t does not return b at t = 1.
 *   5. Raster.  clip = projection_view x (x, h, z, 1) in the meshlet raster's order (((m0 x + m4 h) + m8 z) + m12 per row), then the
 *      raster specification of oxc_raster_visbuffer (oracle/oxc_oracle.c raster_triangle): 24.8 snapping, set-up, top-left rule,
 *      depth, and the clip path for triangles across the near or side planes.  Data word TERRAIN_INSTANCE_ID << prim_bits with the
 *      id = the packing's all-ones id minus one (visbuffer.slang:16-20): 0xFFFFFE00, or 0xFFFFFF80 under OxcCreateInfo::wide_ids.
 *      Packed 64-bit max into the caller's vis buffer.  At equal depth the terrain's word beats every meshlet word (ids below the
 *      sentinel), as in the reference, where the terrain draws after the meshlets under GreaterOrEqual.
 *   6. Winding.  triangle_ccw with cullMode Back keeps the face seen from +y.  The raster draws one winding: area2 < 0 in its
 *      snapped screen coordinates (y down).  A camera above the terrain looking down with the reference's projection (P[1][1]
 *      negated) maps world x to screen x and world z to screen y with positive scales, so (u, v) = (x, z) keeps its orientation on
 *      screen and a triangle must be clockwise in (u, v) to be drawn.  Every triangle of item 3 is therefore handed to the raster
 *      clockwise in (u, v): a flat terrain seen from above is fully drawn, seen from below nothing is.
 *   7. Instances.  draw_cmd->instance_count and visible_patches are read on the device (no read-back: graph-capturable from the first
 *      call); the count is clamped to patch_count.x * patch_count.y, and a slot holding a patch index past that total draws nothing.
 * Triangles with large pixel boxes go through the context's chunk queue of oxc_raster_visbuffer (k_raster_big), so a terrain draw and
 * a meshlet raster of one context must run in stream order, not concurrently on two streams.
 * visible_patches_dev must hold patch_count.x * patch_count.y entries (oxc_cull_terrain's list).  OXC_E_INVALID before any launch
 * for NULL arguments, a zero or > 32768 extent, a zero or > 65536 heightmap side, an empty or > 2^32 - 1 patch grid, misaligned
 * pointers (heightmap 2, visible_patches and draw_cmd 4, vis 8 bytes), and a target_edge_pixels or max_tessellation that is not
 * finite or below 1. */
typedef struct OxcTerrainDrawSettings { /* TerrainData's fields the draw reads (scene.slang:634-647) and Camera::fov */
  OxcTerrainData terrain;
  float inv_world_size[2];   /* 1 / world_size (Passes/Terrain.cpp:20) */
  float target_edge_pixels;  /* default 16 */
  float max_tessellation;    /* default 64 */
  float fov;                 /* vertical field of view, degrees */
} OxcTerrainDrawSettings;
OXC_STATIC_ASSERT(sizeof(OxcTerrainDrawSettings) == 52, "TerrainDrawSettings");
int oxc_draw_terrain(OxcContext* ctx, const uint16_t* heightmap_dev, uint32_t res_x, uint32_t res_y, const OxcTerrainDrawSettings* settings,
                     const uint32_t* visible_patches_dev, const OxcDrawIndirectCommand* draw_cmd_dev, const OxcCullCamera* camera,
                     uint32_t width, uint32_t height, uint64_t* vis_dev, void* stream);

/* Vis-buffer decode, geometry part (SURVEY §8f.1): passes/visbuffer_decode.slang:42-183 via RendererInstance's
 * "vis decode" pass.  Per pixel: texel -> (meshlet instance, triangle) (visbuffer.slang:31-36), triangle re-fetch
 * (scene.slang:363-399), world positions, compute_partial_derivatives (:42-92: analytic perspective-correct
 * barycentrics lambda and their per-pixel derivatives), gradient_of the vertex texture coordinates (:33-40) and the
 * geometric world normal normalize(mul(lambda, to_world_normals)) (:146-147) oct-encoded (common/encoding.slang:17-21).
 * The material evaluation (texture sampling, tangent frame from the sampled normal map, :118-183) is oxc_decode_gbuffer's,
 * below.  The frame's oxc_cull_meshes must have run (it resolves
 * LODs and pointers).  Exactly one of vis64_dev (our packed image) / vis32_dev (the reference's R32UI attachment).
 * Targets are float4-per-pixel planes, any may be NULL:
 *   lambda    = (lambda.xyz, status)  status 0: discarded (clear / terrain texel, :97-99), 1: decoded,
 *                                     2: a vertex index >= Mesh::vertex_count (:115-117, zero output)
 *   ddx / ddy = (d lambda / d pixel x|y .xyz, 0)
 *   uv_normal = (uv.xy, oct(world_normal).xy)       uv_grad = (uv ddx.xy, uv ddy.xy)
 * Meshes without normals / texture coordinates (OxcMesh::vertex_normals / texture_coords == 0) decode them as 0. */
typedef struct OxcDecodeTargets {
  float* lambda;
  float* ddx;
  float* ddy;
  float* uv_normal;
  float* uv_grad;
} OxcDecodeTargets;
int oxc_decode_visbuffer(OxcContext* ctx, const OxcCullCamera* camera, const uint64_t* vis64_dev, const uint32_t* vis32_dev,
                         uint32_t width, uint32_t height, const OxcDecodeTargets* targets /* host struct of device ptrs */,
                         void* stream);

/* Vis-buffer decode into the G-buffer: passes/visbuffer_decode.slang:88-183 with the material functions of scene.slang:110-159.  Same
 * inputs and preconditions as oxc_decode_visbuffer (exactly one of vis64_dev / vis32_dev, the frame's oxc_cull_meshes has run), and
 * the material table of the last oxc_set_materials (OXC_E_STATE without one).  Four float4 planes, row-major, 16-byte aligned; any
 * may be NULL, and a NULL target's images are not sampled:
 *   albedo                       rgba                                          (SV_Target0)
 *   normal                       oct(mapped normal).xy, oct(world normal).zw   (SV_Target1; .zw == oxc_decode_visbuffer's uv_normal.zw,
 *                                                                               so the plane feeds oxc_vsm_resolve_shadows as is)
 *   emissive                     rgb, w = 0                                    (SV_Target2)
 *   metallic_roughness_occlusion metallic, roughness, occlusion, w = 0         (SV_Target3)
 * SPECIFICATION (oracle/oxc_oracle_gbuffer.c orc_decode_gbuffer, bit for bit): IEEE binary32, no contraction, sums in written order.
 *   1. a pixel oxc_decode_visbuffer discards is NOT written (a fragment discard keeps the attachment's contents); a vertex index
 *      >= vertex_count, and a mesh instance whose material_index lies outside the table (it raises OXC_STATUS_BAD_MATERIAL), write
 *      zeros to every target.
 *   2. lambda, its derivatives, the world positions and the world normal n: exactly oxc_decode_visbuffer's arithmetic.
 *   3. uv = uv * uv_size + uv_offset, uv_ddx *= uv_size, uv_ddy *= uv_size (dequantize_half of the material's halves).
 *   4. SampleGrad per image (level-0 size w0 x h0, the material's sampler): mx = uv_ddx.u * w0, my = uv_ddx.v * h0, nx = uv_ddy.u * w0,
 *      ny = uv_ddy.v * h0; from there the level rule of the alpha test above (canonical log2, mag / min choice, clamp, trilinear or
 *      nearest level) and its per-channel filter order.  No anisotropy, LOD bias or clamp.
 *   5. a texel becomes RGBA before filtering: RGBA8_UNORM c / 255; RGBA8_SRGB rgb = the binary32 nearest to the sRGB EOTF of c / 255,
 *      a = c / 255; R8_UNORM (r / 255, 0, 0, 1) — what Vulkan returns; the alpha test keeps reading R8 as alpha; RG8_UNORM
 *      (r / 255, g / 255, 0, 1).
 *   6. albedo = albedo_color * sample (HasAlbedoImage) or albedo_color.
 *   7. p_i = world_i - camera.position; pos_ddx = (ddx0*p0 + ddx1*p1) + ddx2*p2 (ddy likewise); pos_ddx_s = pos_ddx - dot(pos_ddx, n)*n;
 *      js = sign(uv_ddx.x*uv_ddy.y - uv_ddx.y*uv_ddy.x) (NaN -> 0); T = js*(uv_ddy.y*pos_ddx_s - uv_ddx.y*pos_ddy_s), normalized if
 *      js != 0; w = js*sign(dot(pos_ddy, cross(n, pos_ddx))); B = -w*cross(n, T).  HasNormalImage: s = sample.rgb*2 - 1, NormalFlipY
 *      negates s.y, NormalTwoComponent sets s.z = sqrt(saturate(1 - (s.x*s.x + s.y*s.y))) (saturate(NaN) = 0), normal =
 *      normalize((s.x*T + s.y*B) + s.z*n); else normal = n.  normalize(v) = v / sqrt(dot(v, v)).
 *   8. emissive = emissive_color * sample.rgb or emissive_color; (metallic, roughness) = factors * sample.bg or the factors;
 *      occlusion = sample.r or 1.
 * Images named by a flag other than HasAlbedoImage are checked here, not by oxc_set_materials: OXC_E_INVALID, naming the material
 * and the slot, when one lies outside the image table or fails the albedo checks (null or not 4-byte aligned texels, extent,
 * level_count, format), or when the material's sampler has an unknown mode.  Texels are read in software as aligned 32-bit words.
 * No scratch: graph-capturable from the first call. */
typedef struct OxcGBufferTargets { /* host struct of device pointers; float4 per pixel, row-major, 16-byte aligned; any may be NULL */
  float* albedo;
  float* normal;
  float* emissive;
  float* metallic_roughness_occlusion;
} OxcGBufferTargets;
OXC_STATIC_ASSERT(sizeof(OxcGBufferTargets) == 32, "GBufferTargets");
int oxc_decode_gbuffer(OxcContext* ctx, const OxcCullCamera* camera, const uint64_t* vis64_dev, const uint32_t* vis32_dev,
                       uint32_t width, uint32_t height, const OxcGBufferTargets* targets, void* stream);

/* Hierarchical page bitmap build (SURVEY §8f.4): passes/rmvsm_downsample_hpb.slang:15-33 dispatched per level by
 * Shadowmaps.cpp:331-366.  Level 0: byte = page is visible && backed && dirty (VSMPageState bits 1 | 4 | 2,
 * rmvsm.slang:16-28) for every entry of the layers x size x size R32UI virtual page table; level k: 2x2 OR of
 * level k-1.  Output layout == the hpb_dev input of oxc_cull_meshlets_hpb. */
int oxc_build_hpb(OxcContext* ctx, const uint32_t* page_table_dev, uint32_t page_table_size, uint32_t layers,
                  uint8_t* hpb_dev, uint32_t hpb_levels, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Multi-GPU exchange (SURVEY §8e, §8b oxc_mgpu_*; the reference is single-GPU).  One context per GPU / process, mesh instances
 * sharded with oxc_set_shard_auto.  Per frame a sharded host runs
 *     clear, cull_meshes, cull_meshlets(early), raster      (local)
 *     oxc_mgpu_exchange_hiz                                 instead of oxc_build_hiz_packed
 *     cull_meshlets(late), raster                           (local)
 *     oxc_mgpu_exchange_frame                               merged image + everybody's survivor lists
 * and gets bit for bit what one GPU computes for the whole scene (max / set union are associative and commutative).
 *
 * oxc_mgpu_init is COLLECTIVE (every rank calls it): it creates the NCCL communicator from the 128-byte id rank 0 obtained with
 * oxc_mgpu_get_unique_id and handed to the other ranks by any means (the tests broadcast it with torch.distributed; an MPI
 * or socket broadcast does as well), and maps every peer's Hi-Z exchange buffer with CUDA IPC.  oxc_mgpu_init_with_comm adopts
 * a communicator the host already owns (ncclComm_t passed as void*).  NCCL itself is dlopen'ed on first use.
 *
 * exchange_hiz: the rank's point-sampled mip-0 texels are max-reduced directly into every peer's exchange buffer over NVLink
 * peer memory by the sampling kernel itself (only the texels the rank drew a fragment into travel), a per-rank flag is the
 * barrier, then every rank builds the identical pyramid.  Without peer access it falls back to ncclAllReduce(max) of mip 0.
 * exchange_frame: ncclAllReduce(ncclUint64, ncclMax) of the packed vis buffer in place (NULL skips it) + ncclAllGather of
 * {total, early, late, gathered} counters and of fixed-capacity survivor-id segments into the buffers OxcMgpuInfo names; a rank
 * whose survivors exceed survivor_capacity raises OXC_STATUS_SURVIVOR_OVERFLOW (oxc_check_status) — never a silent truncation.
 * ---------------------------------------------------------------------------------------------- */
#define OXC_MGPU_ID_BYTES 128
typedef struct OxcMgpuInfo {
  uint32_t active, rank, world;
  uint32_t survivor_capacity;       /* ids per rank segment */
  uint32_t hiz_over_peer_memory;    /* 1: NVLink peer-memory reduction; 0: NCCL fallback */
  uint32_t* gathered_counts[2];     /* device, per slot: world x {total, early, late, ids gathered} */
  uint32_t* gathered_ids[2];        /* device, per slot: world segments of survivor_capacity global meshlet-instance ids */
} OxcMgpuInfo;
int oxc_mgpu_get_unique_id(uint8_t id[OXC_MGPU_ID_BYTES]);
int oxc_mgpu_init(OxcContext* ctx, uint32_t rank, uint32_t world, const uint8_t id[OXC_MGPU_ID_BYTES],
                  uint32_t survivor_capacity /* 0 = max_meshlet_instances; the ranks agree on the largest value requested */);
int oxc_mgpu_init_with_comm(OxcContext* ctx, void* nccl_comm, uint32_t survivor_capacity);
/* Collective: changes the survivor segment capacity (the ranks agree on the largest value requested; gather buffers are
 * reallocated, OxcMgpuInfo pointers change).  Typical use: init generously, run a few exchanged frames, shrink to a multiple of
 * the survivor counts actually seen — the allgather moves whole segments. */
int oxc_mgpu_set_survivor_capacity(OxcContext* ctx, uint32_t survivor_capacity);
int oxc_mgpu_shutdown(OxcContext* ctx);
int oxc_mgpu_info(OxcContext* ctx, OxcMgpuInfo* out);
int oxc_mgpu_exchange_hiz(OxcContext* ctx, const uint64_t* vis_dev, uint32_t width, uint32_t height, void* stream);
/* A host that overlaps the exchange of frame i (side stream) with frame i + 1 (main stream) copies the frame's survivor list and
 * counters into the slot's staging buffers ON THE MAIN STREAM first (oxc_mgpu_stage_survivors: the context's own list is
 * rewritten by the next frame's cull), then calls oxc_mgpu_exchange_frame with OXC_MGPU_ALREADY_STAGED on the side stream. */
#define OXC_MGPU_ALREADY_STAGED 1u
int oxc_mgpu_stage_survivors(OxcContext* ctx, int slot, void* stream);
int oxc_mgpu_exchange_frame(OxcContext* ctx, uint64_t* vis_dev /* may be NULL */, uint32_t width, uint32_t height, int slot,
                            uint32_t flags, void* stream);

/* VSM page marking (SURVEY §8f.4): passes/rmvsm_mark_visible_pages.slang:19-84 dispatched by Shadowmaps.cpp after the depth
 * pre-pass.  One thread per depth pixel (depth == 0 = sky, skipped): unproject (scene.slang:189-193), clipmap level from the
 * world-space footprint of the pixel diagonal (rmvsm.slang:156-186: log2(d / first_clipmap_texel_length), bias, clamp),
 * project into that clipmap (rmvsm.slang:214-221), page coordinates (:200-206) wrapped by the clipmap's page offset (:129-138),
 * then  prev = atomicOr(page_table[layer][y][x], Visible);  a page that was not visible before is either recorded in
 * page_occupancy[physical address] (already backed) or pushed as an allocation request {x, y, layer}.
 * Canonical arithmetic as everywhere (IEEE f32, no contraction); log2 is the library's own polynomial evaluated with those
 * operations (oxc_exact.cuh canonical_log2 == oracle orc_log2_canonical), so CPU oracle and GPU agree bit for bit — the
 * reference's driver log2 under SLANG fast-math is not bit-defined either.  Deviation: pixels whose page coordinates are
 * invalid are skipped; the reference's wave-scalarisation loop lets the first lane of a wave through with them (:64-74), an
 * out-of-bounds image atomic whose effect depends on the wave composition.
 * Request ORDER is unspecified (atomics), as in the reference. */
typedef struct OxcVsmContext { /* rmvsm.slang:116-127 VSMContext, scalar layout */
  int32_t page_size;
  int32_t page_table_size;
  int32_t physical_page_table_size;
  int32_t curr_clipmap_index;
  int32_t clipmap_count;          /* <= 10 (shared_clipmaps[10], :17) */
  int32_t depth_extent[2];
  float first_clipmap_width;
  float clipmap_selection_bias;
  float virtual_extent;
  float z_length;
  float directional_light_dir[3];
} OxcVsmContext;
int oxc_mark_visible_pages(OxcContext* ctx, const float inv_projection_view[16] /* Camera::inv_projection_view, column-major */,
                           const float resolution[2], const OxcVirtualClipmap* clipmaps /* host, clipmap_count entries */,
                           const OxcVsmContext* vsm, const float* depth_dev, uint32_t* page_tables_dev /* [clipmap][size][size] */,
                           uint32_t* page_occupancy_dev, uint32_t* request_count_dev, int32_t* requests_dev /* int3 per request */,
                           uint32_t request_capacity, void* stream);

/* ---- VSM page bookkeeping (SURVEY §8f.4): the passes of Shadowmaps.cpp:100-430 between the depth image and the shadow raster ----
 * One frame is, on one stream (oxr_vsm_update_pages runs exactly this):
 *   oxc_vsm_begin_frame         vuk::clear_image on sun_moved (:143-148), rmvsm_reset_page_visibility (:150-163), zero-filled
 *                               page_occupancy (:224-232) and request count
 *   oxc_vsm_invalidate_pages    rmvsm_invalidate_pages (:167-222), only when !sun_moved and there are dirty mesh instances
 *   oxc_mark_visible_pages      rmvsm_mark_visible_pages (:234-275), request_count_dev = &allocator->active_request_count
 *   oxc_vsm_allocate_pages      rmvsm_free_invisible_pages, rmvsm_build_free_page_list, rmvsm_allocate_pages (:277-329) and
 *                               rmvsm_mark_dirty_pages (:373-406)
 *   oxc_build_hpb               rmvsm_downsample_hpb (:331-371)
 *   oxc_vsm_clear_dirty_pages   rmvsm_clear_dirty_pages (:408-431)
 * then oxc_cull_meshlets_hpb_dirty_dev culls the shadow casters against the new bitmap.  Everything stays on the device: no call
 * reads a count back, so the sequence can be captured into a CUDA graph.
 * Page table entries: rmvsm.slang:16-34 (Visible 1, Dirty 2, Backed 4, Invalidated 8, AllocationFailed 16; physical page index in
 * bits 16-31).  The physical atlas is an R32F image of physical_page_table_size^2 texels, row-major; physical page p sits at page
 * coordinates (p % n, p / n), n = physical_page_table_size / page_size.
 * Where the reference's outcome depends on the atomics order of the marking or the wave order of the allocation, the library
 * commits to one admissible outcome (specification: oracle/oxc_oracle_vsm.c orc_vsm_*):
 *   - free list: physical pages with occupancy 0 in ascending order
 *   - allocation: the first min(active_request_count, request_capacity) requests are read; one naming an entry outside the table
 *     is skipped (the reference would store out of bounds).  Requests are ranked by the linear address (layer * size + y) * size + x
 *     of their entry; d requests for one entry take d consecutive free-list slots and the entry gets the highest of them below
 *     free_page_count.  An entry whose first slot is past the free count is left unchanged: the reference sets AllocationFailed
 *     on a local copy and returns without storing it.  alloc_cursor = slots handed out
 *   - dirty list: ascending page table address; clipmap_dirty_flags[l] is 0 or 1 for every l < clipmap_count
 *   - invalidation, deviation: every page a box covers is invalidated.  The reference visits the pages of 8 x 8 page sections
 *     with section index < DIRECTIONAL_PAGE_TABLE_SIZE (64 per clipmap): the whole table at its size 64, but for other sizes it
 *     misses the pages beyond 8 * floor(size / 8) and every section past the 64th
 *   - arithmetic as everywhere: IEEE binary32, no contraction, project_aabb of cull.slang:12-47.
 * Every entry point returns OXC_E_INVALID for a null pointer, clipmap_count outside 1..10, page_table_size < 1, a page_size that
 * does not divide physical_page_table_size, more than 65536 physical pages (the 16-bit address) or a physical_page_count other
 * than (physical_page_table_size / page_size)^2. */
typedef struct OxcVsmAllocator { /* rmvsm.slang:228-236 VSMPageAllocator, scalar layout, 40 B (device memory) */
  uint32_t active_request_count;          /* written by oxc_mark_visible_pages, zeroed by oxc_vsm_begin_frame */
  uint32_t dirty_physical_page_count;     /* entries of dirty_physical_page_coords (the clear dispatch's z) */
  uint32_t free_page_count;
  uint32_t alloc_cursor;
  int32_t* requests;                      /* int3 {x, y, layer} per request */
  uint32_t* dirty_physical_page_coords;   /* u32x2 per dirty physical page */
  uint32_t* free_page_list;
} OxcVsmAllocator;
OXC_STATIC_ASSERT(sizeof(OxcVsmAllocator) == 40, "VSMPageAllocator");
/* page_tables_dev[clipmap][size][size]: cleared when sun_moved, else Visible, Dirty and Invalidated cleared (Backed,
 * AllocationFailed, the address and the other bits stay); occupancy_dev[0, physical_page_count) = 0; *request_count_dev = 0. */
int oxc_vsm_begin_frame(OxcContext* ctx, const OxcVsmContext* vsm, int sun_moved, uint32_t* page_tables_dev, uint32_t* occupancy_dev,
                        uint32_t physical_page_count, uint32_t* request_count_dev, void* stream);
/* rmvsm_invalidate_pages.slang:19-111: for every dirty mesh instance (indices into the scene's mesh instances, device) and
 * clipmap, the mesh's bounds (OxcMesh::bounds) under the previous (previous_transforms_dev[transform_index], device) and the
 * current world matrix: project_aabb(clipmap.projection_view_mat * world, z_near), a failed projection invalidates nothing;
 * the clamped uv box covers pages floor(uv_min * size) .. ceil(uv_max * size) - 1, wrapped by the clipmap's page offset; every
 * Backed entry there becomes exactly Invalidated (8).  A dirty index outside the mesh instance table is skipped.  Needs
 * oxc_set_scene; invalidates whenever it is called (the frame sequence skips it on sun_moved). */
int oxc_vsm_invalidate_pages(OxcContext* ctx, const OxcVsmContext* vsm, const OxcVirtualClipmap* clipmaps /* host */,
                             const uint32_t* dirty_mesh_instances_dev, uint32_t dirty_count, const OxcTransformWorld* previous_transforms_dev,
                             uint32_t* page_tables_dev, void* stream);
/* Free invisible pages, free list, allocation and dirty list in one launch (one CTA: the tables are small and a single block
 * makes every scan run in address order).  Writes the allocator's counters and its three pointers (requests_dev, dirty_coords_dev,
 * free_list_dev).  free_list_dev holds physical_page_count entries; dirty_coords_dev holds clipmap_count * size^2 u32x2 entries
 * (any entry may be dirty) and is the kernel's scratch for the per-entry request counts; clipmap_dirty_flags_dev holds
 * clipmap_count u32. */
int oxc_vsm_allocate_pages(OxcContext* ctx, const OxcVsmContext* vsm, uint32_t* page_tables_dev, const uint32_t* occupancy_dev,
                           uint32_t physical_page_count, const int32_t* requests_dev, uint32_t request_capacity, OxcVsmAllocator* allocator_dev,
                           uint32_t* free_list_dev, uint32_t* dirty_coords_dev, uint32_t* clipmap_dirty_flags_dev, void* stream);
/* rmvsm_clear_dirty_pages.slang:12-25: every texel of each of the allocator's dirty pages = 1.0f (the count is read on the
 * device).  A page whose coordinates lie outside the atlas is not written (the image store would be discarded). */
int oxc_vsm_clear_dirty_pages(OxcContext* ctx, const OxcVsmContext* vsm, const OxcVsmAllocator* allocator_dev, const uint32_t* dirty_coords_dev,
                              float* physical_atlas_dev, void* stream);
/* oxc_cull_meshlets_hpb with the clipmap dirty flags read from DEVICE memory (clipmap_count u32, e.g. the flags
 * oxc_vsm_allocate_pages wrote), as the reference binds them (CullGeometry.cpp:214-259): no read-back mid-frame. */
int oxc_cull_meshlets_hpb_dirty_dev(OxcContext* ctx, const OxcCullCamera* camera, const OxcVirtualClipmap* clipmaps /* host */,
                                    const uint32_t* clipmap_dirty_flags_dev, uint32_t clipmap_count, const uint8_t* hpb_dev,
                                    uint32_t hpb_size, uint32_t hpb_levels, void* stream);

/* The VSM shadow raster into the physical atlas: the last step of draw_virtual_shadowmap (Shadowmaps.cpp:433-754,
 * rmvsm_build_draw_commands.slang, rmvsm_draw_physical_pages.slang), drawn in software.  Draws the survivors of the context's
 * last oxc_cull_meshlets_hpb / _hpb_dirty_dev (its list and count stay on the device) into physical_atlas_dev (R32F,
 * physical_page_table_size^2 texels, row-major, written through its R32UI view).  Specification (oracle/oxc_oracle_vsm_draw.c
 * orc_vsm_draw_pages, bit for bit):
 *   - triangles: exactly those cull_triangles keeps with the COARSE camera (all three clip.z >= 0 and det < 1e-4 of PV . W,
 *     cull_triangles.slang:62-69), evaluated once per triangle;
 *   - for every clipmap c with clipmap_dirty_flags_dev[c] != 0 (read on the device): clip = mul(clipmaps[c].projection_view_mat,
 *     (mul(world, (p, 1)).xyz, 1)) in the canonical order; raster target W = H = physical_page_table_size;
 *   - the raster specification of oxc_raster_visbuffer (24.8 snapping, pixel-centre samples, top-left tie-break, z = (za + E_b*dzb)
 *     + E_c*dzc) drawing BOTH windings (cullMode None: a triangle of the other winding is re-oriented; zero area draws nothing);
 *     triangles with a vertex at w <= 0 or beyond the 2^22 snap range go through the vis raster's Sutherland-Hodgman clipper;
 *   - per sample, in f32 in the shader's order: virtual_uv = (px + 0.5, py + 0.5) / physical_page_table_size, page =
 *     i32(floor(virtual_uv * page_table_size)) wrapped by the clipmap's page_offset (rmvsm.slang:129-138); only an entry that is
 *     Backed && Dirty is written, whatever its Visible bit; texel = physical page coordinates * page_size +
 *     i32(mod(floor(virtual_uv * physical_page_table_size), page_size)); a texel outside the atlas is not written;
 *   - the alpha test of oxc_set_materials (the same as the vis-buffer encode's, uv carried through the clipper);
 *   - the sink: fragments with z outside [0, 1] are dropped, texel = min(texel bits, asuint(z)) as u32 (-0 stored as +0).
 * Deviation: the depth is NDC z = clip.z / clip.w.  The reference writes SV_Position.z / SV_Position.w, which is NDC z for the
 * orthographic clipmaps it builds (w = 1) whichever convention the compiler uses for SV_Position.w.
 * The context's scratch (page bitmap, work queue) is allocated by the first call: capture the call into a CUDA graph after one
 * eager call.  Same argument checks as the other oxc_vsm_* calls, plus physical_page_table_size <= 16384 (the snap range);
 * OXC_E_STATE without a scene or before oxc_cull_meshes. */
int oxc_vsm_draw_pages(OxcContext* ctx, const OxcVsmContext* vsm, const OxcCullCamera* coarse, const OxcVirtualClipmap* clipmaps /* host */,
                       const uint32_t* clipmap_dirty_flags_dev, const uint32_t* page_tables_dev, float* physical_atlas_dev, void* stream);
/* Counters of the last oxc_vsm_draw_pages on `stream` (synchronous): out[0] = (triangle, clipmap, dirty page) work items,
 * out[1] = (meshlet, clipmap) pairs whose page rectangle held a dirty page and so reached triangle work. */
int oxc_vsm_draw_stats(OxcContext* ctx, uint32_t out[2], void* stream);

/* The VSM shadow resolve: RendererInstance::resolve_shadowmap (Shadowmaps.cpp:756-822, passes/resolve_shadowmaps.slang:27-209 with
 * the rmvsm.slang helpers it calls), the consumer of the physical atlas.  One value per pixel of the depth_extent[0] x
 * depth_extent[1] image into shadow_dev (R32F, row-major): 1 = lit, 0 = shadowed, the PCF fraction in between.  Inputs are only
 * read: depth_dev (D32F, 0 = sky), normals_dev (float4 per pixel, oct(world normal) in .zw: the uv_normal plane of
 * oxc_decode_visbuffer, 0 where the decode discards), page_tables_dev [clipmap][size][size], physical_atlas_dev
 * (physical_page_table_size^2 R32F).  Specification (oracle/oxc_oracle_vsm_resolve.c orc_vsm_resolve_shadows, bit for bit), in
 * IEEE binary32 with no contraction, IEEE divide / sqrt, dot = (x*x' + y*y') + z*z', mul in row order:
 *   - pixel (x, y): position = (x + 0.5, y + 0.5), tex_coord = position / depth_extent; depth == 0 gives 1;
 *   - normal: both .zw components rounded to binary16 (round to nearest even; the reference's attachment is R16G16B16A16Sfloat),
 *     then normalize(oct_to_vec3(e)) (common/encoding.slang:7-15, which normalizes once itself), normalize(v) = v / sqrt(dot(v, v));
 *   - world point: unproject (scene.slang:189-193); clipmap: exactly oxc_mark_visible_pages' rule (canonical_log2, bias, ceil,
 *     saturating u32, clamp to clipmap_count - 1);
 *   - PCSS (:84-185): 1 centre tap, 16 blocker-search taps, up to 24 PCF taps; noise = hash2(position) (:27-30); a tap looks up the
 *     base clipmap, then base - 1, then base + 1 (indices -1 and clipmap_count miss); a page outside the table or not Backed misses;
 *     a fetched value equal to -1.0 counts as a miss, as in the shader; pow(2, k + 1) is exact; fract(x) = x - floor(x);
 *     lerp(a, b, t) = a + (b - a) * t; base_bias = (quantize + b) + term; max / min return the other operand for a NaN;
 *     accum_depth_world is summed in sample order; hammersley2d(i, N) = (i / N, reversebits(i) * 2^-32);
 *   - sin / cos: the library's own canonical_sincos (oxc_exact.cuh == oracle orc_sincos_canonical): binary64 reduction by
 *     pi/2 and Taylor polynomials, one rounding to binary32; <= 1 ulp on [0, 2 pi], <= 2^-24 absolute for |x| <= 2^21.  The
 *     reference's driver sin / cos under fast-math are not bit-defined.
 * Deviation: a physical address whose texel lies outside the atlas reads 0.0, what robustImageAccess returns (the draw does not
 * write such a texel).  No scratch: graph-capturable from the first call.  Same argument checks as the other oxc_vsm_* calls,
 * plus depth_extent >= 1 and a 16-byte aligned normals_dev. */
int oxc_vsm_resolve_shadows(OxcContext* ctx, const OxcVsmContext* vsm, const float inv_projection_view[16], const float resolution[2],
                            const OxcVirtualClipmap* clipmaps /* host */, const float* depth_dev, const float* normals_dev,
                            const uint32_t* page_tables_dev, const float* physical_atlas_dev, float* shadow_dev, void* stream);

/* Ambient occlusion: RendererInstance::generate_ambient_occlusion (Passes/PBR.cpp:143-311), the visibility-bitmask GTAO of
 * passes/gtao/vbgtao_prefilter.slang, vbgtao_main.slang and vbgtao_denoise.slang.  Three passes in stream order over a width x height
 * frame: the depth prefilter (linear depth, 5 mips), the sector pass (edges and noisy occlusion) and the 3 x 3 edge-aware denoise.
 * Inputs are only read: depth_dev (D32F, reversed Z, 0 = sky), normals_dev (float4 per pixel, oct(world normal) in .zw: the uv_normal
 * plane of oxc_decode_visbuffer or the normal plane of oxc_decode_gbuffer, which carry the same .zw).  The caller owns every plane
 * (OxcGtaoTargets), so the call uses no scratch and is graph-capturable from its first call.  camera.resolution is (width, height).
 * Refused with OXC_E_INVALID: a NULL argument or target, a zero extent or one above 32768, slice_count outside 1..OXC_GTAO_MAX_SLICES,
 * samples_per_slice_side outside 1..OXC_GTAO_MAX_SAMPLES_PER_SIDE, normals_dev not 16-byte aligned, a plane not naturally aligned.
 * SPECIFICATION (oracle/oxc_oracle_gtao.c orc_generate_ambient_occlusion, bit for bit): IEEE binary32, no contraction, IEEE divide /
 * sqrt, sums and products in written order, dot(a, b) = (a.x*b.x + a.y*b.y) + a.z*b.z, mul(M, v) row by row in the same order.
 *   1. linearize(d) = m23 / (d + m22), (m23, m22) = (projection[3][2], projection[2][2]) (glm [column][row], PBR.cpp:183-186).
 *   2. virtual pyramid: level 0 at any (x, y) >= 0 is linearize(depth[min(y, H-1)][min(x, W-1)]); level k at t is
 *      weighted_average(L(k-1, 2t), L(k-1, 2t + (1, 0)), L(k-1, 2t + (0, 1)), L(k-1, 2t + (1, 1))) (vbgtao_prefilter.slang:23-39 with
 *      its own constants).  Only the texels inside max(1, W >> k) x max(1, H >> k) are stored (depth_mips: levels 0..4 packed in
 *      order, each row-major).  This is what the reference's 16 x 16-pixel groups compute, including values from beyond the extent.
 *   3. gathers and point samples are integer texel reads with clamp to edge: the edges read mip 0 at the pixel and its left, right,
 *      top (y - 1) and bottom (y + 1) neighbours; the normal is the pixel's own; the denoise reads the 3 x 3 neighbourhood of the
 *      noisy plane and the pixel and its four direct neighbours of the edges plane.
 *   4. edges (vbgtao_main.slang:69-100): e = (left, right, top, bottom) - centre, slopes, min(|e|, |e + slope|), saturate(1.25 - e /
 *      (centre * 0.011)), packUnorm4x8 = round to nearest even of saturate(c) * 255, .x in the low byte.  Written for every pixel.
 *   5. sky: centre linear depth >= far_clip * 0.999 writes 1 to the noisy plane.
 *   6. SampleLevel(linear_clamp, uv, lambda): levels floor(lambda) and min(floor(lambda) + 1, 4), weight lambda - floor(lambda), both
 *      always read; each level bilinear at uv * size - 0.5 with binary32 weights, top = a00 + wx * (a10 - a00), bottom likewise,
 *      top + wy * (bottom - top), clamp to edge, NaN-safe saturating texel indices; blend (1 - f) * lo + f * hi.  No 8-bit weight
 *      quantisation (deviation, as the alpha test's).  lambda = clamp(canonical_log2(length(offset * resolution)) - 3.3, 0, 4).
 *   7. normal: .zw rounded to binary16 (round to nearest even; the reference's attachment is R16G16B16A16Sfloat), oct_to_vec3 (which
 *      normalizes), mul(view, (n, 0)).xyz, normalize; normalize(v) = v / sqrt(dot(v, v)), length(v) = sqrt(dot(v, v)).
 *   8. noise: index = the reference's 64 x 64 Hilbert index (RendererInstance.cpp:151-170) at (x % 64, y % 64) + 288 * (noise_index
 *      % 64), then frac(0.5 + float(index) * (0.754877666, 0.569840291)) (R2).
 *   9. cos / sin of the slice angle: canonical_sincos (as oxc_vsm_resolve_shadows); fast_acos as written; sign(NaN) = 0,
 *      saturate(NaN) = 0, max / min return the other operand for a NaN, u32(x) truncates and saturates (NaN -> 0), frac(x) = x -
 *      floor(x), countbits = popcount; constants are the binary32 roundings of the shader literals.
 *  10. a NaN texel of the mip chain is stored as 0x7FFFFFFF; the noisy occlusion is stored as binary16 (round to nearest even,
 *      R16F) and read back from it; the final AO is pow(max(denoised, 0), final_power) with canonical_pow (oxc_exact.cuh), written
 *      as binary32 (the value before the reference's R16F store).
 * Hostile depth (NaN, Inf, denormal, negative), normals and settings do not fault and follow the same rules. */
#define OXC_GTAO_MAX_SLICES 16u
#define OXC_GTAO_MAX_SAMPLES_PER_SIDE 8u
typedef struct OxcGtaoSettings { /* SceneGPU.hpp:286-293 VBGTAOSettings */
  float thickness;
  uint32_t slice_count;            /* 1..OXC_GTAO_MAX_SLICES (the reference's presets use 1..9) */
  uint32_t samples_per_slice_side; /* 1..OXC_GTAO_MAX_SAMPLES_PER_SIDE (the presets use 2..3) */
  float effect_radius;
  uint32_t noise_index;
  float final_power;
} OxcGtaoSettings;
typedef struct OxcGtaoCamera {     /* the Camera fields the three passes read (scene.slang:162-188) */
  float projection[16];            /* column-major, as Camera::projection */
  float view[16];                  /* column-major, as Camera::view */
  float far_clip;
} OxcGtaoCamera;
typedef struct OxcGtaoTargets {    /* device pointers, all required */
  float* depth_mips;               /* levels 0..4, level k = max(1, W>>k) x max(1, H>>k) row-major, packed in order */
  uint32_t* edges;                 /* "vbgtao depth differences", R32UI, W x H */
  uint16_t* noisy_occlusion;       /* "vbgtao noisy occlusion", binary16, W x H */
  float* ambient_occlusion;        /* W x H */
} OxcGtaoTargets;
OXC_STATIC_ASSERT(sizeof(OxcGtaoSettings) == 24, "GtaoSettings");
OXC_STATIC_ASSERT(sizeof(OxcGtaoCamera) == 132, "GtaoCamera");
OXC_STATIC_ASSERT(sizeof(OxcGtaoTargets) == 32, "GtaoTargets");
int oxc_generate_ambient_occlusion(OxcContext* ctx, const OxcGtaoCamera* camera, const OxcGtaoSettings* settings, const float* depth_dev,
                                   const float* normals_dev, uint32_t width, uint32_t height, const OxcGtaoTargets* targets, void* stream);

/* Lighting: the pbr_apply_no_atmos variant of RendererInstance::apply_pbr (Passes/PBR.cpp:435-531, passes/pbr_apply_no_atmos.slang
 * :23-127 with the pbr.slang:1-172 functions it calls).  One float4 (RGBA) per pixel of a width x height frame, row-major, into out_dev,
 * from caller-owned device planes; no scratch, so the call is graph-capturable from its first call.  Inputs (OxcPbrInputs):
 *   depth (D32F, reversed Z, 0 = sky); albedo, normal, emissive, metallic_roughness_occlusion: float4 per pixel as oxc_decode_gbuffer
 *   writes them (normal = oct(normal-mapped normal) in .xy, oct(world normal) in .zw); optional, NULL reads as 1.0 (the reference clears
 *   both attachments to White): ambient_occlusion (f32, as oxc_generate_ambient_occlusion writes it) and shadow (f32, as
 *   oxc_vsm_resolve_shadows writes it); contact_shadow (f32), read only under OXC_SCENE_HAS_CONTACT_SHADOWS and then required.
 * lights_dev: settings->light_count OxcLight records (the reference's lights buffer), 16-byte aligned, summed in index order.
 * Refused with OXC_E_INVALID: a NULL required argument or plane, NULL lights with light_count > 0, a NULL contact plane under
 * OXC_SCENE_HAS_CONTACT_SHADOWS, a zero extent or one above 32768, light_count > OXC_MAX_LIGHTS (the reference uploads at most 256),
 * OXC_SCENE_HAS_ATMOSPHERE (that variant needs the sky LUTs), float4 planes, out_dev or lights_dev not 16-byte aligned, f32 planes not
 * 4-byte aligned.  The other flag bits (bloom, FXAA, ...) are ignored, as the shader ignores them.
 * SPECIFICATION (oracle/oxc_oracle_pbr.c orc_apply_pbr, bit for bit): IEEE binary32, no contraction, IEEE divide / sqrt, products and
 * sums left to right as written, dot(a, b) = (a.x*b.x + a.y*b.y) + a.z*b.z, mul(M, v) row by row in the same order (+ M[i][3] * 1.0),
 * normalize(v) = v / sqrt(dot(v, v)), length(v) = sqrt(dot(v, v)), lerp(a, b, t) = a + (b - a) * t, reflect(i, n) = i - (2 * n) *
 * dot(i, n), max / min return the other operand for a NaN, clamp(x, a, b) = min(max(x, a), b), saturate(NaN) = 0, smoothstep(e0, e1, x)
 * = (t * t) * (3 - 2 * t) with t = saturate((x - e0) / (e1 - e0)); constants are the binary32 roundings of the shader's literals;
 * Fd_Lambert = fl(1 / fl(pi)).  Commitments where the shader leaves the outcome open:
 *   1. pixel centre: tex_coord = ((x + 0.5) / W, (y + 0.5) / H); the albedo's SampleLevel at a pixel centre has bilinear weights of
 *      exactly 0, so it is the pixel's own texel.
 *   2. the normal plane's four components are rounded to binary16 (R16G16B16A16F, round to nearest even); both oct_to_vec3
 *      (common/encoding.slang:7-15, which normalizes) follow the written order; N is normalized a second time, as written.
 *   3. the ambient occlusion is rounded to binary16 (R16F); albedo, emissive, metallic / roughness / occlusion, shadow and contact
 *      shadow are read as the binary32 values given (deviation: the reference stores the first three as RGBA8 sRGB, B10G11R11 and
 *      RGBA8 unorm, conversions that are not bit-defined).
 *   4. cos of the cone angles: canonical_sincos; exp2(-16 r - 1) = canonical_pow(2, .); pow(NoV + ao, .) = canonical_pow;
 *      pow(., 5.0) of F_Schlick = canonical_pow5 (oxc_exact.cuh: binary64 x^2, (x^2 * x^2) * x, one rounding; within 1 ulp).
 *   5. a light kind other than OXC_LIGHT_POINT / OXC_LIGHT_SPOT contributes nothing (the shader's if / else if).
 *   6. early returns in shader order: OXC_SCENE_TRANSPARENT_BACKGROUND and depth == 0 gives (0, 0, 0, 0); then OXC_SCENE_HAS_SKY and
 *      depth == 0 gives sky_has_texture ? (1, 1, 1, 1) : sky_solid_color; otherwise the full computation runs, also on sky pixels
 *      without OXC_SCENE_HAS_SKY, with whatever non-finite values follow.
 *   7. output: binary32 RGBA, the value before the reference's B10G11R11 / RGBA16F store (deviation); every NaN is written as
 *      0x7FFFFFFF.  Hostile planes, lights and settings (NaN, Inf, denormals) do not fault and follow the same rules. */
#define OXC_MAX_LIGHTS 256u                          /* GPU::MAX_LIGHTS */
#define OXC_SCENE_HAS_DIRECTIONAL_LIGHT (1u << 0)     /* SceneFlags, SceneGPU.hpp:253-267 */
#define OXC_SCENE_HAS_ATMOSPHERE (1u << 1)
#define OXC_SCENE_HAS_EYE_ADAPTATION (1u << 2)
#define OXC_SCENE_HAS_BLOOM (1u << 3)
#define OXC_SCENE_HAS_FXAA (1u << 4)
#define OXC_SCENE_HAS_GTAO (1u << 5)
#define OXC_SCENE_HAS_FILM_GRAIN (1u << 6)
#define OXC_SCENE_HAS_CHROMATIC_ABERRATION (1u << 7)
#define OXC_SCENE_HAS_VIGNETTE (1u << 8)
#define OXC_SCENE_HAS_CONTACT_SHADOWS (1u << 9)
#define OXC_SCENE_HAS_SKY (1u << 10)
#define OXC_SCENE_TRANSPARENT_BACKGROUND (1u << 11)
#define OXC_LIGHT_DIRECTIONAL 0u                     /* LightKind */
#define OXC_LIGHT_POINT 1u
#define OXC_LIGHT_SPOT 2u
typedef struct OxcLight {          /* GPU::Light, SceneGPU.hpp:241-251 */
  float position[3];
  float intensity;
  float color[3];
  float range;                     /* <= 0: no window, 1 / (d^2 + 0.1) */
  float direction[3];              /* spot only, normalized by the pass */
  float inner_cone_angle;          /* spot only, radians */
  float outer_cone_angle;          /* spot only, radians */
  uint32_t kind;                   /* OXC_LIGHT_* */
  uint32_t pad[2];
} OxcLight;
typedef struct OxcPbrSettings {    /* the pass's specialization constant and push constants (PBR.cpp:436-486) */
  uint32_t scene_flags;            /* OXC_SCENE_* */
  float sun_direction[3];          /* L, used as given */
  float sun_intensity;             /* Li */
  float base_ambient_color[3];     /* the reference passes 0.03 */
  float sky_solid_color[4];        /* Sky (scene.slang:236-240) */
  float sky_ambient_color[3];
  uint32_t sky_has_texture;
  uint32_t light_count;            /* 0..OXC_MAX_LIGHTS */
} OxcPbrSettings;
typedef struct OxcPbrCamera {      /* the Camera fields the pass reads (scene.slang:162-188) */
  float inv_projection_view[16];   /* column-major, as Camera::inv_projection_view */
  float position[3];
} OxcPbrCamera;
typedef struct OxcPbrInputs {      /* device planes, W x H, row-major */
  const float* depth;              /* required, f32 */
  const float* albedo;             /* required, float4 */
  const float* normal;             /* required, float4 */
  const float* emissive;           /* required, float4 */
  const float* metallic_roughness_occlusion; /* required, float4 */
  const float* ambient_occlusion;  /* optional (NULL = 1.0), f32 rounded to binary16 */
  const float* shadow;             /* optional (NULL = 1.0), f32, read under OXC_SCENE_HAS_DIRECTIONAL_LIGHT */
  const float* contact_shadow;     /* f32, read (and required) only under OXC_SCENE_HAS_CONTACT_SHADOWS */
} OxcPbrInputs;
OXC_STATIC_ASSERT(sizeof(OxcLight) == 64, "Light");
OXC_STATIC_ASSERT(sizeof(OxcPbrSettings) == 68, "PbrSettings");
OXC_STATIC_ASSERT(sizeof(OxcPbrCamera) == 76, "PbrCamera");
OXC_STATIC_ASSERT(sizeof(OxcPbrInputs) == 64, "PbrInputs");
int oxc_apply_pbr(OxcContext* ctx, const OxcPbrCamera* camera, const OxcPbrSettings* settings, const OxcLight* lights_dev,
                  const OxcPbrInputs* inputs, uint32_t width, uint32_t height, float* out_dev, void* stream);

/* Contact shadows: RendererInstance's contact_shadows pass (RendererInstance.cpp:990-1020, passes/contact_shadows.slang:29-78 with the
 * raymarch.slang DepthRayMarch / HybridRootFinder / DepthRaymarchDistanceFn code it calls).  One f32 per pixel of a width x height
 * frame, row-major, into out_dev: 1 - shadow, the plane oxc_apply_pbr reads under OXC_SCENE_HAS_CONTACT_SHADOWS.  depth_dev (D32F,
 * reversed Z, 0 = sky) is only read; no scratch, so the call is graph-capturable from its first call.  Sky pixels are marched like any
 * other pixel, as the shader does; PBR apply's own early returns decide what they show.
 * Refused with OXC_E_INVALID, before anything is launched: a NULL argument, a zero extent or one above 32768, steps outside
 * 1..OXC_CONTACT_SHADOW_MAX_STEPS (the reference's editor range; the bound keeps the march at most 64 taps per pixel for any depth),
 * depth_dev or out_dev not 4-byte aligned.  NaN or Inf thickness, length and sun direction are accepted and follow the rules below.
 * SPECIFICATION (oracle/oxc_oracle_contact_shadows.c orc_contact_shadows, bit for bit): IEEE binary32, no contraction, IEEE divide /
 * sqrt, sums and products in written order, dot(a, b) = (a.x*b.x + a.y*b.y) + a.z*b.z (two components: a.x*b.x + a.y*b.y), mul(M, v)
 * row by row in the same order, normalize(v) = v / sqrt(dot(v, v)), length(v) = sqrt(dot(v, v)); sign(NaN) = 0, saturate(NaN) = 0,
 * max / min return the other operand for a NaN, u32(x) truncates and saturates (NaN -> 0), pow(x, 1.0) = x, lerp(0, 1, t) = 0 + (1 -
 * 0) * t, smoothstep(e0, e1, x) = (t * t) * (3 - 2 * t) with t = saturate((x - e0) / (e1 - e0)) (also for e0 > e1); constants are the
 * binary32 roundings of the shader's literals, and (1.0 + bias) is fl(1 + fl(2e-6)) = 0x3F800011 (a Slang literal without suffix is a
 * float; folding the sum in binary64 and rounding once gives the same bits).  For pixel (x, y):
 *   1. uv = ((x + 0.5) / W, (y + 0.5) / H); depth = the nearest tap at uv; cs = (uv * 2 - 1, depth); h = mul(inv_projection_view,
 *      (cs, 1)); ws = h.xyz / h.w.
 *   2. end = ws + normalize(sun_direction) * length; end_cs = (mul(projection, mul(view, (end, 1)))).xyz / w (to_ws); dir = (end_cs -
 *      cs, 0) * sign(end_cs.z) (to_cs); e = (cs, 1) + dir, e /= (e.w >= 0 ? 1 : -1) * max(1e-10, |e.w|), as written.
 *   3. start clip: delta = e.xyz - cs, near = delta < 0 ? (1, 1, 1) : (-1, -1, 0) per component, k = max((near.x - cs.x) / delta.x,
 *      (near.y - cs.y) / delta.y), start = cs + delta * max(0, k).  End clip: delta = e.xyz - start, far = delta >= 0 ? (1, 1, 1) :
 *      (-1, -1, 0), m = min(min(fx, fy), fz) of (far - start) / delta, delta *= min(1, m), end = start + delta.
 *   4. march: uv_s / uv_e = start.xy / end.xy * 0.5 + 0.5, n = max(2, min(steps, u32(floor(length((uv_e - uv_s) * (W, H)) / 1)))),
 *      depth_thickness = thickness * (1 / near_clip).  Steps i = 0..n-1 at t = 0 + (1 - 0) * ((i + 1) / n): p = start + (end - start) *
 *      t, uv = p.xy * 0.5 + 0.5, lin = 1 / bilinear(uv), unf = 1 / nearest(uv), distance = max(lin, unf) * (1 + bias) - 1 / p.z,
 *      penetration = 1 / p.z - min(lin, unf).  The first step with distance < 0 is the candidate; the pixel is in contact when
 *      penetration < depth_thickness and distance < depth_thickness, and then shadow = smoothstep(1, 0.3, penetration /
 *      depth_thickness); otherwise shadow = 0.
 *   5. nearest tap at uv: texel (floor(u * W), floor(v * H)) with NaN-safe saturating indices (oxc_shader_math.cuh sat_i32), clamped to
 *      the edge.  Bilinear tap at uv: x = u * W - 0.5, x0 = floor(x), wx = x - x0 (y likewise), texels x0, x0 + 1 / y0, y0 + 1 with the
 *      same index rule, top = a00 + wx * (a10 - a00), bottom = a01 + wx * (a11 - a01), top + wy * (bottom - top): the GTAO's level tap
 *      (oxc_generate_ambient_occlusion item 6).  Deviation: no 8-bit quantisation of the weights, as the alpha test's.
 *   6. output: 1 - shadow as binary32 (the value of the reference's R32F store); it lies in [0, 1] and is never NaN.
 * Hostile depth (NaN, Inf, denormal, negative) and settings do not fault and follow the same rules. */
#define OXC_CONTACT_SHADOW_MAX_STEPS 64u
typedef struct OxcContactShadowCamera { /* the Camera fields the pass reads (scene.slang:162-188), column-major */
  float inv_projection_view[16];
  float view[16];
  float projection[16];
  float near_clip;
} OxcContactShadowCamera;
typedef struct OxcContactShadowSettings { /* the pass's push constants (contact_shadows.slang:15-20, RendererCVar.cpp:30-34) */
  float sun_direction[3];          /* DirectionalLight::direction, normalized by the pass */
  uint32_t steps;                  /* 1..OXC_CONTACT_SHADOW_MAX_STEPS, the reference's default 8 */
  float thickness;                 /* world units at the near plane, default 0.1 */
  float length;                    /* world-space ray length, default 0.01 */
} OxcContactShadowSettings;
OXC_STATIC_ASSERT(sizeof(OxcContactShadowCamera) == 196, "ContactShadowCamera");
OXC_STATIC_ASSERT(sizeof(OxcContactShadowSettings) == 24, "ContactShadowSettings");
int oxc_contact_shadows(OxcContext* ctx, const OxcContactShadowCamera* camera, const OxcContactShadowSettings* settings, const float* depth_dev,
                        uint32_t width, uint32_t height, float* out_dev, void* stream);

/* Atmosphere lookup tables: the transmittance bake (RendererInstance.cpp:203-226, passes/sky_transmittance.slang) and the per-frame sky
 * view and aerial perspective (Passes/PBR.cpp:11-50 and :96-140, passes/sky_view.slang and passes/sky_aerial_perspective.slang), with the
 * sky.slang / common/math.slang functions they call, on the path the reference takes: no multiple-scattering LUT (eval_multiscattering is
 * false at every call site, so the LUT the reference binds is never sampled), no ground bounce (eval_planet_luminance is false in all three
 * passes).  Each plane holds binary16 RGBA texels (8 B), row-major, x fastest, then y, then z, at the sizes the record gives:
 *   transmittance       transmittance_lut_size.xy: (exp(-optical_depth), 1), 1000 march steps per texel;
 *   sky view            sky_view_lut_size.xy: (L / m, m), m = clamp(max(L.r, L.g, L.b), 2^-14, 65504), 48 steps;
 *   aerial perspective  aerial_perspective_lut_size.xyz: (L, mean transmittance), 2 (z + 1) steps in slice z.
 * oxc_atmosphere_sky_luts taps transmittance_dev (as oxc_atmosphere_transmittance wrote it) and writes both per-frame planes in one launch.
 * No scratch, so both calls are graph-capturable from their first call.  The z sizes of the transmittance and sky-view LUTs and
 * multiscattering_lut_size are not read; terrain_albedo, aerial_perspective_start_km and aerial_perspective_exposure are read only by the
 * passes that consume the tables (the record is the engine's, kept whole).
 * Refused with OXC_E_INVALID, before anything is launched: a NULL argument or plane, a plane not 8-byte aligned, a size the call reads that
 * is 0 or above 4096 (transmittance x / y for both calls; sky view x / y and aerial perspective x / y / z for oxc_atmosphere_sky_luts), a
 * sky-view dimension below 2 (from_sub_uvs_to_unit divides by res - 1), an aerial-perspective depth above 256 (so no thread marches more
 * than 512 steps).  NaN, Inf and denormal atmosphere, camera and sun values are accepted and follow the rules below.
 * SPECIFICATION (oracle/oxc_oracle_atmosphere.c, bit for bit): IEEE binary32, no contraction, IEEE divide / sqrt, sums and products in
 * written order, dot(a, b) = (a.x*b.x + a.y*b.y) + a.z*b.z, mul(M, v) row by row in the same order, normalize(v) = v / sqrt(dot(v, v)),
 * length(v) = sqrt(dot(v, v)), lerp(a, b, t) = a + (b - a) * t, max / min return the other operand for a NaN (equal operands give the
 * second), clamp(x, a, b) = min(max(x, a), b), safe_sqrt(x) = sqrt(max(0, x)); constants are the binary32 roundings of the shaders'
 * literals: PI 0x40490FDB, TAU 0x40C90FDB, CAMERA_SCALE_UNIT 0x3C23D70A, PLANET_RADIUS_OFFSET 0x3A83126F, HALF_MIN_NORMAL 0x38800000,
 * HALF_MAX 0x477FE000, and the folded 1 / (4 PI) = fl(1 / fl(4 * PI)) = 0x3DA2F983, 3 / (16 PI) = 0x3D747645, 1.0 / 3.0 = 0x3EAAAAAB
 * (4 * PI and 16 * PI are exact, so folding in binary32 or in binary64 with one rounding gives the same bits), 3.0 / 2.0 = 1.5.
 * Commitments where the shaders leave the outcome open:
 *   1. exp is canonical_exp (oxc_exact.cuh, binary32 Cody-Waite, within 1 ulp, exp(+-0) = 1, overflow to +inf, underflow through the
 *      subnormals to +0); cos is canonical_cos; pow(x, 3/2) is canonical_pow; acos (beta, constant per call) is canonical_acos (binary64,
 *      one rounding), and so are computed once per call: get_eye_pos, h = length((0, y, 0)) = sqrt(fl(y * y)) (not |y|), beta, PI - beta,
 *      and the four exps of mie_asymmetry of henyey_greenstein_draine_phase.
 *   2. the sky view divides the moved eye position by h before the move (so above the atmosphere the sun frame is per texel), as written.
 *   3. Optional<f32>::value of `none` reads 0: the bake takes the exit distance without checking it, which only a record with atmos_radius
 *      below planet_radius (or NaN) can miss; those texels march 1000 steps of length 0.
 *   4. the MS * scattering_sum term of sun_luminance is kept with MS = 0, so an infinite or NaN sum gives NaN, as in the shader.
 *   5. the transmittance tap: x = u * W - 0.5, x0 = floor(x), wx = x - x0 (y likewise), texels x0, x0 + 1 / y0, y0 + 1 with NaN-safe
 *      saturating indices clamped to the edge, top = a00 + wx * (a10 - a00), bottom likewise, top + wy * (bottom - top), reading the
 *      binary16 texels exactly: the GTAO's level tap without the 8-bit weight quantisation (deviation, as for the alpha test).
 *   6. every texel is stored as binary16 RGBA, rounded to nearest even with subnormals kept, +-inf beyond 65504; every NaN as 0x7FFF.
 *      The aerial perspective does not sanitize: an atmosphere with zero extinction stores 0 / 0 = NaN.
 *   7. the sky view's max(L, 0) returns 0 for a NaN before sanitize replaces +-inf by 0.
 *   8. the aerial perspective's per_slice_depth is f32(size.x / size.z) in integers (1 at 32^3, 0 when z > x); its start_depth,
 *      start_pos and ray_pos are dead (view_height is reassigned before they are read) and not computed.
 * Texel centres are ((x + 0.5) / W, (y + 0.5) / H).  The loops are bounded by 1000, 48 and 2 (z + 1) <= 512 whatever the values. */
#define OXC_ATMOSPHERE_MAX_LUT_SIZE 4096u
#define OXC_ATMOSPHERE_MAX_AERIAL_DEPTH 256u
typedef struct OxcAtmosphere {      /* GPU::Atmosphere (SceneGPU.hpp:158-181), scalar layout */
  float rayleigh_scatter[3];
  float rayleigh_density;
  float mie_scatter[3];
  float mie_density;
  float mie_extinction;
  float mie_asymmetry;
  float ozone_absorption[3];
  float ozone_height;
  float ozone_thickness;
  float terrain_albedo[3];
  float planet_radius;
  float atmos_radius;
  float aerial_perspective_start_km;
  float aerial_perspective_exposure;
  uint32_t transmittance_lut_size[3];
  uint32_t sky_view_lut_size[3];
  uint32_t multiscattering_lut_size[3];
  uint32_t aerial_perspective_lut_size[3];
} OxcAtmosphere;
OXC_STATIC_ASSERT(sizeof(OxcAtmosphere) == 136, "Atmosphere");
int oxc_atmosphere_transmittance(OxcContext* ctx, const OxcAtmosphere* atmosphere, uint16_t* lut_dev, void* stream);
/* camera: inv_projection_view and position of the frame's camera (the aerial perspective's ray directions; both passes' eye height);
 * sun_direction and sun_intensity: DirectionalLight::direction and ::intensity, as given. */
int oxc_atmosphere_sky_luts(OxcContext* ctx, const OxcAtmosphere* atmosphere, const OxcPbrCamera* camera, const float sun_direction[3],
                            float sun_intensity, const uint16_t* transmittance_dev, uint16_t* sky_view_dev, uint16_t* aerial_perspective_dev,
                            void* stream);

/* The sky IBL cube (Passes/PBR.cpp:52-94, passes/sky_ibl.slang, RendererInstance.cpp:187-201 and :1022): the sky light of each of 6
 * faces x 32 x 32 texels, 64 cosine-weighted taps of the sky-view LUT per texel around the texel's direction (sky.slang:296-322
 * get_atmosphere_illuminance_along_ray), plus a sun term, accumulated frame to frame.  The reference runs it every frame under
 * HasAtmosphere && HasDirectionalLight, after the sky view, with sun_ambient_strength 0.15 and frame_index = the engine's frame counter.
 * cube_dev: 6 x 32 x 32 binary16 RGBA texels (48 KiB), face-major, then y, then x fastest; faces 0..5 look along +X, -X, +Y, -Y, +Z, -Z.
 * It is read and written in place: a texel with a > 0 and finite rgb is history, so a zeroed cube (the reference clears it to black)
 * means no history.  transmittance_dev and sky_view_dev are the LUTs oxc_atmosphere_transmittance and oxc_atmosphere_sky_luts wrote,
 * at the record's transmittance_lut_size.xy and sky_view_lut_size.xy; of the camera only the position is read.  No scratch, so the
 * call is graph-capturable; a captured graph replays the frame_index it was captured with.
 * Refused with OXC_E_INVALID, before anything is launched: a NULL argument or plane, a plane not 8-byte aligned, a transmittance size
 * 0 or above 4096, a sky-view size below 2 or above 4096, a cube that shares a byte with either LUT.  NaN, Inf and denormal values in
 * the record, camera, sun, intensities and cube are accepted and follow the rules below.
 * SPECIFICATION (oracle/oxc_oracle_sky_ibl.c, bit for bit): the atmosphere rules above (binary32, no contraction, written order, dot,
 * normalize, length, lerp, max / min with NaN, clamp, safe_sqrt, saturate(x) = min(max(x, 0), 1), its constants and its items 1, 5 and 6),
 * cross(a, b) = (a.y*b.z - a.z*b.y, a.z*b.x - a.x*b.z, a.x*b.y - a.y*b.x), frac(x) = x - floor(x), sanitize(x) = isfinite(x) ? x : 0,
 * f32(u32) rounds to nearest even; constants 0.999 0x3F7FBE77, IGN's 0.06711056 0x3D897143, 0.00583715 0x3BBF4590, 52.9829189
 * 0x4253EE82, 0.61803398875 0x3F1E377A, 2.3283064365386963e-10 0x2F800000, alpha 0.02 0x3CA3D70A, 1e-20 0x1E3CE508, 1e-5 0x3727C5AC,
 * 2.0 * PI = TAU.  For texel (x, y) of face f:
 *   1. uv = (f32(x, y) + 0.5) / 32, dir = normalize(mul(M_f, (uv * 2 - 1, -1))), M_f the shader's mat3 literals read by rows and
 *      mul(M, v) row by row; up = |dir.y| < 0.999 ? (0, 1, 0) : (1, 0, 0), tangent = normalize(cross(up, dir)), bitangent =
 *      cross(dir, tangent).
 *   2. history = the texel as stored, binary16 read exactly; has_history = a > 0 && all(isfinite(rgb)) (NaN, +-inf, a <= 0 or a NaN alpha
 *      mean none).  base = IGN(f32(x, y) + f32(f) * (37, 17)), IGN(p) = frac(52.9829189 * frac(p.x * 0.06711056 + p.y * 0.00583715));
 *      rotation = has_history ? frac(base + f32(frame_index) * 0.61803398875) : base.
 *   3. sample i of 64: u1 = (f32(i) + 0.5) / 64, u2 = frac(radical_inverse_vdc(i) + rotation) (exact for i < 64), phi = TAU * u2, cos and
 *      sin of phi by canonical_sincos, local = (sqrt(u1) cos, sqrt(u1) sin, sqrt(max(0, 1 - u1))), input = normalize((x * tangent +
 *      y * bitangent) + z * dir).  Its value is sanitize(get_atmosphere_illuminance_along_ray(sun, eye, input)) with eye = (0, eye_y, 0):
 *      height = eye_h, up = eye / height and the normalized sun once per call; side = length(cross(up, input)) > 1e-5 ? normalize(that)
 *      : (1, 0, 0); forward = normalize(cross(side, up)); light_on_plane = safe_normalize((dot(sun, forward), dot(sun, side)), (1, 0)),
 *      safe_normalize(v, f) = len2 > 1e-20 ? v * rsqrt(len2) : f with rsqrt(x) = fl(1 / fl(sqrt(x))) (two roundings, where the shader's
 *      rsqrt is approximate); intersect_planet = ray_sphere_intersect_nearest(eye, input, planet_radius).hasValue; then
 *      sky_view_params_to_lut_uv with the per-call beta and PI - beta, acos(dot(input, up)) by canonical_acos (binary64, the same bits on
 *      the device and the host) and atan2(-l.y, -l.x) by canonical_atan2 (binary64, one rounding, within 1 ulp, C99 special cases), and
 *      from_unit_to_sub_uvs; the tap (atmosphere item 5, all four channels) of the sky-view LUT; sanitize(rgb * a).  For a finite
 *      height up is exactly (0, 1, 0) (sqrt(fl(y * y)) = |y|), so the view-zenith cosine is input.y and rounding cannot push it past 1;
 *      an acos argument past +-1 or NaN (a NaN up, from an infinite or NaN height) gives NaN, which reaches safe_sqrt: max(0, NaN) = 0,
 *      so v = 0.5, the horizon row, in both branches.
 *   4. estimate = (((0 + s_0) + s_1) + ... + s_63) / 64 per channel, in index order.  sun term = (((0.15 * T) * sun_intensity) *
 *      saturate(dot(dir, sun))) / PI with the sun as given (not normalized) and T the transmittance tap at
 *      transmittance_params_to_lut_uv(atmos_radius, planet_radius, (eye_y, dot(sun, (0, 1, 0)))); sun_ambient_strength for 0.15.
 *   5. result = min(max(sanitize(estimate + sun term), 0), 65504); stored = has_history ? lerp(history.rgb, result, 0.02) : result, as
 *      (stored, 1) in binary16 (atmosphere item 6).  A finite history and a result in [0, 65504] keep the stored rgb finite: it is never
 *      NaN; a negative finite history decays toward the result. */
#define OXC_SKY_IBL_CUBE_RES 32u
#define OXC_SKY_IBL_SAMPLES 64u
#define OXC_SKY_IBL_CUBE_BYTES (6u * OXC_SKY_IBL_CUBE_RES * OXC_SKY_IBL_CUBE_RES * 8u)
int oxc_atmosphere_sky_ibl(OxcContext* ctx, const OxcAtmosphere* atmosphere, const OxcPbrCamera* camera, const float sun_direction[3],
                           float sun_intensity, float sun_ambient_strength, uint32_t frame_index, const uint16_t* transmittance_dev,
                           const uint16_t* sky_view_dev, uint16_t* cube_dev, void* stream);

/* Lighting under the atmosphere: the pbr_apply variant of RendererInstance::apply_pbr (Passes/PBR.cpp:312-432, passes/pbr_apply.slang
 * :26-184 with the sky.slang functions it calls), which the reference runs instead of oxc_apply_pbr's when the scene has an
 * AtmosphereComponent (HasAtmosphere, RendererInstance.cpp:1442-1460).  One float4 (RGBA) per pixel into out_dev, from the planes and
 * lights oxc_apply_pbr takes (same layouts and alignment) and the sky's four binary16 RGBA planes (OxcPbrSky): the transmittance LUT as
 * oxc_atmosphere_transmittance wrote it, the sky-view and aerial-perspective LUTs as oxc_atmosphere_sky_luts wrote them, the cube as
 * oxc_atmosphere_sky_ibl wrote it.  No scratch, so the call is graph-capturable from its first call.  Settings read: scene_flags,
 * sun_direction (L, as given), sun_intensity (Li), light_count; base_ambient_color and the sky_* fields are not read (the shader overwrites
 * both sky terms) and HasSky changes nothing.  Atmosphere fields read: planet_radius, atmos_radius, aerial_perspective_start_km,
 * aerial_perspective_exposure and the transmittance, sky-view and aerial-perspective sizes.
 * Refused with OXC_E_INVALID, before anything is launched: everything oxc_apply_pbr refuses except OXC_SCENE_HAS_ATMOSPHERE; settings
 * WITHOUT OXC_SCENE_HAS_ATMOSPHERE (that bit selects this shader); a NULL record, sky or sky plane; a sky plane not 8-byte aligned; the LUT
 * sizes oxc_atmosphere_sky_luts refuses.  NaN, Inf and denormal values in the LUTs, cube, record, camera, settings and planes are accepted.
 * SPECIFICATION (oracle/oxc_oracle_pbr_atmosphere.c orc_apply_pbr_atmosphere, bit for bit): oxc_apply_pbr's rules and its items 1-3, 5
 * and 7 (pixel centre, binary16 normal plane and AO, binary32 G-buffer reads, light kinds, output with every NaN 0x7FFFFFFF), the
 * atmosphere's rules (oxc_atmosphere_transmittance: get_eye_pos, canonical_exp / canonical_acos / canonical_atan2, the tap of item 5
 * reading binary16 exactly), cross(a, b) = (a.y*b.z - a.z*b.y, a.z*b.x - a.x*b.z, a.x*b.y - a.y*b.x), normalize of a 2-vector = v /
 * sqrt(v.x*v.x + v.y*v.y).  Commitments where the shader leaves the outcome open:
 *   1. order: TransparentBackground and depth == 0 gives (0, 0, 0, 0); then the prologue, with the pixel's sun transmittance; then
 *      depth == 0 takes the sky path (item 4) and every other pixel the full path.
 *   2. per call, on the host: sun_cos_theta = dot(L, (0, 1, 0)); horizon_darkening = smoothstep(-0.1, 0.3, sun_cos_theta); draw_sun's
 *      min_cos = canonical_cos(fl(fl(1 * PI) / 180)) with the argument 0x3C8EFA35; the camera's eye = get_eye_pos(camera.position) with
 *      altitude h = eye.y as written (not length(eye) as the IBL), horizon = safe_sqrt(h*h - R*R), beta = canonical_acos(horizon / h),
 *      PI - beta.
 *   3. sun transmittance: the transmittance tap at transmittance_params_to_lut_uv(atmos_radius, planet_radius, (get_eye_pos(world).y,
 *      sun_cos_theta)), rgb; direct = (T * Li) * horizon_darkening per channel, not gated by HasDirectionalLight (the shadow read is).
 *   4. sky pixels: right = normalize(cross(up, -V)) with no fallback (NaN for a vertical view, which follows the rules), forward =
 *      normalize(cross(right, up)), light_on_plane = plain normalize((dot(L, forward), dot(L, right))), the planet hit from the camera's
 *      eye, sky_view_params_to_lut_uv as for the IBL, the sky-view tap on all four channels; without a planet hit rgb += (draw_sun(-V, L)
 *      * Li) * T per channel, draw_sun = cos >= min_cos ? 1 : canonical_exp(-offset * 50000) * 0.5 + (1 / (0.02 + offset * 300)) * 0.01
 *      with offset = min_cos - cos, cos = dot(-V, L).  Output (rgb * a, 1); there is no HasSky early return in this shader.
 *   5. aerial perspective (sky.slang:258-293): per_slice_depth = f32(size.x) / f32(size.z), a binary32 division (the LUT pass's item 8
 *      divides integers; the two differ at 32 x 32 x 24); rcp(x) = fl(1 / x); half_slice_depth 0x3F3504F3; near_depth_fade_out = 1.0 /
 *      0.001 folded in binary32 like the other folds, fl(1 / fl(0.001)) = 0x4479FFFF (a binary64 fold would give 0x447A0000).  The 3D tap
 *      is item 5's bilinear rule in slices z0 = floor(w * D - 0.5) and z0 + 1 (same NaN-safe clamped indices), then s0 + wz * (s1 - s0).
 *      Then rgb *= weight, a = 1 - weight * (1 - a), rgb *= exposure; the contribution is rgb * a.
 *   6. cube tap (TextureCube.SampleLevel, linear, level 0): the face by the major axis as in the Vulkan specification's cube map face
 *      selection table, ties to X over Y over Z (X when |x| >= |y| and |x| >= |z|, else Y when |y| >= |z|), the positive face when the
 *      major component is >= 0 (so -0 too); s = 0.5 * (sc / |ma|) + 0.5, t likewise; x = s * 32 - 0.5, the 2 x 2 footprint of item 5
 *      with indices in -1..32.  Seamless, as the specification's cube map edge handling: a texel one step off an edge is the adjacent
 *      face's texel that shares the edge; a corner texel (off both edges, which the specification leaves to the implementation) is
 *      ((inside + across x) + across y) / 3 of the three texels that meet there.  A NaN or zero direction (normalize(lerp(N, R, 1 -
 *      roughness)) is 0 / 0 for R = -N at roughness 0.5) selects by the same comparisons (all NaN: face 5; zero: face 0), reads texels 0 and
 *      1 (NaN-safe indices) and returns NaN.  specular_sky = (rgb * a) * horizon_darkening at that direction, diffuse_sky likewise at N.
 *   7. sum: ((((surface + lights) + indirect) + emission) + aerial), indirect as oxc_apply_pbr's with the two sky terms, surface with the
 *      per-channel direct. */
typedef struct OxcPbrSky {               /* the atmosphere variant's extra inputs, binary16 RGBA, 8-byte aligned */
  const uint16_t* transmittance;         /* transmittance_lut_size.xy, as oxc_atmosphere_transmittance wrote it */
  const uint16_t* sky_view;              /* sky_view_lut_size.xy, as oxc_atmosphere_sky_luts wrote it */
  const uint16_t* aerial_perspective;    /* aerial_perspective_lut_size.xyz */
  const uint16_t* sky_cube;              /* 6 x 32 x 32, oxc_atmosphere_sky_ibl's layout */
} OxcPbrSky;
OXC_STATIC_ASSERT(sizeof(OxcPbrSky) == 32, "PbrSky");
int oxc_apply_pbr_atmosphere(OxcContext* ctx, const OxcPbrCamera* camera, const OxcPbrSettings* settings, const OxcAtmosphere* atmosphere,
                             const OxcLight* lights_dev, const OxcPbrInputs* inputs, const OxcPbrSky* sky, uint32_t width, uint32_t height,
                             float* out_dev, void* stream);

/* Post-processing inputs of the tonemap (RendererInstance.cpp:1270-1286, Passes/PostProcess.cpp): eye adaptation, then bloom.  Both read
 * the lit frame as either PBR apply writes it: width x height float4 (RGBA) per pixel, row-major, 16-byte aligned; alpha is not read.
 * Rules of both (bit for bit with oracle/oxc_oracle_post.c): binary32, no contraction, operations in written order; max / min with the
 * NaN rules of oxc_apply_pbr (a NaN operand yields the other one); clamp(x, a, b) = min(max(x, a), b); lerp(a, b, t) = a + (b - a) * t;
 * f32(u32) rounds to nearest even; every stored NaN is 0x7FFFFFFF.  Deviation from the reference: both read the binary32 lit plane, and
 * bloom keeps every level in binary32, where the reference stores B10G11R11 (whose conversion is not bit-defined).
 *
 * Eye adaptation (PostProcess.cpp:7-77, passes/histogram_generate.slang, histogram_average.slang): the 256-bin luminance histogram of the
 * frame, then the exposure record's update.  The reference runs it under HasEyeAdaptation, which it sets only for a scene with an
 * AutoExposureComponent.  exposure_dev: the persistent record, read and written in place (the reference fills it with 1.0 once, at
 * allocation).  histogram_dev: 256 u32, zeroed by the call on its stream (a memset node in a graph); after the call it holds this frame's
 * bins.  No other scratch, so the call is graph-capturable from its first call.
 * Refused with OXC_E_INVALID, before anything is enqueued: a NULL argument, a frame not 16-byte aligned, a record not 8-byte aligned or a
 * histogram not 4-byte aligned, a zero extent or one above 32768, a histogram or record that shares a byte with the frame or each other.
 * NaN, Inf and denormal settings, delta_time and pixels are accepted and follow the rules below.
 * SPECIFICATION (oracle/oxc_oracle_post.c orc_eye_adaptation):
 *   1. per call, on the host (eye_adaptation_make_params): pixel_count = f32(width * height) (a u32 product); exposure_range = max_exposure
 *      - min_exposure; time_coeff = 1 - canonical_exp(-adaptation_speed * delta_time) (the reference's glm::exp on the host); bias_scale =
 *      (100 * ev100_bias) / 12.5.
 *   2. per pixel: lum = (r * 0.2127 + g * 0.7152) + b * 0.0722 (0x3E59CE07, 0x3F371759, 0x3D93DD98).  lum < 0.001 (0x3A83126F) gives bin
 *      0; otherwise mapped = ((canonical_log2(lum) - min_exposure) / exposure_range) * 254 + 1 and the bin is clamp(sat_i32(mapped), 0,
 *      255), sat_i32 truncating and saturating, NaN -> 0.  So a NaN pixel, a -inf or negative one and one below 0.001 land in bin 0 (NaN
 *      fails the comparison, canonical_log2(NaN) = -3e38 maps below 0); +inf lands in bin 255 (canonical_log2(+inf) = 3e38) for finite
 *      settings with min < max; a finite lum with canonical_log2(lum) < min_exposure has mapped < 1 and lands in bin 0 (bin 1 at equality),
 *      one with canonical_log2(lum) >= max_exposure has mapped >= 255 and lands in bin 255.  NaN settings send every pixel to bin 0.
 *   3. average: weighted = sum over i of bins[i] * i mod 2^32 (the shader's u32 InterlockedAdd; it wraps once more than 16,843,009 pixels
 *      fall in bin 255); avg = f32(weighted) / max(pixel_count - f32(bins[0]), 1) - 1; desired = exp2((avg / 254) * exposure_range +
 *      min_exposure); adapted = last + (desired - last) * time_coeff; ev100 = canonical_log2(adapted * bias_scale); exposure = 1 /
 *      (exp2(ev100) * 1.2) (0x3F99999A).  exp2(x) = canonical_pow(2, x) (binary64 inside, within 1 ulp, the same bits on the host and
 *      the device).  The record receives (adapted, exposure). */
typedef struct OxcEyeAdaptationSettings { /* GPU::EyeAdaptationSettings; the AutoExposureComponent defaults are -11.5, 18, 1.1, 1 */
  float min_exposure;
  float max_exposure;
  float adaptation_speed;
  float ev100_bias;
} OxcEyeAdaptationSettings;
OXC_STATIC_ASSERT(sizeof(OxcEyeAdaptationSettings) == 16, "EyeAdaptationSettings");
typedef struct OxcExposure {              /* HistogramLuminance (passes/histogram.slang) */
  float adapted_luminance;
  float exposure;
} OxcExposure;
OXC_STATIC_ASSERT(sizeof(OxcExposure) == 8, "Exposure");
#define OXC_HISTOGRAM_BIN_COUNT 256u
int oxc_eye_adaptation(OxcContext* ctx, const float* frame_dev, uint32_t width, uint32_t height, const OxcEyeAdaptationSettings* settings,
                       float delta_time, OxcExposure* exposure_dev, uint32_t* histogram_dev, void* stream);

/* Bloom (PostProcess.cpp:79-203, passes/bloom_prefilter.slang, bloom_downsample.slang, bloom_upsample.slang): the prefilter of the frame
 * into level 0 of the downsampled chain, the downsample chain, then the upsample chain; the bloom image the tonemap reads is level 0 of
 * the upsampled chain.  Both chains hold levels 0..n-1 of the half extent, float4 texels, packed in level order, each row-major: level k
 * is max(1, (width / 2) >> k) x max(1, (height / 2) >> k), n = the bit length of max(width / 2, height / 2) (Texture::calculate_mip_count,
 * u32(log2f(m)) + 1; 10 levels at 1920 x 1080, 11 at 3840 x 2160); oxc_bloom_chain_texels gives the texels of one chain.  Level n-1 of
 * the upsampled chain is never written, as in the reference, except for n = 1 (item 6).  The exposure record (oxc_eye_adaptation's) is
 * read only under OXC_SCENE_HAS_EYE_ADAPTATION, where it is required; without it the exposure is 1 and exposure_dev may be NULL.  No
 * scratch, so the call is graph-capturable from its first call.  Settings: the cvars bloom_threshold 1.0, bloom_soft_threshold 0.125,
 * bloom_clamp 4.0, bloom_radius 0.75 by default; bloom_intensity belongs to the tonemap.
 * Refused with OXC_E_INVALID, before anything is launched: what oxc_eye_adaptation refuses for the frame and the record; width or height
 * below 2 (a zero half extent, an image the reference cannot create); NULL or misaligned (16-byte) targets; targets that share a byte
 * with the frame, the record or each other.
 * SPECIFICATION (oracle/oxc_oracle_post.c orc_bloom), binary32 rgb, every stored texel (rgb, 1):
 *   1. taps: the atmosphere's item-5 bilinear rule on binary32 texels: x = u * W - 0.5, x0 = floor(x), wx = x - x0 (y likewise), texels
 *      x0, x0 + 1 / y0, y0 + 1 with NaN-safe saturating indices, top = a00 + wx * (a10 - a00), bottom likewise, top + wy * (bottom - top).
 *      The prefilter and the downsample read ClampToBorder with transparent black (a texel outside the level reads 0, LinearSamplerBorder);
 *      the upsample reads ClampToEdge (LinearSamplerClamped).
 *   2. texel t of a pass: uv = (f32(t) + 0.5) / f32(size), texel_size = 1 / f32(size), size the DESTINATION level's extent in all three
 *      passes; an offset tap at uv + texel_size * (dx, dy), per component, the product first.
 *   3. prefilter (level 0 of downsampled from the frame): the 13 taps a..m; groups (((a + b) + d) + e) * 0.25 * exposure, (b c e f),
 *      (d e g h), (e f h i), (j k l m) likewise; group = min(group, clamp_value); weight = 1 / (1 + luminance(group)) with luminance's
 *      0.299 / 0.587 / 0.114 (not the histogram's weights); prefilter: brightness = max(r, max(g, b)), knee = threshold * soft_threshold,
 *      soft = clamp((brightness - threshold) + knee, 0, 2 * knee), soft = ((soft * soft) * 0.25) / (knee + 1e-5), contribution =
 *      max(soft, brightness - threshold) / max(brightness, 1e-5), (group * contribution) * weight; color_sum and weight_sum add the five
 *      groups in index order from 0; the texel is color_sum / (weight_sum + 1e-5).
 *   4. downsample, for i = 1..n-1, level i - 1 into level i: ((a + c) + g) + i) * 0.03125 + (((b + d) + f) + h) * 0.0625 + ((((e + j) + k) +
 *      l) + m) * 0.125.
 *   5. upsample, for i = n-1..1, into upsampled level i - 1: the 9-tap tent (e * 0.25 + (((b + d) + f) + h) * 0.125) + (((a + c) + g) + i)
 *      * 0.0625 at offsets -1..1 of downsampled level n-1 when i = n-1 and of upsampled level i otherwise; then lerp(tap(downsampled level
 *      i - 1, uv), tent, radius).
 *   6. n = 1 (width and height in 2..3): no upsample runs and the reference's output is its per-frame clear, vuk::Black<float>; the call
 *      writes (0, 0, 0, 1).  vuk's sources are not part of the reference tree, so this value is a commitment, not read from the code. */
typedef struct OxcBloomSettings {
  float threshold;
  float soft_threshold;
  float clamp_value;
  float radius;
  uint32_t scene_flags; /* OXC_SCENE_*: only OXC_SCENE_HAS_EYE_ADAPTATION is read */
} OxcBloomSettings;
OXC_STATIC_ASSERT(sizeof(OxcBloomSettings) == 20, "BloomSettings");
typedef struct OxcBloomTargets { /* float4 texels, 16-byte aligned, oxc_bloom_chain_texels each */
  float* downsampled;
  float* upsampled;
} OxcBloomTargets;
OXC_STATIC_ASSERT(sizeof(OxcBloomTargets) == 16, "BloomTargets");
#define OXC_BLOOM_MAX_LEVELS 15u /* half extents up to 16384 */
/* n, the level count of a width x height frame's chains (0 below 2 x 2), and the float4 texels of one chain (the sum of its level
 * extents): the size helpers of the caller's targets */
uint32_t oxc_bloom_level_count(uint32_t width, uint32_t height);
uint64_t oxc_bloom_chain_texels(uint32_t width, uint32_t height);
int oxc_bloom(OxcContext* ctx, const float* frame_dev, uint32_t width, uint32_t height, const OxcBloomSettings* settings,
              const OxcExposure* exposure_dev, const OxcBloomTargets* targets, void* stream);

/* Tonemap (PostProcess.cpp:205-247, passes/tonemap.slang fs_main, passes/lens.slang): the last step of the post chain, the HDR lit
 * frame to the displayed colour.  One thread per pixel of a width x height frame: the exposure, the bloom composite, the curve, then the
 * lens effects, into out_dev (float4 per pixel, row-major).  frame_dev: the lit frame as either PBR apply writes it, float4, 16-byte
 * aligned.  exposure_dev: oxc_eye_adaptation's record, read and required only under OXC_SCENE_HAS_EYE_ADAPTATION (8-byte aligned).
 * bloom_dev: the bloom image, upsampled level 0 of oxc_bloom's chain, (width / 2) x (height / 2) float4, read and required only under
 * OXC_SCENE_HAS_BLOOM (16-byte aligned).  Flags read: HAS_EYE_ADAPTATION, HAS_BLOOM, HAS_CHROMATIC_ABERRATION, HAS_VIGNETTE,
 * HAS_FILM_GRAIN, TRANSPARENT_BACKGROUND; the others are ignored.  No scratch, so the call is graph-capturable from its first call.
 * Settings: the PostProcessSettings push constants, the pp.exposure cvar (1.0), pp.bloom_intensity (0.1), the component defaults
 * (vignette 0.5, chromatic aberration 0.5, film grain amount 0.6 and scale 0.7), TonemappingComponent's AgX, seed = frame count % 16.
 * Refused with OXC_E_INVALID, before anything is launched: a NULL required argument; a zero extent or one above 32768; frame_dev or
 * out_dev not 16-byte aligned, a required bloom_dev not 16-byte or exposure_dev not 8-byte aligned; tonemap_type above OXC_TONEMAP_GT7;
 * OXC_SCENE_HAS_BLOOM with width or height below 2 (no bloom image exists); out_dev sharing a byte with the frame or a required input
 * (in place included: the chromatic aberration taps read other pixels).  NaN, Inf and denormal settings, records and pixels are
 * accepted and follow the rules below.
 * SPECIFICATION (oracle/oxc_oracle_tonemap.c orc_tonemap), the rules of oxc_eye_adaptation and oxc_bloom (binary32, no contraction,
 * written order, max / min NaN rules, clamp(x, a, b) = min(max(x, a), b), saturate = clamp(x, 0, 1), lerp(a, b, t) = a + (b - a) * t,
 * mul(M, v) = row . v with dot(a, b) = (a.x*b.x + a.y*b.y) + a.z*b.z, mul(A, B) likewise, a scalar times a vector per component,
 * constants the binary32 roundings of the literals); every stored NaN is 0x7FFFFFFF.  Items 5-9 settle what the reference leaves open
 * and are commitments:
 *   1. taps: SampleLevel of a float4 plane through the pass's {linear, linear} sampler; its address mode is vuk's default, which is not
 *      in the reference tree: committed to Repeat (Vulkan's zero value).  The bilinear rule of oxc_bloom item 1 on all four channels,
 *      with texel indices wrapped into 0..n-1 (wrap_index): so column 0 blends with the last column at the left edge.  NaN-safe: the
 *      floor goes through the saturating sat_i32 and a NaN coordinate gives NaN weights.
 *   2. pixel (x, y): tex_coord uv = ((f32(x) + 0.5) / f32(width), (f32(y) + 0.5) / f32(height)) (bloom item 2's rule); source = the
 *      frame's tap at uv.  u * width - 0.5 need not be the integer x, and the rule computes a00 + wx * (a10 - a00) even at wx = 0, so a
 *      non-finite neighbour can reach a pixel.  color = source.rgb * exposure, the record's exposure under HasEyeAdaptation, else
 *      settings->exposure; under HasBloom color += tap(bloom, uv).rgb * bloom_intensity (a bilinear upscale, wrapping at the edges).
 *   3. curve, by tonemap_type: NONE none; ACES ACES_Fitted (ACESInputMat, RRTAndODTFit a = v * (v + 0.0245786) - 0.000090537, b = v *
 *      (0.983729 * v + 0.4329510) + 0.238081, a / b, ACESOutputMat, saturate): outputs in [0, 1]; AGX AgX_DS (max(c, 0), the matrix,
 *      clamp(DualSection(x, 0.1, 1), 0, 1) with DualSection = x < S ? x : peak - (peak - S) * exp((-C * (x - S)) / peak), desaturation
 *      dot with (0.2126729, 0.7151522, 0.0721750), clamp(lerp(d, c, 1.3), 0, 1), the inverse matrix): not bounded, the inverse comes
 *      after the last clamp; GT7 initializeAsSDR + applyToneMapping with the ICtCp UCS in Rec.2020 through com::rec709_to_rec2020 /
 *      rec2020_to_rec709 (via XYZ, two mat . v each way): its Rec.2020 output lies in [0, 1] (min(blended, 2.5) * 0.4, NaN -> 1).
 *   4. chromatic aberration (HasChromaticAberration) REPLACES the colour: its three taps read the raw frame, without exposure, bloom or
 *      curve (reference behaviour).  rg = FfxLensGetRGMag(amount) per call; c = screen_size / 2 in integers; red / green tap at
 *      ((f32(x - c.x) * mag + f32(c.x)) + 0.5) * (1 / f32(2 * c.x)) (y likewise), the .r / .g of the tap; the blue tap at f32(x) *
 *      (1 / f32(2 * c.x)), the pixel's corner, without the + 0.5, its .b.  For an odd width 1 / f32(2 c) is not 1 / width.  At width or
 *      height 1, c = 0 and the coordinates follow IEEE arithmetic (inf, NaN) and item 1's NaN rule; the call is not refused.
 *   5. vignette (HasVignette), before the grain as fs_main calls them: m = canonical_cos((f32(|x - c.x|) / f32(c.x) * amount) * fl(PI
 *      * 0.25)) per axis, squared twice, color *= clamp(m.x * m.y, 0, 1); exactly 1 at the centre pixel.
 *   6. film grain (HasFilmGrain): d = sat_i32(scale / 8) (truncating, saturating, NaN -> 0); the quotient coord / d in i32, truncating,
 *      converted to u32 (a negative one wraps); d = 0, which every scale in (-8, 8) gives (the component's 0.7 included) and which the
 *      shader leaves undefined, gives the quotient -1, all ones, in both components (an explicit branch).  pcg3d16((q.x, q.y, seed)) in
 *      u32 arithmetic mod 2^32; r = f32(v) * 2^-16 - 0.5; simplex(f32(coord) / scale + r) with round() = rint (ties to even, HLSL's
 *      rule; GLSL.std.450 leaves halves open); grain = 1 - 2 * exp2(-length(p) * 3); color += (grain * min(color, 1 - color)) * amount.
 *   7. alpha: the source tap's alpha under TransparentBackground, else 1.
 *   8. transcendentals: exp canonical_exp, log2 canonical_log2, pow canonical_pow, exp2(x) canonical_pow(2, x), cos canonical_cos
 *      (oxc_exact.cuh; the oracle's orc_*_canonical); sqrt and / are IEEE.
 *   9. constants that do not depend on the call, formed once in binary32 in shader order with the same functions (the values the
 *      library keeps as hex and the tests recompute): AgX's sRGB_to_adjusted = mul(sRGB_to_XYZ, XYZ_to_adjusted) as the code writes it
 *      (color_PrimariesToMatrix, color_ComputeCompressionMatrix with compression 0.15, tonemap.slang's inverse) and its inverse; the
 *      DualSection constants; GT7's kA, kB, kC, linearSection * peak, the target 2.5, its UCS intensity, the SDR factor 0.4, 1 - 0.6, 1 / m1,
 *      1 / m2; simplex's F2 and G2.  The unused shader paths (agx_tonemapping, the Jzazbz UCS, initializeAsHDR) are not part of it.
 *   10. output: binary32 RGBA, the value before the reference's store into the caller's attachment format (deviation: that conversion
 *      is not bit-defined). */
#define OXC_TONEMAP_NONE 0u /* TonemapType */
#define OXC_TONEMAP_ACES 1u
#define OXC_TONEMAP_AGX 2u
#define OXC_TONEMAP_GT7 3u
typedef struct OxcTonemapSettings {
  uint32_t scene_flags;               /* OXC_SCENE_*: the six flags above are read */
  uint32_t tonemap_type;              /* OXC_TONEMAP_* */
  float exposure;                     /* pp.exposure, read without HasEyeAdaptation */
  float bloom_intensity;              /* pp.bloom_intensity */
  float chromatic_aberration_amount;
  float vignette_amount;
  float film_grain_scale;
  float film_grain_amount;
  uint32_t film_grain_seed;
} OxcTonemapSettings;
OXC_STATIC_ASSERT(sizeof(OxcTonemapSettings) == 36, "TonemapSettings");
int oxc_tonemap(OxcContext* ctx, const float* frame_dev, uint32_t width, uint32_t height, const OxcTonemapSettings* settings,
                const OxcExposure* exposure_dev, const float* bloom_dev, float* out_dev, void* stream);

/* FXAA (RendererInstance.cpp:1225-1255, passes/fxaa/fxaa.slang fs_main): the anti-aliasing pass between PBR apply and the post chain.
 * The reference runs it under HasFXAA (OXC_SCENE_HAS_FXAA, the pp.fxaa cvar, on by default) on the HDR frame, before eye adaptation,
 * bloom and the tonemap, and its output becomes the frame those three read (std::tie(final_attachment, ...) = fxaa_pass(...)).  The
 * caller gates the call on HasFXAA, as the reference's `if` does.  One thread per pixel of a width x height frame: the 3 x 3 luma
 * neighbourhood, the early exit, the walk along the edge, the sub-pixel term and one final tap, into out_dev (float4 per pixel,
 * row-major).  frame_dev: the lit frame as either PBR apply writes it, float4, 16-byte aligned.  No settings: the reference has none.
 * No scratch, so the call is graph-capturable from its first call.
 * Refused with OXC_E_INVALID, before anything is launched: a NULL argument; a zero extent or one above 32768; frame_dev or out_dev not
 * 16-byte aligned; out_dev sharing a byte with frame_dev (in place included: the taps read other pixels).  NaN, Inf, denormal and
 * negative pixels are accepted and follow the rules below.
 * SPECIFICATION (oracle/oxc_oracle_fxaa.c orc_fxaa), binary32, no contraction, each expression in the shader's written order, left to
 * right; max / min with the NaN rules of oxc_apply_pbr (a NaN operand yields the other one, vmax / vmin); clamp(x, 0, 1) = min(max(x,
 * 0), 1); sqrt and / are IEEE; abs is fabs; every stored NaN is 0x7FFFFFFF:
 *   1. pixel and step: pixel (x, y) has tex_coord uv = ((f32(x) + 0.5) / f32(width), (f32(y) + 0.5) / f32(height)) (oxc_tonemap item 2's
 *      rule); inv = (1 / f32(width), 1 / f32(height)), the push constant inverse_screen_size, formed once per call.
 *   2. taps: Sample(uv) is oxc_bloom item 1's bilinear rule on all four channels with ClampToEdge (LinearSamplerClamped, the sampler of
 *      bloom's upsample): x = u * W - 0.5, x0 = floor(x), wx = x - x0 (y likewise), texels x0, x0 + 1 / y0, y0 + 1 clamped into the
 *      frame (NaN-safe: the floor goes through the saturating sat_i32, a NaN coordinate gives NaN weights).  The frame has one level, so
 *      the implicit-LOD Sample reads level 0.  Sample(uv, int2(dx, dy)) adds the constant offset to the unnormalised coordinate before
 *      the half-texel shift: x = (u * W + dx) - 0.5 (y likewise).  That is Vulkan's texel-offset order; the Vulkan specification is not
 *      in the reference tree, so this order is a commitment.  u * W - 0.5 need not be the integer x, and the rule computes a00 + wx *
 *      (a10 - a00) even at wx = 0: a centre or cross tap is a real bilinear tap, not a texel load, and a non-finite neighbour can reach
 *      a pixel.
 *   3. luma(c) = sqrt((c.r * 0.299 + c.g * 0.587) + c.b * 0.114) with bloom's binary32 weights (0x3E991687, 0x3F1645A2, 0x3DE978D5);
 *      a negative sum gives NaN.
 *   4. early exit: luma_center = luma(Sample(uv)); luma_down, _up, _left, _right of the offsets (0, -1), (0, 1), (-1, 0), (1, 0);
 *      luma_min = min(center, min(min(down, up), min(left, right))), luma_max likewise with max, range = luma_max - luma_min.  If range <
 *      max(0.0312, luma_max * 0.125) the output is the centre tap.  A NaN range fails the comparison and goes on to the walk.
 *   5. the rest of fs_main, line by line: the corners (-1, -1), (1, 1), (-1, 1), (1, -1); down_up = down + up, left_right = left + right,
 *      left_corners = down_left + up_left, down_corners = down_left + down_right, right_corners = down_right + up_right, up_corners =
 *      up_right + up_left; edge_horizontal = (abs(-2 * left + left_corners) + abs(-2 * center + down_up) * 2) + abs(-2 * right +
 *      right_corners), edge_vertical = (abs(-2 * up + up_corners) + abs(-2 * center + left_right) * 2) + abs(-2 * down + down_corners);
 *      is_horizontal = edge_horizontal >= edge_vertical; step = is_horizontal ? inv.y : inv.x; luma1, luma2 = is_horizontal ? (down,
 *      up) : (left, right); gradient1 = luma1 - center, gradient2 = luma2 - center; is1_steepest = abs(gradient1) >= abs(gradient2);
 *      gradient_scaled = 0.25 * max(abs(gradient1), abs(gradient2)); if is1_steepest: step = -step, local_average = 0.5 * (luma1 +
 *      center), else 0.5 * (luma2 + center); current = uv with current.y (horizontal) or .x += step * 0.5; offset = is_horizontal ?
 *      (inv.x, 0) : (0, inv.y); uv1 = current - offset * QUALITY(0), uv2 = current + offset * QUALITY(0); end1 = luma(Sample(uv1)) -
 *      local_average, end2 likewise; reached1 = abs(end1) >= gradient_scaled, reached2 likewise; uv1 -= offset * QUALITY(1) unless
 *      reached1, uv2 += ... unless reached2; unless both are reached, for i = 2..11: end1 = luma(Sample(uv1)) - local_average unless
 *      reached1, end2 likewise, both reached flags recomputed, uv1 -= offset * QUALITY(i) unless reached1, uv2 += ... unless reached2,
 *      and then break when both are reached (the break comes after that step's advance).  end1 and end2 keep their last values for the
 *      variation test.  QUALITY(i) = 1 for i <= 4, 1.5 at 5, 2 for 6..9, 4 at 10, 8 at 11.  distance1 = is_horizontal ? uv.x - uv1.x :
 *      uv.y - uv1.y, distance2 = is_horizontal ? uv2.x - uv.x : uv2.y - uv.y; is_direction1 = distance1 < distance2; distance_final =
 *      min(distance1, distance2); edge_thickness = distance1 + distance2; center_smaller = center < local_average; correct_variation =
 *      is_direction1 ? ((end1 < 0) != center_smaller) : ((end2 < 0) != center_smaller); pixel_offset = (-distance_final /
 *      edge_thickness) + 0.5; final_offset = correct_variation ? pixel_offset : 0; luma_average = (1 / 12) * (((2 * (down_up +
 *      left_right)) + left_corners) + right_corners); sub1 = clamp(abs(luma_average - center) / range, 0, 1); sub2 = ((-2 * sub1 + 3) *
 *      sub1) * sub1; sub_final = (sub2 * sub2) * 0.75; final_offset = max(final_offset, sub_final); final_uv = uv with final_uv.y
 *      (horizontal) or .x += final_offset * step.  A uv component whose offset component is 0 stays bit-identical (uv - 0 * q = uv), so
 *      an implementation may advance only the moving axis.  At most 32 bilinear taps per pixel (1 centre, 4 cross, 4 corners, 2 first
 *      ends, 2 x 10 in the walk, 1 final); the farthest lies 18.5 texels along the edge.
 *   6. constants, the binary32 roundings of the literals: 0.0312 = 0x3CFF9724, 0.125, 0.75, 1.0 / 12.0 = 0x3DAAAAAB (the binary32
 *      quotient and the rounding of the binary64 quotient agree, so the literal's type does not matter).
 *   7. output: Sample(final_uv), or the centre tap on the early exit, all four channels: alpha is filtered like the colour.  A binary32
 *      float4 plane; deviation: it is not converted to the reference's hdr_format attachment (that conversion is not bit-defined). */
int oxc_fxaa(OxcContext* ctx, const float* frame_dev, uint32_t width, uint32_t height, float* out_dev, void* stream);

int oxc_get_outputs(OxcContext* ctx, OxcOutputs* out);
/* Instrumentation hook: 128 u64 counters that builds with -DOXC_RASTER_STATS fill (tools/raster_stats.py); zero otherwise. */
void* oxc_debug_stats_ptr(OxcContext* ctx);

/* Plumbing for hosts without their own CUDA bindings (the ctypes tests / bench): async copy on `stream`
 * (kind 0 = host->device, 1 = device->host, 2 = device->device), stream sync, raw device allocations. */
int oxc_copy(OxcContext* ctx, void* dst, const void* src, uint64_t bytes, int kind, void* stream);
int oxc_sync(OxcContext* ctx, void* stream);
int oxc_device_alloc(OxcContext* ctx, uint64_t bytes, void** out);
int oxc_device_free(OxcContext* ctx, void* ptr);
/* Test hook: evaluates both device implementations of com::dequantize_half (common/math.slang:193-201) on all
 * 65536 inputs into two float[65536] device arrays. */
int oxc_debug_dequantize_half(OxcContext* ctx, float* canonical_dev, float* hw_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * oxr_* — host-side mirror of the reference's frame sequencing (C++ class ox::RendererInstance in
 * oxylus_b200/csrc/host/renderer_instance.hpp) exported for non-C++ callers.  One call runs
 *   run_geometry_pass(false) -> generate_hiz -> run_geometry_pass(true)
 * (RendererInstance.cpp:842-884) with HOST inputs and HOST outputs.
 * ---------------------------------------------------------------------------------------------- */
typedef struct OxrRenderer OxrRenderer;

typedef struct OxrFrameResult {
  OxcMeshletInstanceVisibility visibility; /* total / early / late */
  uint32_t draw_index_count_early;         /* draw_cmd.index_count of the early pass */
  uint32_t draw_index_count_late;
  uint64_t raster_triangles;               /* triangles rasterised this frame */
} OxrFrameResult;

int oxr_create(int device, const OxcCreateInfo* info, uint32_t width, uint32_t height, OxrRenderer** out);
void oxr_destroy(OxrRenderer* r);
OxcContext* oxr_context(OxrRenderer* r);
/* RendererInstance::update */
int oxr_update(OxrRenderer* r, const OxcSceneDesc* scene);
/* dirty-range transform upload (RendererInstance.cpp:16-109,1590-1599) from HOST memory, async on the renderer's
 * stream (ordered before the next oxr_render) */
int oxr_update_transforms(OxrRenderer* r, const OxcTransformWorld* transforms, uint32_t first, uint32_t count);
/* Depth laid down by passes outside this path (terrain, RendererInstance.cpp:862-873): a width x height D32F HOST
 * image copied to the device once and merged into every following frame; NULL removes it. */
int oxr_set_external_depth(OxrRenderer* r, const float* depth_host);
/* The terrain of RendererInstance::render (Passes/Terrain.cpp:159-277, RendererInstance.cpp:864-880): copies the res_x x res_y R16
 * heightmap and the patch min / max (float2 per patch, row-major) from HOST memory with the settings of oxc_draw_terrain, and allocates
 * the visible-patch list, the draw command and the persistent patch visibility mask (zeroed).  With a terrain set, each geometry pass
 * of oxr_render / oxr_submit runs oxc_cull_terrain (TestFrustum | TestOcclusion, | LatePass in the late pass) and oxc_draw_terrain
 * right after its meshlet raster, before generate_hiz in the early pass.  Those two take the camera by value, so oxr_submit enqueues a
 * frame with a terrain without its CUDA graphs.  heightmap_host == NULL removes the terrain (the frame is the terrain-less one again).
 * Either call drops the captured frame graphs.  OXC_E_INVALID for a missing min / max or settings, a zero or > 65536 side, an empty or
 * > 2^32 - 1 patch grid, or a target_edge_pixels / max_tessellation that is not finite or below 1; the terrain is removed then. */
int oxr_set_terrain(OxrRenderer* r, const uint16_t* heightmap_host, uint32_t res_x, uint32_t res_y, const float* patch_minmax_host,
                    const OxcTerrainDrawSettings* settings);
/* MainGeometryContext::draw_overdraw (RendererInstance.cpp:771-776): the encode pass's fragment counter (oxc_raster_overdraw, both
 * passes) of the frame that oxr_render / oxr_wait completed last, for the camera it was rendered with; width x height u32 to the
 * host.  Synchronous; the frame's own outputs are not touched. */
int oxr_overdraw(OxrRenderer* r, const OxcCullCamera* camera, uint32_t* overdraw_host);
/* oxc_set_materials on the renderer's context (alpha-tested discard of the vis-buffer encode, visbuffer_encode.slang:54-66);
 * NULL switches it off.  Re-captures the frame graphs: the raster's launch sequence changes with it. */
int oxr_set_materials(OxrRenderer* r, const OxcMaterialTable* table);
/* RendererInstance::render geometry section.  occluder_depth_host (may be NULL) is a width x height
 * D32F image uploaded THIS frame and merged into the frame depth before the early pass (replaces the image of
 * oxr_set_external_depth).  Outputs may be NULL.  Synchronous. */
int oxr_render(OxrRenderer* r, const OxcCullCamera* camera, const float* occluder_depth_host,
               uint32_t* vis32_host, float* depth_host, uint32_t* visible_indices_host,
               uint32_t visible_indices_capacity, OxrFrameResult* result);

/* Pipelined frames: oxr_submit enqueues the frame and the device->host copies of its results (separate copy
 * stream, double-buffered staging) and returns a ticket (0/1) without waiting; oxr_wait blocks until that frame's
 * outputs are in the caller's (pinned) host buffers and fills `result`.  At most two frames in flight; a slot's
 * ticket must be waited before the slot is reused.  Survivor ids: min(capacity, max_meshlet_instances) entries are
 * copied; the valid prefix is result->visibility.early + late. */
int oxr_submit(OxrRenderer* r, const OxcCullCamera* camera, uint32_t* vis32_host, float* depth_host,
               uint32_t* visible_indices_host, uint32_t visible_indices_capacity, int* ticket);
int oxr_wait(OxrRenderer* r, int ticket, OxrFrameResult* result);

/* RendererInstance::draw_virtual_shadowmap page loop (Shadowmaps.cpp:100-430, steps up to the shadow raster): the renderer owns the
 * virtual page table, the HPB, occupancy, requests, the allocator and its lists, the clipmap dirty flags and the physical atlas
 * (allocated by the first call, re-allocated when the shape changes: the table then starts cleared and the atlas zeroed), and runs
 * the sequence of oxc_vsm_begin_frame on its stream from the depth of the frame oxr_render / oxr_wait completed last.  Previous
 * transforms (invalidation) are the values each transform had before the oxr_update_transforms that last changed it.  Synchronous. */
typedef struct OxrVsmPageContext {
  OxcVsmContext vsm;                       /* page_size, page_table_size, physical_page_table_size, clipmap_count, ... */
  OxcVirtualClipmap clipmaps[10];          /* clipmap_count used */
  float inv_projection_view[16];           /* Camera::inv_projection_view of the frame */
  float resolution[2];
  uint32_t sun_moved;
  uint32_t dirty_mesh_instance_count;
  const uint32_t* dirty_mesh_instances;    /* host, dirty_mesh_instance_count indices (Scene.cpp dirty_mesh_instance_indices) */
  uint32_t hpb_levels;                     /* 1..16 */
} OxrVsmPageContext;
typedef struct OxrVsmPages {               /* device pointers, valid until the next oxr_vsm_update_pages with another shape */
  uint32_t* page_tables;                   /* [clipmap][size][size] */
  uint8_t* hpb;                            /* oxc_build_hpb layout */
  uint32_t* page_occupancy;
  int32_t* requests;                       /* request_capacity int3 */
  OxcVsmAllocator* allocator;
  uint32_t* free_page_list;
  uint32_t* dirty_physical_page_coords;
  uint32_t* clipmap_dirty_flags;
  float* physical_atlas;
  uint32_t page_table_size, clipmap_count, physical_page_count, physical_atlas_size, hpb_levels, request_capacity;
} OxrVsmPages;
int oxr_vsm_update_pages(OxrRenderer* r, const OxrVsmPageContext* context);
int oxr_vsm_pages(OxrRenderer* r, OxrVsmPages* out);
/* RendererInstance::draw_virtual_shadowmap's last step (Shadowmaps.cpp:433-754): cull_geometry with use_hpb for the coarse camera
 * (clipmap 9's projection_view as projection_view, near_clip = z_near, position = -light_dir): oxc_cull_meshes, then
 * oxc_cull_meshlets_hpb_dirty_dev on the device dirty flags, then oxc_vsm_draw_pages into the renderer's atlas, with the clipmaps,
 * flags, HPB and page table of the last oxr_vsm_update_pages, on the renderer's stream.  Synchronous.  It runs on a second context
 * the renderer keeps with the same scene, transforms and materials, so the next oxr_render / oxr_submit computes exactly what it
 * would have without it, and oxr_overdraw still sees the last frame's survivors.  OXC_E_STATE before an oxr_vsm_update_pages.
 * Footprint: oxr_create makes that context with the renderer's OxcCreateInfo (max_views raised to 10), and every oxr_update /
 * oxr_update_transforms / oxr_set_materials is applied to it as well — a second device copy of the scene blob and tables and of
 * the per-meshlet-instance buffers, plus 16 MiB of draw scratch at the first call.  The scene reaches the renderer only through
 * oxr_update, so the context cannot be made later from it.  If the context cannot be created or kept in step (out of device memory),
 * the camera path is unaffected and this call returns OXC_E_CAPACITY. */
int oxr_vsm_draw_shadows(OxrRenderer* r, const OxcCullCamera* coarse);
/* RendererInstance::resolve_shadowmap (Shadowmaps.cpp:756-822): on the frame oxr_render / oxr_wait completed last, oxc_decode_visbuffer
 * with `camera` (the camera that frame was rendered with) into a uv_normal plane the renderer allocates at the first call, then
 * oxc_vsm_resolve_shadows with the shape, clipmaps, inv_projection_view and resolution of the last oxr_vsm_update_pages, the
 * renderer's atlas and the frame's depth; width x height floats to shadow_host.  Synchronous.  The camera frame's outputs, the page
 * table and the atlas are left as they were.  OXC_E_STATE before an oxr_vsm_update_pages;
 * OXC_E_CAPACITY, with the camera path left usable, when the 20 B / pixel of its own planes cannot be allocated. */
int oxr_vsm_resolve_shadows(OxrRenderer* r, const OxcCullCamera* camera, float* shadow_host);
/* RendererInstance's vis decode pass (visbuffer_decode.slang:88-183): oxc_decode_gbuffer on the frame oxr_render / oxr_wait completed
 * last, with `camera` (the camera that frame was rendered with) and the table of the last oxr_set_materials, into planes the renderer
 * allocates at the first call (64 B / pixel); each non-NULL host pointer receives width x height float4.  Synchronous.  Pixels the
 * decode discards hold 0.  The frame's outputs are left as they were.  OXC_E_CAPACITY, with the camera path left usable, when the
 * planes cannot be allocated. */
int oxr_decode_gbuffer(OxrRenderer* r, const OxcCullCamera* camera, float* albedo_host, float* normal_host, float* emissive_host,
                       float* metallic_roughness_occlusion_host);
/* RendererInstance::generate_ambient_occlusion (PBR.cpp:143-311): on the frame oxr_render / oxr_wait completed last, oxc_decode_visbuffer
 * with `camera` into the uv_normal plane oxr_vsm_resolve_shadows uses (one plane for both calls), then oxc_generate_ambient_occlusion
 * on the frame's depth with gtao_camera and settings; width x height floats to ao_host.  Its own planes (depth mips, edges, noisy and
 * final occlusion, about 16 B / pixel) are allocated at the first call.  Synchronous.  The frame's outputs are left as they were.
 * OXC_E_CAPACITY, with the camera path left usable, when the planes cannot be allocated. */
int oxr_generate_ambient_occlusion(OxrRenderer* r, const OxcCullCamera* camera, const OxcGtaoCamera* gtao_camera,
                                   const OxcGtaoSettings* settings, float* ao_host);
/* RendererInstance::apply_pbr (PBR.cpp:435-531, no atmosphere) with the passes before it, on the frame oxr_render / oxr_wait completed
 * last, on the renderer's stream, synchronous:
 *   1. the G-buffer decode with `camera` and the table of the last oxr_set_materials (as oxr_decode_gbuffer);
 *   2. cast_shadows != 0: the shadow resolve with the state of the last oxr_vsm_update_pages / oxr_vsm_draw_shadows (OXC_E_STATE
 *      without one); otherwise the shadow plane reads 1, as the reference's without cast_shadows;
 *   3. OXC_SCENE_HAS_GTAO: oxc_generate_ambient_occlusion with gtao_camera and gtao_settings (both required then);
 *   4. oxc_apply_pbr with pbr_camera, settings and settings->light_count records of lights_host, uploaded into a renderer-owned
 *      OXC_MAX_LIGHTS-record buffer.
 * The resolve and the GTAO read the G-buffer's normal plane (its .zw equals oxc_decode_visbuffer's uv_normal.zw).  width x height
 * float4 to rgba_host.  OXC_SCENE_HAS_CONTACT_SHADOWS is refused (OXC_E_INVALID): oxr_apply_pbr_with_contact_shadows below runs the
 * contact-shadow pass and takes the flag.  The planes (G-buffer, resolve, GTAO, about 100 B / pixel, and 16 B / pixel of output) are
 * allocated at the first call that needs them; OXC_E_CAPACITY, with the camera path left usable, when they cannot be.  The frame's
 * outputs are left as they were. */
int oxr_apply_pbr(OxrRenderer* r, const OxcCullCamera* camera, const OxcPbrCamera* pbr_camera, const OxcPbrSettings* settings,
                  const OxcLight* lights_host, int cast_shadows, const OxcGtaoCamera* gtao_camera, const OxcGtaoSettings* gtao_settings,
                  float* rgba_host);
/* The contact_shadows pass (RendererInstance.cpp:990-1020): oxc_contact_shadows on the depth of the frame oxr_render / oxr_wait
 * completed last, into a 4 B / pixel plane the renderer allocates at the first call; width x height floats to contact_host.
 * Synchronous.  The frame's outputs are left as they were.  OXC_E_CAPACITY, with the camera path left usable, when the plane cannot be
 * allocated; OXC_E_INVALID for settings oxc_contact_shadows refuses. */
int oxr_contact_shadows(OxrRenderer* r, const OxcContactShadowCamera* contact_camera, const OxcContactShadowSettings* settings,
                        float* contact_host);
/* oxr_apply_pbr with OXC_SCENE_HAS_CONTACT_SHADOWS accepted: under that flag the contact-shadow pass runs in the reference's place,
 * after the shadow resolve and before the GTAO, with contact_camera and contact_settings (both required then), and oxc_apply_pbr reads
 * its plane.  Without the flag it computes exactly what oxr_apply_pbr computes and the two contact arguments are not read. */
int oxr_apply_pbr_with_contact_shadows(OxrRenderer* r, const OxcCullCamera* camera, const OxcPbrCamera* pbr_camera, const OxcPbrSettings* settings,
                                       const OxcLight* lights_host, int cast_shadows, const OxcGtaoCamera* gtao_camera,
                                       const OxcGtaoSettings* gtao_settings, const OxcContactShadowCamera* contact_camera,
                                       const OxcContactShadowSettings* contact_settings, float* rgba_host);
/* RendererInstance::apply_pbr with an atmosphere (PBR.cpp:312-432) and the passes before it, on the renderer's stream, synchronous:
 *   1. the per-frame LUTs and the sky IBL cube update exactly as oxr_atmosphere_sky_ibl makes them (the same planes, the bake at the
 *      first use, the same cube and call counter, which this call advances) with pbr_camera, settings->sun_direction and ->sun_intensity;
 *   2. the G-buffer decode, shadow resolve, contact shadows and GTAO as oxr_apply_pbr_with_contact_shadows runs them;
 *   3. oxc_apply_pbr_atmosphere over those planes and tables, the record's sizes replaced by the renderer's extents.
 * settings must carry OXC_SCENE_HAS_ATMOSPHERE and OXC_SCENE_HAS_DIRECTIONAL_LIGHT (OXC_E_INVALID otherwise, before anything is
 * enqueued): the reference updates its sky tables only under HasDirectionalLight (RendererInstance.cpp:1022), so HasAtmosphere
 * without it samples tables no pass wrote in that frame.  width x height float4 to rgba_host.  OXC_E_CAPACITY as oxr_apply_pbr. */
int oxr_apply_pbr_atmosphere(OxrRenderer* r, const OxcCullCamera* camera, const OxcPbrCamera* pbr_camera, const OxcPbrSettings* settings,
                             const OxcAtmosphere* atmosphere, const OxcLight* lights_host, int cast_shadows, const OxcGtaoCamera* gtao_camera,
                             const OxcGtaoSettings* gtao_settings, const OxcContactShadowCamera* contact_camera,
                             const OxcContactShadowSettings* contact_settings, float* rgba_host);
/* The atmosphere's lookup tables as the reference makes them, on the renderer's stream, synchronous.  At its first call the renderer
 * allocates its three planes at the reference's extents (transmittance 256 x 64, sky view 312 x 192, aerial perspective 32 x 32 x 32; about
 * 0.7 MiB) and bakes the transmittance LUT once with the DEFAULT record (GPU::Atmosphere{} with those sizes), as the reference's init does:
 * a scene's atmosphere never reaches the transmittance LUT.  Every call then runs oxc_atmosphere_sky_luts with a copy of the caller's
 * record whose four size fields are replaced by the renderer's extents (RendererInstance.cpp:1456-1459), the camera and the sun.  Each
 * non-NULL host pointer receives its plane (binary16 RGBA, 8 B per texel).  The frame's outputs are left as they were.  OXC_E_CAPACITY,
 * with the camera path left usable, when the planes cannot be allocated. */
int oxr_atmosphere_luts(OxrRenderer* r, const OxcAtmosphere* atmosphere, const OxcPbrCamera* camera, const float sun_direction[3],
                        float sun_intensity, uint16_t* transmittance_host, uint16_t* sky_view_host, uint16_t* aerial_perspective_host);
/* The sky IBL cube as the reference makes it each frame, on the renderer's stream, synchronous: the per-frame LUTs exactly as
 * oxr_atmosphere_luts makes them (the same planes, the bake at the first call), then oxc_atmosphere_sky_ibl over them into a cube the
 * renderer owns (allocated and zeroed at the first call, as the reference clears its cube to black) with sun_ambient_strength 0.15 and
 * frame_index = the number of earlier oxr_atmosphere_sky_ibl calls on this renderer (0 at the first).  That count equals the reference's
 * frame counter when the call runs once per frame from the engine's first frame.  cube_host (may be NULL) receives the cube, 6 x 32 x 32
 * binary16 RGBA (48 KiB).  The frame's outputs are left as they were.  OXC_E_CAPACITY, with the camera path left usable, when the
 * planes cannot be allocated; a failed call does not advance the count. */
int oxr_atmosphere_sky_ibl(OxrRenderer* r, const OxcAtmosphere* atmosphere, const OxcPbrCamera* camera, const float sun_direction[3],
                           float sun_intensity, uint16_t* cube_host);
/* The post chain's source: oxr_eye_adaptation, oxr_bloom and oxr_tonemap read the lit plane of the renderer's last oxr_apply_pbr* call,
 * or, after a successful oxr_fxaa, the FXAA plane, as the reference's final_attachment becomes FXAA's output.  The next oxr_apply_pbr*
 * makes the lit plane the source again.
 * Eye adaptation (PostProcess.cpp:7-77) on the post chain's source, on the renderer's stream, synchronous: oxc_eye_adaptation into the renderer's exposure record and histogram.  The first call allocates both and fills the record
 * with (1, 1), as the reference's vuk::fill does; the record persists across calls.  exposure_host (may be NULL) receives the record
 * after the call.  OXC_E_INVALID before any oxr_apply_pbr* call; OXC_E_CAPACITY, with the camera path left usable, when the record cannot
 * be allocated.  The frame's outputs and the source plane are left as they were. */
int oxr_eye_adaptation(OxrRenderer* r, const OxcEyeAdaptationSettings* settings, float delta_time, OxcExposure* exposure_host);
/* Bloom (PostProcess.cpp:79-203) of the post chain's source, on the renderer's stream, synchronous: oxc_bloom into the renderer's two chains
 * (allocated at the first call), reading the renderer's exposure record under OXC_SCENE_HAS_EYE_ADAPTATION (OXC_E_STATE before an
 * oxr_eye_adaptation then).  bloom_host (may be NULL) receives upsampled level 0, (width / 2) x (height / 2) float4.  OXC_E_INVALID before
 * any oxr_apply_pbr* call or for a frame below 2 x 2; OXC_E_CAPACITY, with the camera path left usable, when the chains cannot be
 * allocated.  The frame's outputs and the source plane are left as they were. */
int oxr_bloom(OxrRenderer* r, const OxcBloomSettings* settings, float* bloom_host);
/* Tonemap (PostProcess.cpp:205-247) of the post chain's source, on the renderer's stream, synchronous: oxc_tonemap into a plane the renderer
 * owns (allocated at the first call), reading the renderer's exposure record under OXC_SCENE_HAS_EYE_ADAPTATION and its bloom image
 * (upsampled level 0) under OXC_SCENE_HAS_BLOOM.  rgba_host (may be NULL) receives width x height float4.  OXC_E_INVALID before any
 * oxr_apply_pbr* call; OXC_E_STATE under HasEyeAdaptation before an oxr_eye_adaptation and under HasBloom before an oxr_bloom;
 * OXC_E_CAPACITY, with the camera path left usable, when the plane cannot be allocated.  The source plane, the record and the bloom
 * chains are left as they were. */
int oxr_tonemap(OxrRenderer* r, const OxcTonemapSettings* settings, float* rgba_host);
/* FXAA (RendererInstance.cpp:1225-1255) of the lit plane of the renderer's last oxr_apply_pbr* call, on the renderer's stream,
 * synchronous: oxc_fxaa into a plane the renderer owns (allocated at the first call), which then becomes the post chain's source until
 * the next oxr_apply_pbr*.  It always reads the lit plane, so a second call gives the same plane.  The caller gates it on HasFXAA and
 * runs it once per frame, between PBR apply and eye adaptation, as the reference does.  rgba_host (may be NULL) receives width x height
 * float4.  OXC_E_INVALID before any oxr_apply_pbr* call; OXC_E_CAPACITY, with the camera path left usable, when the plane cannot be
 * allocated.  The lit plane is left as it was. */
int oxr_fxaa(OxrRenderer* r, float* rgba_host);

/* ------------------------------------------------------------------------------------------------
 * oxb_* — mesh builder (SURVEY §8f.2): host-side producer of the blob layout above, mirroring build_gltf_mesh
 * (Oxylus/src/Asset/AssetManager_GLTF.cpp:481-771) after the glTF accessors are read.  Pure host code (no CUDA).
 * The four meshoptimizer v1.2 calls of the reference (not vendored in /root/reference) are restated from their
 * published definitions — fetch remap, quantizeHalf, quantizeSnorm, computeMeshletBounds' normal cone — and the clusteriser
 * (meshopt_buildMeshlets) by a greedy spatial clusteriser of the same scheme (cluster_mode 1; not bit-compatible with
 * meshoptimizer's clusters); coarser LODs are caller-supplied index buffers or (auto_lods) generated by an edge-collapse
 * simplifier of meshopt_simplifyWithAttributes' scheme (oxb_simplify below).  Meshlets hold <= 64 vertices, <= 64 triangles
 * (Model.hpp:27-28).
 * ---------------------------------------------------------------------------------------------- */
typedef struct OxbMeshInput {
  const float* positions;  /* vertex_count x 3 */
  const float* normals;    /* vertex_count x 3, or NULL */
  const float* texcoords;  /* vertex_count x 2, or NULL */
  uint32_t vertex_count;
  uint32_t lod_count;      /* 1..OXC_MESH_MAX_LODS */
  const uint32_t* lod_indices[OXC_MESH_MAX_LODS]; /* triangle lists in input vertex numbering; [0] = full detail */
  uint32_t lod_index_counts[OXC_MESH_MAX_LODS];
  float lod_errors[OXC_MESH_MAX_LODS];            /* MeshLOD::error (cull_meshes.slang:35-57 LOD selection) */
  uint32_t cluster_mode;   /* 0: meshlets follow the caller's triangle order; 1: spatial clusteriser first (the role of
                              meshopt_buildMeshlets, AssetManager_GLTF.cpp:630-676): adjacency-first greedy growth, nearest
                              unused centroid when the meshlet has no unused neighbour */
  uint32_t auto_lods;      /* 1: lod_count must be 1; LOD 1.. are generated like AssetManager_GLTF.cpp:596-641 — each simplified
                              from the previous one to half its index count (normals as attributes, borders locked), MeshLOD::error
                              = previous error + the step's relative error; the chain ends when the simplifier stalls more than
                              50 % above its target, a step's error exceeds 0.5 or fewer than two triangles remain */
} OxbMeshInput;
typedef struct OxbMesh OxbMesh;
const char* oxb_last_error(void);
int oxb_build_mesh(const OxbMeshInput* in, OxbMesh** out);
uint64_t oxb_mesh_blob_size(const OxbMesh* m);            /* multiple of 16 */
uint32_t oxb_mesh_lod0_meshlet_count(const OxbMesh* m);   /* for MeshInstance::meshlet_instance_visibility_offset sums, Scene.cpp:1255-1260 */
/* Copies the mesh's blob to dst (= scene blob + base_offset, 16-byte aligned) and writes the OxcMesh record with every
 * offset (also inside the copied MeshLOD table) rebased by base_offset: the tables OxcSceneDesc expects. */
int oxb_mesh_emit(const OxbMesh* m, uint64_t base_offset, uint8_t* dst, OxcMesh* mesh_out);
void oxb_mesh_free(OxbMesh* m);
/* The role of meshopt_simplifyWithAttributes as build_gltf_mesh calls it (AssetManager_GLTF.cpp:604-628: attributes = normals
 * with weight 1, meshopt_SimplifyLockBorder, relative error): edge collapses onto existing vertices, quadric error metric over
 * positions + normal attribute quadrics per wedge, mesh borders locked, attribute seams kept closed, 2-manifolds stay
 * 2-manifold.  dst holds index_count entries; returns the new index count (it may stay above target_index_count) or a negative
 * OXC_E_* code.  normals may be NULL.  *result_error (may be NULL): largest position error of a performed collapse relative to
 * the extent of the vertex buffer.  Same scheme as meshoptimizer, not its bits (csrc/host/mesh_simplifier.cpp). */
int64_t oxb_simplify(uint32_t* dst, const uint32_t* indices, uint64_t index_count, const float* positions, const float* normals, uint32_t vertex_count,
                     uint64_t target_index_count, float target_error, float* result_error);

#ifdef __cplusplus
}
#endif
#endif /* OXCULL_H_ */
