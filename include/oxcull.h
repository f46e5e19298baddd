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
  OXC_STATUS_BAD_GEOMETRY = 1 << 1,     /* a micro index >= vertex_count or a vertex index >= Mesh::vertex_count (triangle skipped) */
  OXC_STATUS_SURVIVOR_OVERFLOW = 1 << 2,/* oxc_mgpu_exchange_frame: a rank's survivor list exceeded the gather capacity (truncated) */
  OXC_STATUS_ID_OVERFLOW = 1 << 3,      /* a vis-buffer id did not fit the id bits of the packing (pixel skipped) */
  OXC_STATUS_CLIP_OVERFLOW = 1 << 5,    /* more triangles crossed the near / guard-band planes than the clip queue holds (2^20): the rest was dropped */
  OXC_STATUS_BAD_MATERIAL = 1 << 6,     /* a MeshInstance::material_index outside the table of oxc_set_materials (rasterised as opaque) */
  OXC_STATUS_PEER_TIMEOUT = 1 << 4      /* oxc_mgpu_exchange_hiz: a peer did not raise its flag within 30 s (OXC_MGPU_TIMEOUT_MS); that frame's pyramid is incomplete */
};
int oxc_check_status(OxcContext* ctx, void* stream, uint32_t* flags_out /* may be NULL */);
/* CUDA-graph support: while a DEVICE camera buffer is bound, oxc_cull_meshes / oxc_cull_meshlets (and the InstCull refresh of
 * the triangle passes) read projection_view / position / near_clip / resolution / acceptable_lod_error from it instead of from the
 * by-value copy of their `camera` argument, so a captured frame replays with whatever camera the host copied into the buffer
 * before the launch (the host mirror's oxr_submit does exactly that).  The `camera` argument is still required: host-side
 * decisions (mesh_instance_count, "same camera as the InstCull cache") use it; pass the same camera for every pass of a frame.
 * NULL unbinds. */
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
 * (instance table changed => zero_fill_pass, :1651-1665). */
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

enum OxcImageFormat { OXC_IMAGE_RGBA8_UNORM = 0 /* alpha = byte 3 (sRGB variants: alpha is linear) */, OXC_IMAGE_R8_UNORM = 1 /* alpha only */ };
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
 * oxc_raster_visbuffer does this by itself since round 2 (it queues those triangles while it rasterises), so a host only needs
 * this entry point after a raster that ran with the queue exhausted (OXC_STATUS_CLIP_OVERFLOW); drawing a triangle twice is
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
 * (base index from cull_triangles_cmd.x, which is reset first).  Requires OxcCreateInfo::max_views >= clipmap_count.
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

/* Vis-buffer decode, geometry part (SURVEY §8f.1): passes/visbuffer_decode.slang:42-183 via RendererInstance's
 * "vis decode" pass.  Per pixel: texel -> (meshlet instance, triangle) (visbuffer.slang:31-36), triangle re-fetch
 * (scene.slang:363-399), world positions, compute_partial_derivatives (:42-92: analytic perspective-correct
 * barycentrics lambda and their per-pixel derivatives), gradient_of the vertex texture coordinates (:33-40) and the
 * geometric world normal normalize(mul(lambda, to_world_normals)) (:146-147) oct-encoded (common/encoding.slang:17-21).
 * The material evaluation (texture sampling, tangent frame from the sampled normal map, :118-183) needs the engine's
 * material and image tables and is not part of this library.  The frame's oxc_cull_meshes must have run (it resolves
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
