// oxc_types.cuh — device-side records of the H100 meshlet visibility pipeline.
//
// HBM layout (DESIGN.md §layout):
//   meshlet_instances  N x 8 B   (SceneGPU.hpp:106-109)      streamed, coalesced 64-bit loads
//   meshlet bounds     16 B each (SceneGPU.hpp:84-90)        one 128-bit load per meshlet
//   InstCull           I x 272 B per camera                   per-mesh-instance terms the reference
//                                                            recomputes per meshlet (mvp, 6 planes,
//                                                            normal matrix, scale) hoisted here; read
//                                                            through L1 as warp-broadcast 128-bit loads
//   InstGeom           I x 64 B                               resolved pointer chase for the triangle passes
//   visibility mask    ceil(M/32) x 4 B                       persistent across frames
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/oxcull.h"

namespace oxc {

// Per mesh instance, per camera.  17 x 16 B.  Every float is produced with the oracle's exact
// operation order (see oxc_exact.cuh), so hoisting it out of the per-meshlet loop is bit-neutral.
struct __align__(16) InstCull {
  float4 plane[6];     // normalize_plane(rows of mvp), cull.slang:58-71: (n.xyz, w)
  float4 mvp_row[4];   // mvp = mul(projection_view, world), row i
  float4 world_row[3]; // rows 0..2 of world
  float4 nrm[3];       // nrm[k].xyz = cross rows r_k of the normal matrix (scene.slang:291-298); nrm[0].w = max row length
  uint32_t bounds_lo, bounds_hi; // device address of MeshLOD::meshlet_bounds for the selected LOD
  uint32_t vis_offset;           // MeshInstance::meshlet_instance_visibility_offset
  uint32_t meshlet_count;        // meshlets emitted for this instance (0 = culled at mesh level)
};
static_assert(sizeof(InstCull) == 272, "InstCull");

// Per mesh instance: the mesh -> lod -> {meshlets, micro indices, vertex indices, positions} chase
// (cull_triangles.slang:44-52) resolved once per cull_meshes.
struct __align__(16) InstGeom {
  const OxcMeshlet* meshlets;
  const uint32_t* local_triangle_indices;
  const uint32_t* indirect_vertex_indices;
  const uint2* vertex_positions; // u16x4
  const uint32_t* vertex_normals; // 10:10:10 packed (scene.slang:486-489); null when the mesh has none
  const uint32_t* texture_coords; // half2 per vertex (scene.slang:491-497); null when the mesh has none
  uint32_t transform_index;
  uint32_t vertex_count;          // Mesh::vertex_count (visbuffer_decode.slang:115)
  uint32_t pad[2];
};
static_assert(sizeof(InstGeom) == 64, "InstGeom");

// Per view, per mesh instance (multi-view cull): just the six planes.
struct __align__(16) InstPlanes {
  float4 plane[6];
};

// Per clipmap, per mesh instance (shadow-clipmap cull): planes + rows of mul(clipmap.pv, world).
struct __align__(16) InstView {
  float4 plane[6];
  float4 row[4];
};

struct HizDesc {
  const float* data;
  uint32_t width, height, levels;
  uint32_t level_offset[OXC_HIZ_MAX_LEVELS];
};

struct CullParams {
  const uint2* slabs; // (mesh instance, meshlet) of meshlet-instance index 32 k, written by the expansion
  const OxcMeshletInstance* meshlet_instances;
  const InstCull* inst;
  OxcMeshletInstanceVisibility* vis;
  uint32_t* visible_indices;
  uint32_t* mask;
  OxcDispatchIndirectCommand* tri_cmd;
  const uint32_t* id_base; // may be null
  HizDesc hiz;
  float cam_pos[3];
  float near_clip;
  const OxcCullCamera* cam_dev; // non-null: position / near_clip are read from this device camera instead
};

} // namespace oxc
