// kernels_cull.cuh — mesh-level cull + expansion, the two-pass meshlet cull, the multi-view cull.
// Reference: Oxylus/src/Render/Shaders/passes/{cull_meshes,cull_meshlets_hiz,cull_meshlets,cull_meshlets_hpb}.slang
#pragma once
#include "oxc_filtered.cuh"

namespace oxc {

#ifdef OXC_HOST_SOUNDNESS_HARNESS
OXC_DI void prefetch_l1(const void*) {} // host builds of the headers (tests/): a hint has no result
#else
OXC_DI void prefetch_l1(const void* ptr) { asm volatile("prefetch.global.L1 [%0];" ::"l"(ptr)); }
#endif

#ifndef OXC_CULL_MESHES_THREADS
#define OXC_CULL_MESHES_THREADS 64
#endif
constexpr int CULL_MESHES_THREADS = OXC_CULL_MESHES_THREADS;
constexpr int CULL_THREADS = 256;
#ifndef OXC_CULL_ITEMS
#define OXC_CULL_ITEMS 2
#endif
#ifndef OXC_CULL_MIN_BLOCKS
#define OXC_CULL_MIN_BLOCKS 3
#endif
constexpr int CULL_ITEMS = OXC_CULL_ITEMS;               // meshlet instances per thread per tile
constexpr int CULL_TILE = CULL_THREADS * CULL_ITEMS;   // 512 per CTA iteration -> one atomic per 512

struct MeshesParams {
  const OxcMesh* meshes;
  OxcMeshInstance* mesh_instances;
  const OxcTransformWorld* transforms;
  InstCull* inst;
  InstGeom* geom;
  const float* lod_aabb; // [mesh][OXC_MESH_MAX_LODS][6]: union AABB (min xyz, max xyz) of the decoded meshlet boxes
  uint32_t* counts;      // per mesh instance of the shard (index - first)
  uint32_t* block_sums;
  uint32_t first, count; // shard
  uint32_t flags;
  int select;            // 1: full cull_meshes (frustum + LOD select + counts); 0: refresh InstCull for a new camera only
  OxcCullCamera cam;
  const OxcCullCamera* cam_dev; // oxc_bind_camera_buffer: read the camera from device memory (CUDA-graph replays with a new camera)
};

// cull_meshes.slang:17-61 — one thread per mesh instance of the shard.  Besides the reference's outputs
// (lod_index write-back, meshlet count) it materialises InstCull / InstGeom for the later passes.
__global__ void __launch_bounds__(CULL_MESHES_THREADS) k_cull_meshes(const __grid_constant__ MeshesParams pp) {
  const MeshesParams& p = pp;
  const OxcCullCamera& cam = pp.cam_dev ? *pp.cam_dev : pp.cam;
  const uint32_t local = blockIdx.x * CULL_MESHES_THREADS + threadIdx.x;
  uint32_t meshlet_count = 0;
  if (local < p.count) {
    const uint32_t mi = p.first + local;
    OxcMeshInstance inst = p.mesh_instances[mi];
    const OxcMesh* mesh = &p.meshes[inst.mesh_index];
    const float* world = p.transforms[inst.transform_index].world;
    float w[16];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const float4 c = __ldg(reinterpret_cast<const float4*>(world) + k);
      w[k * 4 + 0] = c.x; w[k * 4 + 1] = c.y; w[k * 4 + 2] = c.z; w[k * 4 + 3] = c.w;
    }
    float4 rows[4], planes[6];
    mul_mm_rows(cam.projection_view, w, rows); // :32
    frustum_planes(rows, planes);
    const OxcMeshLOD* lods = reinterpret_cast<const OxcMeshLOD*>(mesh->lods);
    uint32_t lod_index = inst.lod_index;
    if (p.select) {
      lod_index = 0;
      const float bcx = mesh->bounds.aabb_center[0], bcy = mesh->bounds.aabb_center[1], bcz = mesh->bounds.aabb_center[2];
      const float bex = mesh->bounds.aabb_extent[0], bey = mesh->bounds.aabb_extent[1], bez = mesh->bounds.aabb_extent[2];
      if ((p.flags & OXC_CULL_TEST_FRUSTUM) && test_frustum_rows(planes, bcx, bcy, bcz, bex, bey, bez)) { // :34
        if (p.flags & OXC_CULL_SELECT_LOD) { // :35-57
          const float4 w0 = make_float4(w[0], w[4], w[8], w[12]), w1 = make_float4(w[1], w[5], w[9], w[13]),
                       w2 = make_float4(w[2], w[6], w[10], w[14]);
          const float cx = row_dot4(w0, bcx, bcy, bcz, 1.0f), cy = row_dot4(w1, bcx, bcy, bcz, 1.0f),
                      cz = row_dot4(w2, bcx, bcy, bcz, 1.0f);
          const float ex = fabsf(row_dot4(w0, bex, bey, bez, 0.0f)), ey = fabsf(row_dot4(w1, bex, bey, bez, 0.0f)),
                      ez = fabsf(row_dot4(w2, bex, bey, bez, 0.0f));
          const float rough_extent = omax(ex, omax(ey, ez));
          const float dist = omax(fs(length3(fs(cx, cam.position[0]), fs(cy, cam.position[1]), fs(cz, cam.position[2])),
                                     fm(0.5f, rough_extent)), 0.0f);
          const float pixel_size_at_1m = fd(2.0f, omax(cam.resolution[0], cam.resolution[1]));
          const float aabb_size_at_1m = fd(rough_extent, dist);
          const float rough_pixel_size = fd(aabb_size_at_1m, pixel_size_at_1m);
          for (uint32_t i = 1; i < mesh->lod_count; i++) {
            const float err = fm(rough_pixel_size, lods[i].error);
            if (err < cam.acceptable_lod_error) lod_index = i;
            else break;
          }
        }
        meshlet_count = lods[lod_index].meshlet_count; // :59
      }
      if (meshlet_count > 0) p.mesh_instances[mi].lod_index = lod_index; // :76
      else lod_index = inst.lod_index;                                   // untouched when culled
    } else {
      meshlet_count = p.inst[mi].meshlet_count; // keep what the last cull_meshes decided
    }
    const OxcMeshLOD* lod = &lods[lod_index];
    InstCull ic;
#pragma unroll
    for (int k = 0; k < 6; k++) ic.plane[k] = planes[k];
#pragma unroll
    for (int k = 0; k < 4; k++) ic.mvp_row[k] = rows[k];
    ic.world_row[0] = make_float4(w[0], w[4], w[8], w[12]);
    ic.world_row[1] = make_float4(w[1], w[5], w[9], w[13]);
    ic.world_row[2] = make_float4(w[2], w[6], w[10], w[14]);
    // scene.slang:291-298: basis[i] = column i of world3; r0 = cross(b1,b2), r1 = cross(b2,b0), r2 = cross(b0,b1)
    const float b0x = w[0], b0y = w[1], b0z = w[2], b1x = w[4], b1y = w[5], b1z = w[6], b2x = w[8], b2y = w[9], b2z = w[10];
#define OXC_CROSS(ax, ay, az, bx, by, bz) \
  make_float4(fs(fm(ay, bz), fm(az, by)), fs(fm(az, bx), fm(ax, bz)), fs(fm(ax, by), fm(ay, bx)), 0.0f)
    ic.nrm[0] = OXC_CROSS(b1x, b1y, b1z, b2x, b2y, b2z);
    ic.nrm[1] = OXC_CROSS(b2x, b2y, b2z, b0x, b0y, b0z);
    ic.nrm[2] = OXC_CROSS(b0x, b0y, b0z, b1x, b1y, b1z);
#undef OXC_CROSS
    // scene.slang:304-309 (Slang world[i] = row i)
    ic.nrm[0].w = omax(length3(w[0], w[4], w[8]), omax(length3(w[1], w[5], w[9]), length3(w[2], w[6], w[10])));
    {  // nrm[1].w: 1.0 when every mvp entry is finite and |x| <= 2^60 (precondition of the filtered projection)
      bool ok = true;
#pragma unroll
      for (int k = 0; k < 4; k++)
        ok = ok && fabsf(rows[k].x) <= 1.152921504606847e18f && fabsf(rows[k].y) <= 1.152921504606847e18f &&
             fabsf(rows[k].z) <= 1.152921504606847e18f && fabsf(rows[k].w) <= 1.152921504606847e18f;
      ic.nrm[1].w = ok ? 1.0f : 0.0f;
    }
    {  // nrm[2].w: 1.0 when every meshlet box of the selected LOD is provably inside all six planes for the canonical test, so
       // the per-meshlet frustum test can be skipped (bound: union_box_inside_frustum, oxc_filtered.cuh)
      const float* ua = p.lod_aabb + ((size_t)inst.mesh_index * OXC_MESH_MAX_LODS + lod_index) * 6;
      ic.nrm[2].w = union_box_inside_frustum(planes, ua, p.lod_aabb != nullptr) ? 1.0f : 0.0f;
    }
    const uint64_t baddr = lod->meshlet_bounds;
    ic.bounds_lo = (uint32_t)baddr;
    ic.bounds_hi = (uint32_t)(baddr >> 32);
    ic.vis_offset = inst.meshlet_instance_visibility_offset;
    ic.meshlet_count = meshlet_count;
    p.inst[mi] = ic;
    if (p.select) {
      InstGeom g;
      g.meshlets = reinterpret_cast<const OxcMeshlet*>(lod->meshlets);
      g.local_triangle_indices = reinterpret_cast<const uint32_t*>(lod->local_triangle_indices);
      g.indirect_vertex_indices = reinterpret_cast<const uint32_t*>(lod->indirect_vertex_indices);
      g.vertex_positions = reinterpret_cast<const uint2*>(mesh->vertex_positions);
      g.vertex_normals = reinterpret_cast<const uint32_t*>(mesh->vertex_normals);
      g.texture_coords = reinterpret_cast<const uint32_t*>(mesh->texture_coords);
      g.transform_index = inst.transform_index;
      g.vertex_count = mesh->vertex_count;
      g.pad[0] = g.pad[1] = 0;
      p.geom[mi] = g;
      p.counts[local] = meshlet_count;
    }
  }
  if (!p.select) return;
  // block sum of meshlet counts (WaveActiveSum :64, one level up)
  __shared__ uint32_t warp_sums[CULL_MESHES_THREADS / 32];
  uint32_t v = meshlet_count;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < CULL_MESHES_THREADS / 32; k++) s += warp_sums[k];
    p.block_sums[blockIdx.x] = s;
  }
}

// Multi-GPU id base without communication: the number of meshlet instances the mesh instances [0, first) emit
// under this camera (same frustum test + LOD selection as k_cull_meshes, count only).  Every rank can evaluate it
// locally because the small tables are replicated; integer sum => order independent.
__global__ void __launch_bounds__(CULL_MESHES_THREADS) k_count_prefix_meshlets(const __grid_constant__ MeshesParams p, uint32_t* id_base) {
  const OxcCullCamera& cam = p.cam_dev ? *p.cam_dev : p.cam;
  const uint32_t mi = blockIdx.x * CULL_MESHES_THREADS + threadIdx.x;
  uint32_t meshlet_count = 0;
  if (mi < p.first) {
    const OxcMeshInstance inst = p.mesh_instances[mi];
    const OxcMesh* mesh = &p.meshes[inst.mesh_index];
    const float* world = p.transforms[inst.transform_index].world;
    float w[16];
#pragma unroll
    for (int k = 0; k < 16; k++) w[k] = world[k];
    float4 rows[4], planes[6];
    mul_mm_rows(cam.projection_view, w, rows);
    frustum_planes(rows, planes);
    const OxcMeshLOD* lods = reinterpret_cast<const OxcMeshLOD*>(mesh->lods);
    const float bcx = mesh->bounds.aabb_center[0], bcy = mesh->bounds.aabb_center[1], bcz = mesh->bounds.aabb_center[2];
    const float bex = mesh->bounds.aabb_extent[0], bey = mesh->bounds.aabb_extent[1], bez = mesh->bounds.aabb_extent[2];
    if ((p.flags & OXC_CULL_TEST_FRUSTUM) && test_frustum_rows(planes, bcx, bcy, bcz, bex, bey, bez)) {
      uint32_t lod_index = 0;
      if (p.flags & OXC_CULL_SELECT_LOD) {
        const float4 w0 = make_float4(w[0], w[4], w[8], w[12]), w1 = make_float4(w[1], w[5], w[9], w[13]),
                     w2 = make_float4(w[2], w[6], w[10], w[14]);
        const float cx = row_dot4(w0, bcx, bcy, bcz, 1.0f), cy = row_dot4(w1, bcx, bcy, bcz, 1.0f), cz = row_dot4(w2, bcx, bcy, bcz, 1.0f);
        const float ex = fabsf(row_dot4(w0, bex, bey, bez, 0.0f)), ey = fabsf(row_dot4(w1, bex, bey, bez, 0.0f)),
                    ez = fabsf(row_dot4(w2, bex, bey, bez, 0.0f));
        const float rough_extent = omax(ex, omax(ey, ez));
        const float dist = omax(fs(length3(fs(cx, cam.position[0]), fs(cy, cam.position[1]), fs(cz, cam.position[2])),
                                   fm(0.5f, rough_extent)), 0.0f);
        const float pixel_size_at_1m = fd(2.0f, omax(cam.resolution[0], cam.resolution[1]));
        const float rough_pixel_size = fd(fd(rough_extent, dist), pixel_size_at_1m);
        for (uint32_t i = 1; i < mesh->lod_count; i++) {
          if (fm(rough_pixel_size, lods[i].error) < cam.acceptable_lod_error) lod_index = i;
          else break;
        }
      }
      meshlet_count = lods[lod_index].meshlet_count;
    }
  }
  uint32_t v = meshlet_count;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0 && v) atomicAdd(id_base, v);
}

// One-time per scene: union AABB of the DECODED meshlet boxes (c +- e/2) of every (mesh, LOD).  One warp per
// (mesh, lod).  Feeds the instance-level "provably inside the frustum" shortcut.
__global__ void k_lod_union_aabb(const OxcMesh* __restrict__ meshes, uint32_t n_meshes, float* __restrict__ out) {
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n_meshes * OXC_MESH_MAX_LODS) return;
  const uint32_t m = w / OXC_MESH_MAX_LODS, l = w % OXC_MESH_MAX_LODS;
  float mn[3] = {3.0e38f, 3.0e38f, 3.0e38f}, mx[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
  bool bad = false;
  if (l < meshes[m].lod_count) {
    const OxcMeshLOD* lod = reinterpret_cast<const OxcMeshLOD*>(meshes[m].lods) + l;
    const uint4* b = reinterpret_cast<const uint4*>(lod->meshlet_bounds);
    for (uint32_t i = lane; i < lod->meshlet_bounds_count; i += 32) {
      const uint4 v = b[i];
      const float c[3] = {dequantize_half(v.x & 0xFFFFu), dequantize_half(v.x >> 16), dequantize_half(v.y & 0xFFFFu)};
      const float e[3] = {dequantize_half(v.z & 0xFFFFu), dequantize_half(v.z >> 16), dequantize_half(v.w & 0xFFFFu)};
#pragma unroll
      for (int a = 0; a < 3; a++) {
        const float h = fabsf(e[a]) * 0.5f;
        const float a0 = c[a] - h, a1 = c[a] + h;
        bad = bad || !(fabsf(a0) <= 3.0e38f) || !(fabsf(a1) <= 3.0e38f) || !(e[a] >= 0.0f); // the shortcut's bound assumes h >= 0
        mn[a] = fminf(mn[a], a0); mx[a] = fmaxf(mx[a], a1);
      }
    }
  } else bad = true;
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
  bad = __any_sync(0xffffffffu, bad);
  if (lane == 0) {
    float* o = out + (size_t)w * 6;
    if (bad) { o[0] = o[1] = o[2] = 1.0f; o[3] = o[4] = o[5] = -1.0f; } // empty => shortcut disabled
    else { o[0] = mn[0]; o[1] = mn[1]; o[2] = mn[2]; o[3] = mx[0]; o[4] = mx[1]; o[5] = mx[2]; }
  }
}

// exclusive scan of the per-block sums in one CTA; publishes the totals the reference accumulates with
// atomics (cull_meshes.slang:66-72): visibility.total and cull_meshlets_cmd.x = ceil(total / 64).
__global__ void __launch_bounds__(1024) k_scan_block_sums(uint32_t* block_sums, uint32_t n_blocks,
                                                          OxcMeshletInstanceVisibility* vis,
                                                          OxcDispatchIndirectCommand* cmd, uint32_t capacity, uint32_t* status) {
  __shared__ uint32_t warp_tot[32];
  __shared__ uint32_t carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (uint32_t base = 0; base < n_blocks; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    const uint32_t v = i < n_blocks ? block_sums[i] : 0u;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
      if ((threadIdx.x & 31) >= o) inc += t;
    }
    if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = inc;
    __syncthreads();
    if (threadIdx.x < 32) {
      uint32_t w = warp_tot[threadIdx.x], winc = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
        if (threadIdx.x >= o) winc += t;
      }
      warp_tot[threadIdx.x] = winc - w; // exclusive
    }
    __syncthreads();
    const uint32_t carry = carry_s;
    const uint32_t excl = carry + warp_tot[threadIdx.x >> 5] + inc - v;
    if (i < n_blocks) block_sums[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    uint32_t total = carry_s;
    if (total > capacity) { // backstop (oxc_set_scene already refuses scenes that cannot fit): clamp, never write out of bounds
      total = capacity;
      atomicOr(status, (uint32_t)OXC_STATUS_MESHLET_OVERFLOW);
    }
    vis->total_visible_meshlet_instances = total;
    vis->early_visible_meshlet_instances = 0;
    vis->late_visible_meshlet_instances = 0;
    cmd->x = (total + 63u) / 64u; // CULLING_MESHLET_COUNT, cull_meshes.slang:70-71
    cmd->y = 1;
    cmd->z = 1;
  }
}

// cull_meshes.slang:74-84 — expansion.  Deterministic: ascending mesh instance, ascending meshlet.
// One warp per mesh instance writes its run with coalesced 64-bit stores.  EXPAND_SPLIT CTAs share one 256-instance block of
// the scan (each redoes the block's cheap scan and expands 256 / EXPAND_SPLIT of its instances): with one CTA per block the
// 8 MB of a 1 M scene would be written by only ~25 CTAs.
constexpr int EXPAND_SPLIT = 8;
__global__ void __launch_bounds__(CULL_MESHES_THREADS) k_expand_meshlet_instances(const uint32_t* __restrict__ counts,
                                                                                 const uint32_t* __restrict__ block_offsets,
                                                                                 uint32_t first, uint32_t count,
                                                                                 OxcMeshletInstance* out, uint32_t capacity, uint2* slabs) {
  __shared__ uint32_t offs[CULL_MESHES_THREADS];
  __shared__ uint32_t cnts[CULL_MESHES_THREADS];
  __shared__ uint32_t warp_tot[CULL_MESHES_THREADS / 32];
  const uint32_t block = blockIdx.x / EXPAND_SPLIT, part = blockIdx.x % EXPAND_SPLIT;
  const uint32_t local = block * CULL_MESHES_THREADS + threadIdx.x;
  const uint32_t v = local < count ? counts[local] : 0u;
  uint32_t inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
    if ((threadIdx.x & 31) >= o) inc += t;
  }
  if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = inc;
  __syncthreads();
  uint32_t wbase = 0;
  for (int k = 0; k < (int)(threadIdx.x >> 5); k++) wbase += warp_tot[k];
  offs[threadIdx.x] = block_offsets[block] + wbase + inc - v;
  cnts[threadIdx.x] = v;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint2* o2 = reinterpret_cast<uint2*>(out);
  constexpr uint32_t PER_PART = CULL_MESHES_THREADS / EXPAND_SPLIT;
  for (uint32_t k = part * PER_PART + warp; k < (part + 1) * PER_PART; k += CULL_MESHES_THREADS / 32) {
    const uint32_t n = cnts[k];
    if (n == 0) continue;
    const uint32_t base = offs[k];
    const uint32_t mi = first + block * CULL_MESHES_THREADS + k;
    for (uint32_t j = lane; j < n && base + j < capacity; j += 32) {
      o2[base + j] = make_uint2(mi, j);
      if (((base + j) & 31u) == 0u) slabs[(base + j) >> 5] = make_uint2(mi, j); // slab table: 8 B per 32 meshlet instances
    }
  }
}

// ------------------------------------------------------------------------------------------------
// The meshlet cull.  cull_meshlets_hiz.slang:19-88 (HIZ path) / cull_meshlets.slang:21-73 (plain).
//   OCC  = HAS_FLAG(CULL_FLAGS, TestOcclusion)   (mask read/modify, :45-51,81-87)
//   LATE = HAS_FLAG(CULL_FLAGS, LatePass)
//   HIZ  = use_hiz: project_aabb + test_occlusion run when OCC || LATE (:61, any-bit HAS_FLAG)
//   ZERO = the pyramid is known to be the per-frame cleared image (early pass, SURVEY §8a quirk 1)
//
// Round-2 design: a three-stage pipeline with WARP-PRIVATE shared-memory queues, so every expensive stage runs on 32 live
// lanes whatever fraction of the input reaches it (running each stage on the lanes of a fixed tile leaves most lanes of the
// expensive occlusion stage idle).
//
//   stage 0  one lane per meshlet-instance INDEX, 32 consecutive indices ("slab") per warp.  The (mesh instance, meshlet)
//            pair is recovered from the slab table (8 B per 32 meshlets, written by the expansion) plus the per-instance
//            meshlet counts — the 8 B/meshlet id stream of round 1 is no longer read.  Mask bit -> was_visible.
//            Early pass: only was_visible items need any work (:57) -> queue 0.   Late pass: every item -> stage A.
//   stage A  one 128-bit bounds load, half decode, frustum (instance-inside flag, else centre-inside filter, else
//            canonical), filtered cone.  Items that still need the Hi-Z test -> queue 1; the others are final.
//   stage B  filtered projection + occlusion on 32 queue entries; margin-ambiguous entries -> queue 2.
//   stage C  canonical project_aabb + test_occlusion on 32 ambiguous entries (a fraction of a percent of the input).
//   finish   mask update = one XOR of the changed bits per touched word per warp (reference: an atomic or/and per lane,
//            :81-87); survivors go to a warp-private staging buffer flushed with ONE pair of global atomics per ~100
//            survivors (reference: three atomics per surviving lane, :70-78).
// A queue holds < 32 entries between slabs; a stage runs as soon as its queue reaches 32, and once more (partially filled)
// when the warp runs out of slabs.  Outputs are bit-identical to the canonical path for every input (oxc_filtered.cuh);
// survivor ORDER is unspecified, as in the reference (atomics order, SURVEY §8a quirk 8).
// ------------------------------------------------------------------------------------------------
constexpr int CULL_WARPS = CULL_THREADS / 32;
constexpr int CULL_Q = 64;        // queue capacity per warp (< 32 carried over + <= 32 appended)
constexpr int CULL_EMIT = 128;    // survivor staging per warp (flushed above 96)

// queue 0 entry (early pass): where the bounds are + what to update.  16 + 4 B.
// queue 1 / 2 entry: decoded bounds + the same bookkeeping.  32 + 4 B.
template <bool Q0>
struct __align__(16) CullShared {
  uint32_t hiz_off[OXC_HIZ_MAX_LEVELS];
  float s8_lut[256]; // scene.slang:408-418: i8 / 127.0 for every i8 (IEEE divide, once per CTA)
  uint4 q0a[CULL_WARPS][Q0 ? CULL_Q : 1];     // bounds ptr lo, hi | mesh instance | meshlet-instance index
  uint32_t q0b[CULL_WARPS][Q0 ? CULL_Q : 1];  // mask bit index (was_visible is implied)
  uint4 q1a[CULL_WARPS][CULL_Q];     // cx cy cz ex
  uint4 q1b[CULL_WARPS][CULL_Q];     // ey ez | mesh instance | meshlet-instance index
  uint32_t q1c[CULL_WARPS][CULL_Q];  // mask bit index | was_visible << 31
  uint4 q2a[CULL_WARPS][CULL_Q];
  uint4 q2b[CULL_WARPS][CULL_Q];
  uint32_t q2c[CULL_WARPS][CULL_Q];
  uint32_t emit[CULL_WARPS][CULL_EMIT];
};

template <bool HIZ, bool OCC, bool LATE, bool ZERO>
struct CullWarp {
  using Shared = CullShared<OCC && !LATE>;
  const CullParams& p;
  Shared& sh;
  const uint32_t lane, warp, lane_lt;
  const uint32_t early_count, id_base;
  float cam_pos[3], near_clip; // from the kernel parameters, or from the bound device camera
  uint32_t n0 = 0, n1 = 0, n2 = 0, ne = 0; // warp-uniform fill levels

  OXC_DI CullWarp(const CullParams& p_, Shared& sh_, uint32_t early, uint32_t idb)
      : p(p_), sh(sh_), lane(threadIdx.x & 31), warp(threadIdx.x >> 5), lane_lt((1u << (threadIdx.x & 31)) - 1u), early_count(early), id_base(idb) {
    if (p_.cam_dev) {
      cam_pos[0] = p_.cam_dev->position[0]; cam_pos[1] = p_.cam_dev->position[1]; cam_pos[2] = p_.cam_dev->position[2];
      near_clip = p_.cam_dev->near_clip;
    } else {
      cam_pos[0] = p_.cam_pos[0]; cam_pos[1] = p_.cam_pos[1]; cam_pos[2] = p_.cam_pos[2];
      near_clip = p_.near_clip;
    }
  }

  // ---- survivor staging: one pair of global atomics per flush ----
  OXC_DI void flush() {
    __syncwarp();
    uint32_t base = 0;
    if (lane == 0 && ne) {
      if (!HIZ) base = atomicAdd(&p.tri_cmd->x, ne);                                            // cull_meshlets.slang:64
      else {
        if (!LATE) base = atomicAdd(&p.vis->early_visible_meshlet_instances, ne);              // :70
        else base = atomicAdd(&p.vis->late_visible_meshlet_instances, ne) + early_count;        // :72-73
        atomicAdd(&p.tri_cmd->x, ne);                                                           // :78
      }
    }
    base = __shfl_sync(0xffffffffu, base, 0);
    for (uint32_t j = lane; j < ne; j += 32) p.visible_indices[base + j] = sh.emit[warp][j];    // :76
    __syncwarp();
    ne = 0;
  }

  // ---- verdict -> mask + survivor list.  vi = mask bit index, idx = local meshlet-instance index ----
  OXC_DI void finish(bool active, bool visible, bool was_visible, uint32_t vi, uint32_t idx) {
    if (OCC) { // :81-87 mask rewrite: XOR of the changed bits, aggregated per word within the warp
      const bool changed = active && (visible != was_visible);
      if (__any_sync(0xffffffffu, changed)) {
        const uint32_t word = vi >> 5, bit = 1u << (vi & 31);
        const uint32_t peers = __match_any_sync(0xffffffffu, changed ? word : 0xFFFFFFFFu);
        const uint32_t delta = __reduce_or_sync(peers, changed ? bit : 0u);
        if (changed && lane == (uint32_t)(__ffs(peers) - 1)) atomicXor(&p.mask[word], delta);
      }
    }
    const bool emit = active && visible && (!LATE || !was_visible); // :67
    const uint32_t bal = __ballot_sync(0xffffffffu, emit);
    if (bal) {
      if (emit) sh.emit[warp][ne + __popc(bal & lane_lt)] = idx + id_base;
      ne += __popc(bal);
      if (ne > CULL_EMIT - 32) flush();
    }
  }

  // ---- stage C: canonical evaluation of `cnt` margin-ambiguous entries from the top of queue 2 ----
  OXC_DI void stage_c(uint32_t cnt) {
    __syncwarp();
    const bool active = lane < cnt;
    bool visible = true, was = false;
    uint32_t vi = 0, idx = 0;
    if (active) {
      const uint32_t j = n2 - cnt + lane;
      const uint4 a = sh.q2a[warp][j], b = sh.q2b[warp][j];
      const uint32_t c = sh.q2c[warp][j];
      vi = c & 0x7FFFFFFFu; was = (c >> 31) != 0; idx = b.w;
      const InstCull* ic = p.inst + b.z;
      const float4 r0 = __ldg(&ic->mvp_row[0]), r1 = __ldg(&ic->mvp_row[1]), r2 = __ldg(&ic->mvp_row[2]), r3 = __ldg(&ic->mvp_row[3]);
      ScreenAabb sa;
      if (project_aabb(r0, r1, r2, r3, near_clip, __uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(a.w),
                       __uint_as_float(b.x), __uint_as_float(b.y), sa))
        visible = !test_occlusion(sa, p.hiz.data, p.hiz.width, p.hiz.height, p.hiz.levels, sh.hiz_off);
    }
    n2 -= cnt;
    __syncwarp();
    finish(active, visible, was, vi, idx);
  }

  // ---- stage B: filtered projection + occlusion on `cnt` entries from the top of queue 1 ----
  OXC_DI void stage_b(uint32_t cnt) {
    __syncwarp();
    const bool active = lane < cnt;
    Tri t = TRI_TRUE;
    bool was = false;
    uint32_t vi = 0, idx = 0, c = 0;
    uint4 a = make_uint4(0, 0, 0, 0), b = a;
    if (active) {
      const uint32_t j = n1 - cnt + lane;
      a = sh.q1a[warp][j]; b = sh.q1b[warp][j]; c = sh.q1c[warp][j];
      vi = c & 0x7FFFFFFFu; was = (c >> 31) != 0; idx = b.w;
      const InstCull* ic = p.inst + b.z;
      const float4 r0 = __ldg(&ic->mvp_row[0]), r1 = __ldg(&ic->mvp_row[1]), r2 = __ldg(&ic->mvp_row[2]), r3 = __ldg(&ic->mvp_row[3]);
      t = occlusion_visible_fast(r0, r1, r2, r3, near_clip, __uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z),
                                 __uint_as_float(a.w), __uint_as_float(b.x), __uint_as_float(b.y), p.hiz.data, p.hiz.width, p.hiz.height,
                                 p.hiz.levels, sh.hiz_off, __ldg(&ic->nrm[1].w) != 0.0f);
    }
    n1 -= cnt;
    __syncwarp();
    const bool amb = active && t == TRI_AMBIGUOUS;
    const uint32_t bal = __ballot_sync(0xffffffffu, amb);
    if (bal) {
      if (amb) {
        const uint32_t j = n2 + __popc(bal & lane_lt);
        sh.q2a[warp][j] = a; sh.q2b[warp][j] = b; sh.q2c[warp][j] = c;
      }
      n2 += __popc(bal);
    }
    finish(active && !amb, t == TRI_TRUE, was, vi, idx);
    if (n2 >= 32) stage_c(32);
  }

  // ---- stage A: bounds -> frustum -> cone; `active` lanes hold (bounds pointer, mesh instance, index, mask bit, was) ----
  OXC_DI void stage_a(bool active, const uint4 b, uint32_t inst, uint32_t idx, uint32_t vi, bool was) {
    bool visible = active;
    bool queue = false;
    float cx = 0.f, cy = 0.f, cz = 0.f, ex = 0.f, ey = 0.f, ez = 0.f;
    if (active) {
      const InstCull* ic = p.inst + inst;
      // scene.slang:401-435 unpack: u16x3 center | i8x2 cone xy | u16x3 extent | i8 cone z | i8 cutoff
      cx = dequantize_half_hw(b.x & 0xFFFFu); cy = dequantize_half_hw(b.x >> 16); cz = dequantize_half_hw(b.y & 0xFFFFu);
      ex = dequantize_half_hw(b.z & 0xFFFFu); ey = dequantize_half_hw(b.z >> 16); ez = dequantize_half_hw(b.w & 0xFFFFu);
      // :59 frustum (the three tests commute).  Skipped when the whole instance is provably inside every plane for the
      // canonical test (InstCull::nrm[2].w, see k_cull_meshes); else decided by the centre-inside filter when it can.
      if (__ldg(&ic->nrm[2].w) == 0.0f && !frustum_centre_inside(ic->plane, cx, cy, cz, ex, ey, ez))
        visible = test_frustum_planes(ic->plane, cx, cy, cz, ex, ey, ez);
      // :58 cone
      const float cutoff = sh.s8_lut[((b.w >> 24) + 128u) & 0xFFu];
      if (visible && cutoff < 1.0f) {
        const ConeInputs ci = cone_inputs(ic, cx, cy, cz, ex, ey, ez, sh.s8_lut[(((b.y >> 16) & 0xFFu) + 128u) & 0xFFu],
                                          sh.s8_lut[((b.y >> 24) + 128u) & 0xFFu], sh.s8_lut[(((b.w >> 16) & 0xFFu) + 128u) & 0xFFu],
                                          cam_pos[0], cam_pos[1], cam_pos[2]);
        const Tri t = cone_visible_fast(ci, cutoff);
        visible = t == TRI_AMBIGUOUS ? cone_visible_exact(ci, cutoff) : (t == TRI_TRUE);
      }
      // :61-65 occlusion
      if (HIZ && (OCC || LATE) && visible) {
        queue = true;
        if (ZERO) queue = !cleared_hiz_surely_visible(__ldg(&ic->mvp_row[2]), __ldg(&ic->mvp_row[3]), cx, cy, cz, ex, ey, ez);
      }
    }
    if (HIZ) {
      const uint32_t bal = __ballot_sync(0xffffffffu, queue);
      if (bal) {
        if (queue) {
          const uint32_t j = n1 + __popc(bal & lane_lt);
          sh.q1a[warp][j] = make_uint4(__float_as_uint(cx), __float_as_uint(cy), __float_as_uint(cz), __float_as_uint(ex));
          sh.q1b[warp][j] = make_uint4(__float_as_uint(ey), __float_as_uint(ez), inst, idx);
          sh.q1c[warp][j] = vi | (was ? 0x80000000u : 0u);
        }
        n1 += __popc(bal);
      }
    }
    finish(active && !queue, visible, was, vi, idx);
    if (HIZ && n1 >= 32) stage_b(32);
  }

  // ---- stage A fed from queue 0 (early pass) ----
  OXC_DI void stage_a_from_q0(uint32_t cnt) {
    __syncwarp();
    const bool active = lane < cnt;
    uint4 a = make_uint4(0, 0, 0, 0);
    uint32_t vi = 0;
    if (active) { a = sh.q0a[warp][n0 - cnt + lane]; vi = sh.q0b[warp][n0 - cnt + lane]; }
    n0 -= cnt;
    __syncwarp();
    uint4 b = make_uint4(0, 0, 0, 0);
    if (active) b = __ldg(reinterpret_cast<const uint4*>(((uint64_t)a.y << 32) | a.x)); // MeshletBounds of a was_visible item
    stage_a(active, b, a.z, a.w, vi, true);
  }

  // ---- stage 0, software-pipelined over the warp's slabs ----
  // The index -> (mesh instance, meshlet) -> {mask word, bounds} resolution is a chain of three dependent loads; a warp
  // owns only a handful of slabs, so the chain of slab k+1.. is issued while slab k is being tested:
  //     iteration k:   issue  slab-table entry of k+3,  InstCull tail of k+2,  mask word + bounds of k+1;   test k
  // (without the pipeline the kernel waits on the dependent InstCull -> mask -> bounds chain of every slab: latency-bound.)
  struct Resolved { // slab whose mask word / bounds are in flight
    uint4 bounds;
    uint32_t maskw, inst, idx, vi;
    bool valid;
  };

  OXC_DI uint2 load_slab_entry(uint32_t s, uint32_t n_slabs) const { return s < n_slabs ? __ldg(&p.slabs[s]) : make_uint2(0u, 0u); }
  OXC_DI uint4 load_tail(uint32_t s, uint32_t n_slabs, uint2 sl) const {
    return s < n_slabs ? __ldg(reinterpret_cast<const uint4*>(&p.inst[sl.x].bounds_lo)) : make_uint4(0, 0, 0, 0xFFFFFFFFu);
  }
  // finish the resolution of slab s (entry sl, first instance's tail already here) and put the mask word and — when the
  // pass needs every item (late / no mask) — the bounds in flight
  OXC_DI Resolved resolve(uint32_t s, uint32_t total, uint2 sl, uint4 tail) {
    Resolved r;
    r.idx = s * 32u + lane;
    r.valid = r.idx < total; // also false for s >= n_slabs
    uint32_t cur = sl.x, m = sl.y + lane;
    if (r.valid) {
      while (m >= tail.w) { // the slab runs past this mesh instance (instances with no meshlets are stepped over)
        m -= tail.w;
        cur++;
        tail = __ldg(reinterpret_cast<const uint4*>(&p.inst[cur].bounds_lo));
      }
    }
    const uint4* bptr = reinterpret_cast<const uint4*>(((uint64_t)tail.y << 32) | tail.x) + m;
    r.inst = cur;
    r.vi = tail.z + m; // :45-49
    r.maskw = 0xFFFFFFFFu; // :44 (no occlusion flag: treated as previously visible)
    if (OCC && r.valid) r.maskw = __ldg(&p.mask[r.vi >> 5]); // plain load: only this launch's owner lane changes the bit
    r.bounds = make_uint4(0, 0, 0, 0);
    if (r.valid) { // the 272-byte InstCull record of the lane's mesh instance -> L1, one slab ahead of its first use: without this
                   // stage A paid 4-5 serialised L2 round trips (flag, planes, normal matrix, rows — each behind a branch)
      const char* rec = reinterpret_cast<const char*>(p.inst + cur);
      prefetch_l1(rec); prefetch_l1(rec + 128); prefetch_l1(rec + 256);
    }
    if (OCC && !LATE) { // early pass: the bounds are fetched by stage A for the was_visible items only; keep the address
      r.bounds.x = (uint32_t)(uint64_t)bptr; r.bounds.y = (uint32_t)((uint64_t)bptr >> 32);
      if (r.valid) prefetch_l1(bptr);
    } else if (r.valid) {
      // every item of the pass needs its bounds: one 128-bit load per lane, issued a slab ahead (when the slab lies in one mesh
      // instance, the warp's 32 consecutive 16-byte records are four full 128-byte lines in one instruction)
      r.bounds = __ldg(bptr);
    }
    return r;
  }

  OXC_DI void consume(const Resolved& r) {
    const bool was = ((r.maskw >> (r.vi & 31)) & 1u) != 0;
    const bool need = r.valid && (LATE || was); // :57
    if (OCC && !LATE) {
      // early pass: items that were not visible need no test at all (visible = was_visible && ..., mask unchanged, nothing
      // emitted) — the rest is compacted so stage A runs on full warps
      const uint32_t bal = __ballot_sync(0xffffffffu, need);
      if (bal) {
        if (need) {
          const uint32_t j = n0 + __popc(bal & lane_lt);
          sh.q0a[warp][j] = make_uint4(r.bounds.x, r.bounds.y, r.inst, r.idx);
          sh.q0b[warp][j] = r.vi;
        }
        n0 += __popc(bal);
        if (n0 >= 32) stage_a_from_q0(32);
      }
    } else {
      stage_a(need, r.bounds, r.inst, r.idx, r.vi, was);
    }
  }

  OXC_DI void run(uint32_t first_slab, uint32_t stride, uint32_t total) {
    const uint32_t n_slabs = (total + 31u) >> 5;
    if (first_slab >= n_slabs) return;
    // prologue: fill the pipeline
    uint2 sl1 = load_slab_entry(first_slab, n_slabs);
    uint2 sl2 = load_slab_entry(first_slab + stride, n_slabs);
    uint2 sl3 = load_slab_entry(first_slab + 2 * stride, n_slabs);
    uint4 tail1 = load_tail(first_slab, n_slabs, sl1);
    uint4 tail2 = load_tail(first_slab + stride, n_slabs, sl2);
    Resolved r0 = resolve(first_slab, total, sl1, tail1);
    for (uint32_t s = first_slab; s < n_slabs; s += stride) {
      // issue the loads of the slabs ahead ...
      const uint2 sl4 = load_slab_entry(s + 3 * stride, n_slabs);
      const uint4 tail3 = load_tail(s + 2 * stride, n_slabs, sl3);
      const Resolved r1 = resolve(s + stride, total, sl2, tail2);
      // ... and test this one while they are in flight
      consume(r0);
      r0 = r1; sl2 = sl3; sl3 = sl4; tail2 = tail3;
    }
  }

  OXC_DI void drain() {
    if (OCC && !LATE) { if (n0) stage_a_from_q0(n0); }
    if (HIZ) {
      if (n1) stage_b(n1);
      if (n2) stage_c(n2);
    }
    if (ne) flush();
  }
};

// launch bounds: OXC_CULL_MIN_BLOCKS = 3 CTAs / SM for every variant.  At 4 (64 registers) the sm_90a build of the late pass
// spills; at 3 (80 registers) it does not, and its time on H100 SXM stays within run-to-run spread (BASELINE.md 5.2)
template <bool HIZ, bool OCC, bool LATE, bool ZERO>
__global__ void __launch_bounds__(CULL_THREADS, OXC_CULL_MIN_BLOCKS) k_cull_meshlets(const __grid_constant__ CullParams p) {
  extern __shared__ __align__(16) unsigned char cull_smem_raw[];
  using Shared = CullShared<OCC && !LATE>;
  Shared& sh = *reinterpret_cast<Shared*>(cull_smem_raw);
  if (threadIdx.x < OXC_HIZ_MAX_LEVELS) sh.hiz_off[threadIdx.x] = p.hiz.level_offset[threadIdx.x];
  sh.s8_lut[threadIdx.x] = s8_over_127((int)threadIdx.x - 128);
  __syncthreads();
  const uint32_t total = p.vis->total_visible_meshlet_instances; // :26
  const uint32_t early_count = LATE ? p.vis->early_visible_meshlet_instances : 0u; // :73 (final: the early kernel has completed)
  const uint32_t id_base = p.id_base ? __ldg(p.id_base) : 0u;
  CullWarp<HIZ, OCC, LATE, ZERO> w(p, sh, early_count, id_base);
  w.run(blockIdx.x * CULL_WARPS + (threadIdx.x >> 5), gridDim.x * CULL_WARPS, total);
  w.drain();
}

// ------------------------------------------------------------------------------------------------
// Multi-view batched cull (reference analogue: cull_meshlets_hpb.slang:27-99 loops <=10 clipmaps per
// meshlet).  Bounds are read ONCE per meshlet instance; per view: cone (directional, :53-54, or
// positional) AND frustum against that view's planes.  Output bit v of view_bits[i], per-view counts.
// ------------------------------------------------------------------------------------------------
struct MultiViewParams {
  const OxcMeshletInstance* meshlet_instances;
  const InstCull* inst;             // view-independent terms (normal matrix, world rows, bounds ptr)
  const InstPlanes* view_planes;    // [n_views][I]
  const OxcMeshletInstanceVisibility* vis;
  uint32_t* view_bits;
  uint32_t* view_counts;
  uint32_t n_views, inst_stride;
  int directional;
  float view_pos[OXC_MAX_VIEWS][4]; // camera.position per view (light direction when directional)
};

__global__ void __launch_bounds__(CULL_THREADS) k_cull_meshlets_multiview(const __grid_constant__ MultiViewParams p) {
  __shared__ uint32_t cnt_s[OXC_MAX_VIEWS];
  if (threadIdx.x < OXC_MAX_VIEWS) cnt_s[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t total = p.vis->total_visible_meshlet_instances;
  const uint2* mi2 = reinterpret_cast<const uint2*>(p.meshlet_instances);
  uint32_t local_cnt[OXC_MAX_VIEWS];
#pragma unroll
  for (int v = 0; v < OXC_MAX_VIEWS; v++) local_cnt[v] = 0;
  for (uint32_t i = blockIdx.x * CULL_THREADS + threadIdx.x; i < total; i += gridDim.x * CULL_THREADS) {
    const uint2 mi = __ldg(&mi2[i]);
    const InstCull* ic = p.inst + mi.x;
    const uint4 tail = __ldg(reinterpret_cast<const uint4*>(&ic->bounds_lo));
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(((uint64_t)tail.y << 32) | tail.x) + mi.y);
    const float cx = dequantize_half(b.x & 0xFFFFu), cy = dequantize_half(b.x >> 16), cz = dequantize_half(b.y & 0xFFFFu);
    const int axq = (int)(int8_t)((b.y >> 16) & 0xFF), ayq = (int)(int8_t)(b.y >> 24);
    const float ex = dequantize_half(b.z & 0xFFFFu), ey = dequantize_half(b.z >> 16), ez = dequantize_half(b.w & 0xFFFFu);
    const int azq = (int)(int8_t)((b.w >> 16) & 0xFF), cutq = (int)(int8_t)(b.w >> 24);
    const float cutoff = s8_over_127(cutq);
    const float ax = s8_over_127(axq), ay = s8_over_127(ayq), az = s8_over_127(azq);
    float wax = 0.f, way = 0.f, waz = 0.f;
    if (p.directional && cutoff < 1.0f) world_cone_axis(ic, ax, ay, az, wax, way, waz);
    uint32_t bits = 0;
    for (uint32_t v = 0; v < p.n_views; v++) {
      bool vis = true;
      if (cutoff < 1.0f) {
        if (p.directional) vis = !(dot3(wax, way, waz, p.view_pos[v][0], p.view_pos[v][1], p.view_pos[v][2]) >= cutoff);
        else vis = cone_visible_positional(ic, cx, cy, cz, ex, ey, ez, ax, ay, az, cutoff, p.view_pos[v][0],
                                           p.view_pos[v][1], p.view_pos[v][2]);
      }
      if (vis) vis = test_frustum_planes(p.view_planes[(size_t)v * p.inst_stride + mi.x].plane, cx, cy, cz, ex, ey, ez);
      if (vis) bits |= 1u << v;
    }
    p.view_bits[i] = bits;
#pragma unroll
    for (int v = 0; v < OXC_MAX_VIEWS; v++) local_cnt[v] += (bits >> v) & 1u;
  }
#pragma unroll
  for (int v = 0; v < OXC_MAX_VIEWS; v++) {
    uint32_t c = local_cnt[v];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&cnt_s[v], c);
  }
  __syncthreads();
  if (threadIdx.x < OXC_MAX_VIEWS && cnt_s[threadIdx.x]) atomicAdd(&p.view_counts[threadIdx.x], cnt_s[threadIdx.x]);
}

// ------------------------------------------------------------------------------------------------
// Shadow-clipmap cull — passes/cull_meshlets_hpb.slang:27-99 + cull.slang:137-166 (canonical arithmetic)
// ------------------------------------------------------------------------------------------------
struct HpbParams {
  const OxcMeshletInstance* meshlet_instances;
  const InstCull* inst;          // built for the coarse view `camera`
  const InstView* views;         // [clipmap][inst_stride]
  const OxcMeshletInstanceVisibility* vis;
  uint32_t* visible_indices;
  OxcDispatchIndirectCommand* tri_cmd;
  const uint32_t* id_base;
  const uint8_t* hpb;
  uint32_t hpb_size, hpb_levels, clipmap_count, inst_stride;
  uint32_t dirty_mask;           // bit c: clipmap_dirty_flags[c] != 0
  const uint32_t* dirty_dev;     // k_cull_meshlets_hpb<true>: the flags in device memory instead (CullGeometry.cpp:214-259)
  float view_dir[3];             // camera.position (= -light_dir)
  float z_near[OXC_MAX_VIEWS];
  int page_offset[OXC_MAX_VIEWS][2];
};

// max(0, ceil(log2(x))) evaluated on the bits of the float: exact, no libm
OXC_DI uint32_t ceil_log2_f32(float x) {
  if (!(x > 1.0f)) return 0u;
  const uint32_t b = __float_as_uint(x);
  if ((b >> 23) == 255u) return 255u;
  return (uint32_t)((int)(b >> 23) - 127 + ((b & 0x7FFFFFu) ? 1 : 0));
}

OXC_DI bool hpb_tap(const HpbParams& p, uint32_t layer, uint32_t level, float u, float v) {
  size_t off = 0;
  for (uint32_t l = 0; l < level; l++) { uint32_t sl = p.hpb_size >> l; sl = sl < 1 ? 1 : sl; off += (size_t)p.clipmap_count * sl * sl; }
  uint32_t sz = p.hpb_size >> level;
  sz = sz < 1 ? 1 : sz;
  int x = __float2int_rz(floorf(fm(u, (float)sz))), y = __float2int_rz(floorf(fm(v, (float)sz)));
  x = min(max(x, 0), (int)sz - 1);
  y = min(max(y, 0), (int)sz - 1);
  return __ldg(p.hpb + off + ((size_t)layer * sz + (size_t)y) * sz + (size_t)x) != 0;
}

OXC_DI bool test_vsm_page(const HpbParams& p, const ScreenAabb& a, uint32_t layer) {
  const float hs = (float)p.hpb_size;
  const float pox = fd((float)p.page_offset[layer][0], hs), poy = fd((float)p.page_offset[layer][1], hs);
  const float box_w = fm(fs(a.maxx, a.minx), hs), box_h = fm(fs(a.maxy, a.miny), hs);
  uint32_t mip = ceil_log2_f32(omax(box_w, box_h));
  mip = mip > p.hpb_levels - 1 ? p.hpb_levels - 1 : mip;
#define OXC_FRACT(x) fs((x), floorf(x))
  const float u0 = fa(a.minx, pox), u1 = fa(a.maxx, pox), v0 = fa(a.miny, poy), v1 = fa(a.maxy, poy);
  const bool tl = hpb_tap(p, layer, mip, OXC_FRACT(u0), OXC_FRACT(v0));
  const bool tr = hpb_tap(p, layer, mip, OXC_FRACT(u1), OXC_FRACT(v0));
  const bool bl = hpb_tap(p, layer, mip, OXC_FRACT(u0), OXC_FRACT(v1));
  const bool br = hpb_tap(p, layer, mip, OXC_FRACT(u1), OXC_FRACT(v1));
#undef OXC_FRACT
  return tl | tr | bl | br;
}

template <bool DEV_FLAGS>
__global__ void __launch_bounds__(CULL_THREADS) k_cull_meshlets_hpb(const __grid_constant__ HpbParams p) {
  __shared__ uint32_t warp_cnt[CULL_THREADS / 32];
  __shared__ uint32_t base_s;
  uint32_t dirty_mask = p.dirty_mask;
  if (DEV_FLAGS) {
    dirty_mask = 0u;
    for (uint32_t ci = 0; ci < p.clipmap_count; ci++) dirty_mask |= (__ldg(&p.dirty_dev[ci]) != 0u ? 1u : 0u) << ci;
  }
  const uint32_t total = p.vis->total_visible_meshlet_instances;
  const uint32_t id_base = p.id_base ? __ldg(p.id_base) : 0u;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint2* mi2 = reinterpret_cast<const uint2*>(p.meshlet_instances);
  const uint32_t n_tiles = (total + CULL_THREADS - 1) / CULL_THREADS;
  for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const uint32_t i = tile * CULL_THREADS + threadIdx.x;
    bool visible = false;
    if (i < total) {
      const uint2 mi = __ldg(&mi2[i]);
      const InstCull* ic = p.inst + mi.x;
      const uint4 tail = __ldg(reinterpret_cast<const uint4*>(&ic->bounds_lo));
      const uint4 b = __ldg(reinterpret_cast<const uint4*>(((uint64_t)tail.y << 32) | tail.x) + mi.y);
      const float cx = dequantize_half(b.x & 0xFFFFu), cy = dequantize_half(b.x >> 16), cz = dequantize_half(b.y & 0xFFFFu);
      const float ex = dequantize_half(b.z & 0xFFFFu), ey = dequantize_half(b.z >> 16), ez = dequantize_half(b.w & 0xFFFFu);
      const float cutoff = s8_over_127((int)(int8_t)(b.w >> 24));
      bool cone_vis = true; // :53-54
      if (cutoff < 1.0f) {
        float wax, way, waz;
        world_cone_axis(ic, s8_over_127((int)(int8_t)((b.y >> 16) & 0xFF)), s8_over_127((int)(int8_t)(b.y >> 24)),
                        s8_over_127((int)(int8_t)((b.w >> 16) & 0xFF)), wax, way, waz);
        cone_vis = !(dot3(wax, way, waz, p.view_dir[0], p.view_dir[1], p.view_dir[2]) >= cutoff);
      }
      if (cone_vis && test_frustum_planes(ic->plane, cx, cy, cz, ex, ey, ez)) { // :56
        for (uint32_t ci = 0; ci < p.clipmap_count; ci++) { // :59-79
          if (!((dirty_mask >> ci) & 1u)) continue;
          const InstView* v = p.views + (size_t)ci * p.inst_stride + mi.x;
          if (!test_frustum_planes(v->plane, cx, cy, cz, ex, ey, ez)) continue;
          ScreenAabb sa;
          if (project_aabb(__ldg(&v->row[0]), __ldg(&v->row[1]), __ldg(&v->row[2]), __ldg(&v->row[3]), p.z_near[ci], cx, cy, cz, ex, ey, ez, sa))
            visible = test_vsm_page(p, sa, ci);
          else visible = true;
          if (visible) break;
        }
      }
    }
    const uint32_t bal = __ballot_sync(0xffffffffu, visible);
    if (lane == 0) warp_cnt[warp] = __popc(bal);
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t s = 0;
#pragma unroll
      for (int w = 0; w < CULL_THREADS / 32; w++) { const uint32_t c = warp_cnt[w]; warp_cnt[w] = s; s += c; }
      base_s = s ? atomicAdd(&p.tri_cmd->x, s) : 0u; // :91
    }
    __syncthreads();
    if (visible) p.visible_indices[base_s + warp_cnt[warp] + __popc(bal & ((1u << lane) - 1u))] = i + id_base; // :96
    __syncthreads();
  }
}

// projection_view of every view, passed BY VALUE as a kernel parameter (1 KB): no host->device copy of a caller / stack
// array is recorded, so the entry points are safe under stream capture
struct ViewMatrices {
  float m[OXC_MAX_VIEWS][16];
};

__global__ void k_prepare_inst_views(const OxcMeshInstance* __restrict__ mesh_instances, const OxcTransformWorld* __restrict__ transforms,
                                     const __grid_constant__ ViewMatrices view_pv, uint32_t n_views, uint32_t first,
                                     uint32_t count, uint32_t inst_stride, InstView* out) {
  const uint32_t local = blockIdx.x * blockDim.x + threadIdx.x;
  if (local >= count) return;
  const uint32_t mi = first + local;
  const float* world = transforms[mesh_instances[mi].transform_index].world;
  float w[16];
#pragma unroll
  for (int k = 0; k < 16; k++) w[k] = world[k];
  for (uint32_t v = 0; v < n_views; v++) {
    float pv[16];
#pragma unroll
    for (int k = 0; k < 16; k++) pv[k] = view_pv.m[v][k];
    float4 rows[4], planes[6];
    mul_mm_rows(pv, w, rows);
    frustum_planes(rows, planes);
    InstView iv;
#pragma unroll
    for (int k = 0; k < 6; k++) iv.plane[k] = planes[k];
#pragma unroll
    for (int k = 0; k < 4; k++) iv.row[k] = rows[k];
    out[(size_t)v * inst_stride + mi] = iv;
  }
}

// ------------------------------------------------------------------------------------------------
// Terrain patch cull — passes/terrain_cull.slang:19-83 (canonical arithmetic throughout: patch counts are small)
// ------------------------------------------------------------------------------------------------
struct TerrainParams {
  OxcTerrainData terrain;
  const float2* patch_minmax;
  uint32_t* visible_patches;
  uint32_t* mask;
  OxcDrawIndirectCommand* draw_cmd;
  HizDesc hiz;
  OxcCullCamera cam;
  uint32_t flags;
};

__global__ void __launch_bounds__(256) k_cull_terrain(const __grid_constant__ TerrainParams p) {
  __shared__ uint32_t hiz_off[OXC_HIZ_MAX_LEVELS];
  __shared__ float4 planes_s[6];
  __shared__ float4 rows_s[4];
  __shared__ uint32_t warp_cnt[8];
  __shared__ uint32_t base_s;
  if (threadIdx.x < OXC_HIZ_MAX_LEVELS) hiz_off[threadIdx.x] = p.hiz.level_offset[threadIdx.x];
  if (threadIdx.x == 0) { // planes of projection_view itself (terrain_cull.slang:50 passes camera.projection_view as mvp)
    float4 rows[4], planes[6];
    const float* m = p.cam.projection_view;
    for (int i = 0; i < 4; i++) rows[i] = make_float4(m[0 * 4 + i], m[1 * 4 + i], m[2 * 4 + i], m[3 * 4 + i]);
    frustum_planes(rows, planes);
    for (int i = 0; i < 6; i++) planes_s[i] = planes[i];
    for (int i = 0; i < 4; i++) rows_s[i] = rows[i];
  }
  __syncthreads();
  const OxcTerrainData& t = p.terrain;
  const uint32_t patch_total = t.patch_count[0] * t.patch_count[1];
  const uint32_t patch_index = blockIdx.x * 256 + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  bool emit = false;
  if (patch_index < patch_total) {
    const uint32_t px = patch_index % t.patch_count[0], py = patch_index / t.patch_count[0];
    const float pcx = (float)t.patch_count[0], pcy = (float)t.patch_count[1];
    const float cminx = fa(t.world_min[0], fm(fd((float)px, pcx), t.world_size[0]));
    const float cminy = fa(t.world_min[1], fm(fd((float)py, pcy), t.world_size[1]));
    const float cmaxx = fa(t.world_min[0], fm(fd((float)(px + 1), pcx), t.world_size[0]));
    const float cmaxy = fa(t.world_min[1], fm(fd((float)(py + 1), pcy), t.world_size[1]));
    const float2 b = __ldg(&p.patch_minmax[patch_index]);
    const float cx = fm(fa(cminx, cmaxx), 0.5f);
    const float cy = fa(t.base_height, fm(fm(fa(b.x, b.y), 0.5f), t.height_scale));
    const float cz = fm(fa(cminy, cmaxy), 0.5f);
    const float ex = fs(cmaxx, cminx), ey = omax(fm(t.height_scale, fs(b.y, b.x)), 1e-3f), ez = fs(cmaxy, cminy);
    const uint32_t word = patch_index >> 5, bit = 1u << (patch_index & 31);
    const bool was_visible = (p.mask[word] & bit) != 0u;
    bool visible = (p.flags & OXC_CULL_LATE_PASS) ? true : was_visible;
    if (p.flags & OXC_CULL_TEST_FRUSTUM) {
      float4 pl[6];
#pragma unroll
      for (int i = 0; i < 6; i++) pl[i] = planes_s[i];
      visible = visible && test_frustum_rows(pl, cx, cy, cz, ex, ey, ez);
    }
    if ((p.flags & (OXC_CULL_TEST_OCCLUSION | OXC_CULL_LATE_PASS)) != 0 && visible) {
      ScreenAabb sa;
      if (project_aabb(rows_s[0], rows_s[1], rows_s[2], rows_s[3], p.cam.near_clip, cx, cy, cz, ex, ey, ez, sa))
        visible = !test_occlusion(sa, p.hiz.data, p.hiz.width, p.hiz.height, p.hiz.levels, hiz_off);
    }
    emit = visible && (!(p.flags & OXC_CULL_LATE_PASS) || !was_visible);
    if ((p.flags & (OXC_CULL_TEST_OCCLUSION | OXC_CULL_LATE_PASS)) && visible != was_visible) atomicXor(&p.mask[word], bit);
  }
  const uint32_t bal = __ballot_sync(0xffffffffu, emit);
  if (lane == 0) warp_cnt[warp] = __popc(bal);
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t s = 0;
    for (int w = 0; w < 8; w++) { const uint32_t c = warp_cnt[w]; warp_cnt[w] = s; s += c; }
    base_s = s ? atomicAdd(&p.draw_cmd->instance_count, s) : 0u; // :76
  }
  __syncthreads();
  if (emit) p.visible_patches[base_s + warp_cnt[warp] + __popc(bal & ((1u << lane) - 1u))] = patch_index; // :81
}

__global__ void k_reset_terrain_cmd(OxcDrawIndirectCommand* c) { c->vertex_count = 4; c->instance_count = 0; c->first_vertex = 0; c->first_instance = 0; }

// per view planes for the multi-view cull: planes of mul(view.projection_view, world)
__global__ void k_prepare_view_planes(const OxcMeshInstance* __restrict__ mesh_instances,
                                      const OxcTransformWorld* __restrict__ transforms, const __grid_constant__ ViewMatrices views,
                                      uint32_t n_views, uint32_t first, uint32_t count, uint32_t inst_stride,
                                      InstPlanes* out) {
  const uint32_t local = blockIdx.x * blockDim.x + threadIdx.x;
  if (local >= count) return;
  const uint32_t mi = first + local;
  const float* world = transforms[mesh_instances[mi].transform_index].world;
  float w[16];
#pragma unroll
  for (int k = 0; k < 16; k++) w[k] = world[k];
  for (uint32_t v = 0; v < n_views; v++) {
    float pv[16];
#pragma unroll
    for (int k = 0; k < 16; k++) pv[k] = views.m[v][k];
    float4 rows[4], planes[6];
    mul_mm_rows(pv, w, rows);
    frustum_planes(rows, planes);
    InstPlanes ip;
#pragma unroll
    for (int k = 0; k < 6; k++) ip.plane[k] = planes[k];
    out[(size_t)v * inst_stride + mi] = ip;
  }
}

} // namespace oxc
