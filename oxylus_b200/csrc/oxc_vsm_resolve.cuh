// oxc_vsm_resolve.cuh — the VSM shadow resolve of one pixel (passes/resolve_shadowmaps.slang:27-209 with the rmvsm.slang helpers
// it calls) as pure per-thread functions: unproject, clipmap selection, normal offset, PCSS (1 centre tap, 16 blocker-search taps,
// up to 24 PCF taps), each tap a page-table lookup plus an atlas fetch with the clipmap -1 / +1 fall-back.
// No warp intrinsics, no shared memory: tests compile this source for the host.
// Specification: include/oxcull.h (comment above oxc_vsm_resolve_shadows) == oracle/oxc_oracle_vsm_resolve.c, operation for operation.
#pragma once
#include "oxc_shader_math.cuh"

namespace oxc {

// com::hammersley2d (common/math.slang:189-191): (i / N, reversebits(i) * 2^-32); host precomputation of the kernel's constants
__host__ __device__ inline void vsm_hammersley(uint32_t i, uint32_t n, float& a, float& b) {
  uint32_t v = 0;
  for (int k = 0; k < 32; k++) v |= ((i >> k) & 1u) << (31 - k);
  a = (float)i / (float)n;
  b = (float)v * 2.3283064365386963e-10f;
}

constexpr int VSM_RESOLVE_BLOCKER_SAMPLES = 16, VSM_RESOLVE_PCF_SAMPLES = 24; // resolve_shadowmaps.slang:19-20

struct VsmResolveParams {
  float4 inv_pv_row[4];        // rows of Camera::inv_projection_view
  float inv_res_half[2];       // (1 / resolution) * 0.5
  float clipmap_row[10][4][4]; // rows of every clipmap's projection_view_mat
  int page_offset[10][2];
  int ortho[10];               // row 3 is exactly (0, 0, 0, 1)
  float ham[VSM_RESOLVE_BLOCKER_SAMPLES + VSM_RESOLVE_PCF_SAMPLES][2]; // hammersley2d(i, 16), then hammersley2d(i, 24)
  float light[3];              // VSMContext::directional_light_dir
  const float* depth;
  const float4* normals;       // oct(world normal) in .zw
  const uint32_t* page_tables;
  const float* atlas;
  float* shadow;
  int width, height, size, clipmap_count, page_size, atlas_size, phys_per_row;
  float texel_length, bias, z_length;
};

// rmvsm.slang:147-154 get_first_clipmap_texel_length with the oracle's operation order (host floats: IEEE, no contraction)
__host__ inline float vsm_first_texel_length(const OxcVsmContext& vsm) {
  volatile float scale_ratio = (float)(vsm.page_table_size - 1) / (float)vsm.page_table_size;
  volatile float effective_width = vsm.first_clipmap_width * scale_ratio;
  volatile float twice = effective_width * 2.0f;
  return twice / vsm.virtual_extent;
}

// the camera and clipmap fields the page marking (VsmMarkParams) and the resolve (VsmResolveParams) share, from the C ABI's arguments
template <class P>
__host__ inline void vsm_fill_view(P& p, const float inv_pv[16], const float resolution[2], const OxcVirtualClipmap* clipmaps,
                                   const OxcVsmContext& vsm) {
  for (int i = 0; i < 4; i++) p.inv_pv_row[i] = make_float4(inv_pv[i], inv_pv[4 + i], inv_pv[8 + i], inv_pv[12 + i]);
  // (1.0 / resolution) * 0.5 with the oracle's operation order (host floats: IEEE, no contraction)
  p.inv_res_half[0] = (1.0f / resolution[0]) * 0.5f; p.inv_res_half[1] = (1.0f / resolution[1]) * 0.5f;
  for (int k = 0; k < vsm.clipmap_count; k++) {
    for (int i = 0; i < 4; i++)
      for (int j = 0; j < 4; j++) p.clipmap_row[k][i][j] = clipmaps[k].projection_view_mat[j * 4 + i];
    p.page_offset[k][0] = clipmaps[k].page_offset[0]; p.page_offset[k][1] = clipmaps[k].page_offset[1];
  }
  p.texel_length = vsm_first_texel_length(vsm);
  p.bias = vsm.clipmap_selection_bias;
}

// the kernel's parameters from the C ABI's arguments (oxc_vsm_resolve_shadows, and the host build of the tests)
__host__ inline VsmResolveParams vsm_resolve_make_params(const OxcVsmContext& vsm, const float inv_pv[16], const float resolution[2],
                                                         const OxcVirtualClipmap* clipmaps, const float* depth, const float* normals,
                                                         const uint32_t* page_tables, const float* atlas, float* shadow) {
  VsmResolveParams p{};
  vsm_fill_view(p, inv_pv, resolution, clipmaps, vsm);
  for (int k = 0; k < vsm.clipmap_count; k++) {
    const float* m = clipmaps[k].projection_view_mat;
    p.ortho[k] = m[3] == 0.0f && m[7] == 0.0f && m[11] == 0.0f && m[15] == 1.0f;
  }
  for (int i = 0; i < VSM_RESOLVE_BLOCKER_SAMPLES; i++) vsm_hammersley((uint32_t)i, VSM_RESOLVE_BLOCKER_SAMPLES, p.ham[i][0], p.ham[i][1]);
  for (int i = 0; i < VSM_RESOLVE_PCF_SAMPLES; i++)
    vsm_hammersley((uint32_t)i, VSM_RESOLVE_PCF_SAMPLES, p.ham[VSM_RESOLVE_BLOCKER_SAMPLES + i][0], p.ham[VSM_RESOLVE_BLOCKER_SAMPLES + i][1]);
  for (int i = 0; i < 3; i++) p.light[i] = vsm.directional_light_dir[i];
  p.depth = depth; p.normals = reinterpret_cast<const float4*>(normals); p.page_tables = page_tables; p.atlas = atlas; p.shadow = shadow;
  p.width = vsm.depth_extent[0]; p.height = vsm.depth_extent[1]; p.size = vsm.page_table_size; p.clipmap_count = vsm.clipmap_count;
  p.page_size = vsm.page_size; p.atlas_size = vsm.physical_page_table_size; p.phys_per_row = vsm.physical_page_table_size / vsm.page_size;
  p.z_length = vsm.z_length;
  return p;
}

struct VsmBasis { float tx, ty, tz, bx, by, bz; };

// resolve_shadowmaps.slang:77-82 perpendicular_basis: depends only on L
OXC_DI VsmBasis vsm_perpendicular_basis(float lx, float ly, float lz) {
  const bool y_axis = fabsf(ly) < 0.999f;
  const float ax = y_axis ? 0.0f : 1.0f, ay = y_axis ? 1.0f : 0.0f, az = 0.0f;
  const float cx = fs(fm(ay, lz), fm(az, ly)), cy = fs(fm(az, lx), fm(ax, lz)), cz = fs(fm(ax, ly), fm(ay, lx)); // cross(axis, L)
  const float len = fsq(dot3(cx, cy, cz, cx, cy, cz));
  VsmBasis b;
  b.tx = fd(cx, len); b.ty = fd(cy, len); b.tz = fd(cz, len);
  b.bx = fs(fm(ly, b.tz), fm(lz, b.ty)); b.by = fs(fm(lz, b.tx), fm(lx, b.tz)); b.bz = fs(fm(lx, b.ty), fm(ly, b.tx)); // cross(L, t)
  return b;
}

// scene.slang:189-193 unproject_uv with the rows of inv_projection_view.  P: the kernel parameters (VsmMarkParams of the page
// marking, VsmResolveParams here), read for inv_pv_row, inv_res_half, texel_length, bias and clipmap_count.
template <class P>
OXC_DI void vsm_unproject(const P& p, float u, float v, float depth, float& x, float& y, float& z) {
  const float nx = fs(fm(u, 2.0f), 1.0f), ny = fs(fm(v, 2.0f), 1.0f);
  const float hx = row_dot4(p.inv_pv_row[0], nx, ny, depth, 1.0f), hy = row_dot4(p.inv_pv_row[1], nx, ny, depth, 1.0f);
  const float hz = row_dot4(p.inv_pv_row[2], nx, ny, depth, 1.0f), hw = row_dot4(p.inv_pv_row[3], nx, ny, depth, 1.0f);
  x = fd(hx, hw); y = fd(hy, hw); z = fd(hz, hw);
}

// rmvsm.slang:156-188 get_clipmap_index (VMS_USE_DIAG_PIXEL_FOOTPRINT): the world distance between the unprojected left and right
// ends of the pixel, log2 of it over the first clipmap's texel length, bias, ceil, saturating u32, clamped to the last clipmap.
// k_vsm_mark_visible_pages runs the same operations written out inline (called through this function its SASS changes).
template <class P>
OXC_DI uint32_t vsm_select_clipmap(const P& p, float u, float v, float d) {
  float ax, ay, az, bx, by, bz;
  vsm_unproject(p, fs(u, p.inv_res_half[0]), fa(v, p.inv_res_half[1]), d, ax, ay, az);
  vsm_unproject(p, fa(u, p.inv_res_half[0]), fa(v, p.inv_res_half[1]), d, bx, by, bz);
  const float dx = fs(ax, bx), dy = fs(ay, by), dz = fs(az, bz);
  const float dist = fsq(fa(fa(fm(dx, dx), fm(dy, dy)), fm(dz, dz)));
  float level_f = canonical_log2(fd(dist, p.texel_length));
  level_f = level_f > 0.0f ? level_f : 0.0f;
  const float lf = ceilf(fa(p.bias, level_f));
  uint32_t ci = lf >= 4294967296.0f ? 0xFFFFFFFFu : (lf > 0.0f ? __float2uint_rz(lf) : 0u);
  ci = ci > (uint32_t)(p.clipmap_count - 1) ? (uint32_t)(p.clipmap_count - 1) : ci;
  return ci;
}

// rmvsm.slang:200-206 get_virt_coords + :129-138 page_coords_virtual_to_wrapped (com::mod on floats): false = no page
OXC_DI bool vsm_wrapped_page(float cu, float cv, int size, int off_x, int off_y, int& wx, int& wy) {
  if (cu < 0.0f || cv < 0.0f || cu > 1.0f || cv > 1.0f) return false;
  const float fsz = (float)size;
  const int vx = sat_i32(floorf(fm(cu, fsz))), vy = sat_i32(floorf(fm(cv, fsz)));
  if (vx < 0 || vy < 0 || vx > size - 1 || vy > size - 1) return false;
  const float fox = (float)(vx + off_x), foy = (float)(vy + off_y);
  wx = (int)fs(fox, fm(fsz, floorf(fd(fox, fsz))));
  wy = (int)fs(foy, fm(fsz, floorf(fd(foy, fsz))));
  return !(wx < 0 || wy < 0 || wx > size - 1 || wy > size - 1);
}

// rmvsm.slang:214-221 get_clipmap_info: clip uv and projected depth.  A clipmap whose row 3 is exactly (0, 0, 0, 1) has w = 1
// exactly for a finite point, so the three divides are identities and are skipped.
OXC_DI void vsm_clipmap_info(const VsmResolveParams& p, int ci, float x, float y, float z, float& cu, float& cv, float& pd) {
  const float(*cr)[4] = p.clipmap_row[ci];
  const float lx = fa(fa(fa(fm(cr[0][0], x), fm(cr[0][1], y)), fm(cr[0][2], z)), fm(cr[0][3], 1.0f));
  const float ly = fa(fa(fa(fm(cr[1][0], x), fm(cr[1][1], y)), fm(cr[1][2], z)), fm(cr[1][3], 1.0f));
  const float lz = fa(fa(fa(fm(cr[2][0], x), fm(cr[2][1], y)), fm(cr[2][2], z)), fm(cr[2][3], 1.0f));
  if (p.ortho[ci] && fabsf(x) <= 3.40282347e38f && fabsf(y) <= 3.40282347e38f && fabsf(z) <= 3.40282347e38f) {
    cu = fm(fa(lx, 1.0f), 0.5f); cv = fm(fa(ly, 1.0f), 0.5f); pd = lz;
    return;
  }
  const float lw = fa(fa(fa(fm(cr[3][0], x), fm(cr[3][1], y)), fm(cr[3][2], z)), fm(cr[3][3], 1.0f));
  cu = fm(fa(fd(lx, lw), 1.0f), 0.5f); cv = fm(fa(fd(ly, lw), 1.0f), 0.5f); pd = fd(lz, lw);
}

constexpr float VSM_DEPTH_MISS = -1.0f; // resolve_shadowmaps.slang:25

// resolve_shadowmaps.slang:32-61 sample_vsm_shadow_depth.  A texel outside the atlas reads 0 (robustImageAccess).
OXC_DI float vsm_sample_depth(const VsmResolveParams& p, int ci, float x, float y, float z) {
  if (ci < 0 || ci >= p.clipmap_count) return VSM_DEPTH_MISS;
  float cu, cv, pd;
  vsm_clipmap_info(p, ci, x, y, z, cu, cv, pd);
  int wx, wy;
  if (!vsm_wrapped_page(cu, cv, p.size, p.page_offset[ci][0], p.page_offset[ci][1], wx, wy)) return VSM_DEPTH_MISS;
  const uint32_t e = __ldg(&p.page_tables[((size_t)ci * p.size + (size_t)wy) * p.size + (size_t)wx]);
  if (!(e & 4u)) return VSM_DEPTH_MISS; // Backed
  const uint32_t addr = e >> 16, n = (uint32_t)p.phys_per_row;
  const float fP = (float)p.atlas_size, fps = (float)p.page_size;
  const float tx = (float)sat_i32(floorf(fm(cu, fP))), ty = (float)sat_i32(floorf(fm(cv, fP))); // :56
  const int ix = (int)fs(tx, fm(fps, floorf(fd(tx, fps)))), iy = (int)fs(ty, fm(fps, floorf(fd(ty, fps)))); // :57 com::mod
  const long long ax = (long long)(addr % n) * p.page_size + ix, ay = (long long)(addr / n) * p.page_size + iy; // :55, 58
  if (ax < 0 || ay < 0 || ax >= p.atlas_size || ay >= p.atlas_size) return 0.0f;
  return __ldg(&p.atlas[(size_t)ay * p.atlas_size + (size_t)ax]);
}

// :63-75 sample_vsm_shadow_depth_with_fallback
OXC_DI float vsm_sample_fallback(const VsmResolveParams& p, int ci, float x, float y, float z) {
  const float d0 = vsm_sample_depth(p, ci, x, y, z);
  if (d0 != VSM_DEPTH_MISS) return d0;
  const float d1 = vsm_sample_depth(p, ci - 1, x, y, z);
  if (d1 != VSM_DEPTH_MISS) return d1;
  const float d2 = vsm_sample_depth(p, ci + 1, x, y, z);
  if (d2 != VSM_DEPTH_MISS) return d2;
  return VSM_DEPTH_MISS;
}

// :27-30 hash2 of the pixel position (x + 0.5, y + 0.5)
OXC_DI void vsm_hash2(float px, float py, float& n0, float& n1) {
  const float d0 = fa(fm(px, 127.1f), fm(py, 311.7f)), d1 = fa(fm(px, 269.5f), fm(py, 183.3f));
  n0 = frac(fm(canonical_sin(d0), 43758.5453f));
  n1 = frac(fm(canonical_sin(d1), 43758.5453f));
}

// one PCSS tap (:119-127 / :161-169): returns the fall-back depth at the offset point, bias_norm through `bias_norm`
OXC_DI float vsm_tap(const VsmResolveParams& p, const VsmBasis& b, int ci, float ox, float oy, float oz, float hx, float hy, float nx,
                     float ny, float radius, float nol, float base_bias, float inv_z, float& bias_norm) {
  const float xi_x = frac(fa(hx, nx)), xi_y = frac(fa(hy, ny));
  const float r = fm(fsq(xi_x), radius);
  const float theta = fm(xi_y, 6.28318548f); // TAU
  float s, c;
  canonical_sincos(theta, s, c);
  const float dx = fm(r, fa(fm(b.tx, c), fm(b.bx, s))), dy = fm(r, fa(fm(b.ty, c), fm(b.by, s))), dz = fm(r, fa(fm(b.tz, c), fm(b.bz, s)));
  const float pcf_bias = fm(2.0f, r);
  bias_norm = fm(inv_z, fa(base_bias, fa(pcf_bias, fm(fs(0.0f, pcf_bias), nol)))); // lerp(a, b, t) = a + (b - a) * t
  return vsm_sample_fallback(p, ci, fa(ox, dx), fa(oy, dy), fa(oz, dz));
}

// :84-185 pcss_shadow.  *pcf: set when the PCF loop ran.
OXC_DI float vsm_pcss(const VsmResolveParams& p, const VsmBasis& b, int ci, float wx, float wy, float wz, float nx, float ny, float nz,
                      float n0, float n1, bool* pcf) {
  const float lx = p.light[0], ly = p.light[1], lz = p.light[2];
  const float nol = vmax(dot3(nx, ny, nz, lx, ly, lz), 0.0f);
  const float cts = fm((float)(1 << (ci + 1)), p.texel_length);          // pow(2, ci + 1) * first texel length
  const float bb = fm(fm(1.41421356f, cts), 0.5f);
  float term = bb;
  if (nol < 0.99f) {
    const float cx = fs(fm(ny, lz), fm(nz, ly)), cy = fs(fm(nz, lx), fm(nx, lz)), cz = fs(fm(nx, ly), fm(ny, lx));
    term = fd(fm(bb, length3(cx, cy, cz)), vmax(nol, 0.1f));
  }
  const float base_bias = fa(fa(2.38418579e-07f, bb), term);               // quantize = 2 / 2^23
  const float inv_z = fd(1.0f, p.z_length);
  const float now = fm(cts, fa(1.0f, fm(2.0f, fs(1.0f, nol))));
  const float ox = fa(wx, fm(nx, now)), oy = fa(wy, fm(ny, now)), oz = fa(wz, fm(nz, now));
  float cu, cv, d_recv;
  vsm_clipmap_info(p, ci, ox, oy, oz, cu, cv, d_recv);
  const float d_recv_world = fm(d_recv, p.z_length);
  const float center = vsm_sample_fallback(p, ci, ox, oy, oz);
  float accum = 0.0f;
  uint32_t blockers = 0, valid = 0;
  for (int i = 0; i < VSM_RESOLVE_BLOCKER_SAMPLES; i++) {
    float bias_norm;
    const float d = vsm_tap(p, b, ci, ox, oy, oz, p.ham[i][0], p.ham[i][1], n0, n1, 0.1f, nol, base_bias, inv_z, bias_norm);
    if (d == VSM_DEPTH_MISS) continue;
    valid++;
    if (fa(d, bias_norm) < d_recv) { accum = fa(accum, fm(d, p.z_length)); blockers++; }
  }
  const float hard_bias_norm = fm(inv_z, base_bias);
  const float hard = center == VSM_DEPTH_MISS ? 1.0f : (fa(center, hard_bias_norm) < d_recv ? 0.0f : 1.0f);
  if (valid == 0u) return hard;
  if (blockers == 0u) return 1.0f;
  if (blockers == valid) return 0.0f;
  *pcf = true;
  const float d_blocker_world = fd(accum, (float)blockers);
  const float radius = vmin(0.1f, fm(fs(d_recv_world, d_blocker_world), 0.002f));
  float lit = 0.0f;
  uint32_t valid_pcf = 0;
  for (int i = 0; i < VSM_RESOLVE_PCF_SAMPLES; i++) {
    float bias_norm;
    const float* h = p.ham[VSM_RESOLVE_BLOCKER_SAMPLES + i];
    const float d = vsm_tap(p, b, ci, ox, oy, oz, h[0], h[1], n1, n0, radius, nol, base_bias, inv_z, bias_norm); // noise.yx
    if (d == VSM_DEPTH_MISS) continue;
    valid_pcf++;
    if (fa(d, bias_norm) >= d_recv) lit = fa(lit, 1.0f);
  }
  if (valid_pcf == 0u) return hard;
  return fd(lit, (float)valid_pcf);
}

// :187-209 fs_main for pixel (x, y).  *pcf: set when the pixel ran the PCF loop.
OXC_DI float vsm_resolve_pixel(const VsmResolveParams& p, const VsmBasis& b, int x, int y, bool* pcf) {
  const size_t pix = (size_t)y * p.width + x;
  const float d = __ldg(&p.depth[pix]);
  if (d == 0.0f) return 1.0f;
  const float4 nrm = __ldg(&p.normals[pix]);
  // common/encoding.slang:7-15 oct_to_vec3 of the binary16 .ba, then normalize again (:199)
  const float ex = round_to_half(nrm.z), ey = round_to_half(nrm.w);
  float vx = ex, vy = ey;
  const float vz = fs(fs(1.0f, fabsf(ex)), fabsf(ey));
  const float sx = vx >= 0.0f ? 1.0f : -1.0f, sy = vy >= 0.0f ? 1.0f : -1.0f;
  if (vz < 0.0f) { vx = fm(fs(1.0f, fabsf(ey)), sx); vy = fm(fs(1.0f, fabsf(ex)), sy); }
  const float l0 = length3(vx, vy, vz);
  const float ux = fd(vx, l0), uy = fd(vy, l0), uz = fd(vz, l0);
  const float l1 = length3(ux, uy, uz);
  const float nx = fd(ux, l1), ny = fd(uy, l1), nz = fd(uz, l1);
  const float px = fa((float)x, 0.5f), py = fa((float)y, 0.5f);
  const float u = fd(px, (float)p.width), v = fd(py, (float)p.height);
  float wx, wy, wz;
  vsm_unproject(p, u, v, d, wx, wy, wz);
  const int ci = (int)vsm_select_clipmap(p, u, v, d);
  float n0, n1;
  vsm_hash2(px, py, n0, n1);
  return vsm_pcss(p, b, ci, wx, wy, wz, nx, ny, nz, n0, n1, pcf);
}

} // namespace oxc
