/*
 * oxc_oracle_gbuffer.c — CPU ORACLE (test infrastructure) of the vis-buffer decode into the G-buffer: passes/visbuffer_decode.slang:
 * 88-183 with Material::sample_* of scene.slang:110-159.  Same rules as oxc_oracle.c: plain C11, IEEE binary32 with round to nearest,
 * no contraction, IEEE divide / sqrt, dot(a, b) = (a.x*b.x + a.y*b.y) + a.z*b.z, sums in the order written.  One translation unit
 * with oxc_oracle.c, included below, so that it runs the decode's geometry (orc_decode_visbuffer) and the alpha test's sampler
 * helpers (alpha_wrap, alpha_f2i, orc_log2_canonical).  Built into liboxc_oracle_gbuffer.so by oracle/pyoracle_gbuffer.py:
 *   gcc -O2 -std=c11 -ffp-contract=off -fno-fast-math -fPIC -shared oxc_oracle_gbuffer.c -lm
 *
 * SPECIFICATION of orc_decode_gbuffer (include/oxcull.h oxc_decode_gbuffer repeats it):
 *   1. a pixel orc_decode_visbuffer discards (status 0) is not written; status 2 (a vertex index >= vertex_count) and a material_index
 *      outside the table write zeros to every plane.
 *   2. lambda, ddx, ddy, uv and its gradients: orc_decode_visbuffer's planes; the world positions (mul(world, p), p.w = 1) and the
 *      world normal n = normalize(mul(lambda, to_world_normals)) with that function's arithmetic.
 *   3. uv = uv*uv_size + uv_offset, ddx *= uv_size, ddy *= uv_size (:117-122).
 *   4. SampleGrad: mx = ddx.u*w0, my = ddx.v*h0, nx = ddy.u*w0, ny = ddy.v*h0, rho^2 = max(mx*mx + my*my, nx*nx + ny*ny), lambda =
 *      0.5*log2_canonical(rho^2), then the alpha test's level rule (oxc_oracle.c spec step 4) and its per-channel filter order; an
 *      image with one level and equal mag / min filters samples level 0 with that filter.
 *   5. texel -> RGBA before filtering: RGBA8_UNORM c/255; RGBA8_SRGB rgb = sRGB EOTF of c/255 rounded once to binary32, a = c/255;
 *      R8_UNORM (r/255, 0, 0, 1); RG8_UNORM (r/255, g/255, 0, 1).
 *   6-8. albedo, tangent frame and normal map, emissive, metallic / roughness / occlusion as include/oxcull.h states them.
 */
#include "oxc_oracle.c"

#include "oxc_oracle_gbuffer.h"

static float gb_srgb[256];
static int gb_srgb_ready = 0;
static uint64_t gb_fetches = 0; /* texel fetches since the last reset (orc_gbuffer_texel_fetches) */

uint64_t orc_gbuffer_texel_fetches(int reset) {
  const uint64_t n = gb_fetches;
  if (reset) gb_fetches = 0;
  return n;
}

void orc_srgb_table(float out[256]) {
  for (int c = 0; c < 256; c++) {
    const double x = (double)c / 255.0;
    out[c] = (float)(x <= 0.04045 ? x / 12.92 : pow((x + 0.055) / 1.055, 2.4));
  }
}

static uint32_t gb_bytes(uint32_t format) { return format == OXC_IMAGE_R8_UNORM ? 1u : (format == OXC_IMAGE_RG8_UNORM ? 2u : 4u); }

static void gb_texel(uint32_t format, const uint8_t* base, uint32_t w, uint32_t x, uint32_t y, float o[4]) {
  if (!gb_srgb_ready) { orc_srgb_table(gb_srgb); gb_srgb_ready = 1; }
  gb_fetches++;
  const uint8_t* t = base + ((size_t)y * w + x) * gb_bytes(format);
  if (format == OXC_IMAGE_R8_UNORM) { o[0] = (float)t[0] / 255.0f; o[1] = 0.0f; o[2] = 0.0f; o[3] = 1.0f; return; }
  if (format == OXC_IMAGE_RG8_UNORM) { o[0] = (float)t[0] / 255.0f; o[1] = (float)t[1] / 255.0f; o[2] = 0.0f; o[3] = 1.0f; return; }
  if (format == OXC_IMAGE_RGBA8_SRGB) { o[0] = gb_srgb[t[0]]; o[1] = gb_srgb[t[1]]; o[2] = gb_srgb[t[2]]; }
  else { o[0] = (float)t[0] / 255.0f; o[1] = (float)t[1] / 255.0f; o[2] = (float)t[2] / 255.0f; }
  o[3] = (float)t[3] / 255.0f;
}

typedef struct GbSampler { uint32_t mag, min, mip, au, av; } GbSampler;

static GbSampler gb_sampler(const OxcSamplerDesc* s) {
  GbSampler r = {OXC_FILTER_LINEAR, OXC_FILTER_LINEAR, OXC_MIPMAP_LINEAR, OXC_ADDRESS_REPEAT, OXC_ADDRESS_REPEAT}; /* Texture.hpp:38-45 */
  if (s) { r.mag = s->mag_filter; r.min = s->min_filter; r.mip = s->mipmap_mode; r.au = s->address_u; r.av = s->address_v; }
  return r;
}

static void gb_sample_level(const OxcAlphaImage* im, GbSampler s, uint32_t level, uint32_t filter, float u, float v, float out[4]) {
  const uint8_t* base = (const uint8_t*)im->texels_dev;
  uint32_t w = im->width, h = im->height;
  for (uint32_t l = 0; l < level; l++) {
    base += (size_t)w * h * gb_bytes(im->format);
    w = w > 1 ? w >> 1 : 1;
    h = h > 1 ? h >> 1 : 1;
  }
  const float fw = (float)w, fh = (float)h;
  if (filter == OXC_FILTER_NEAREST) {
    const int ix = alpha_f2i(floorf(u * fw)), iy = alpha_f2i(floorf(v * fh));
    gb_texel(im->format, base, w, alpha_wrap(ix, w, s.au), alpha_wrap(iy, h, s.av), out);
    return;
  }
  const float x = u * fw - 0.5f, y = v * fh - 0.5f;
  const float x0 = floorf(x), y0 = floorf(y);
  const float wx = x - x0, wy = y - y0;
  const int ix = alpha_f2i(x0), iy = alpha_f2i(y0);
  const uint32_t xa = alpha_wrap(ix, w, s.au), xb = alpha_wrap((int64_t)ix + 1, w, s.au);
  const uint32_t ya = alpha_wrap(iy, h, s.av), yb = alpha_wrap((int64_t)iy + 1, h, s.av);
  float a00[4], a10[4], a01[4], a11[4];
  gb_texel(im->format, base, w, xa, ya, a00); gb_texel(im->format, base, w, xb, ya, a10);
  gb_texel(im->format, base, w, xa, yb, a01); gb_texel(im->format, base, w, xb, yb, a11);
  for (int c = 0; c < 4; c++) {
    const float top = a00[c] + wx * (a10[c] - a00[c]), bot = a01[c] + wx * (a11[c] - a01[c]);
    out[c] = top + wy * (bot - top);
  }
}

static void gb_sample_grad(const OxcAlphaImage* im, GbSampler s, float u, float v, float dxu, float dxv, float dyu, float dyv, float out[4]) {
  const uint32_t levels = im->level_count ? im->level_count : 1;
  if (levels <= 1 && s.mag == s.min) { gb_sample_level(im, s, 0, s.min, u, v, out); return; }
  const float w0 = (float)im->width, h0 = (float)im->height;
  const float mx = dxu * w0, my = dxv * h0, nx = dyu * w0, ny = dyv * h0;
  const float rx2 = mx * mx + my * my, ry2 = nx * nx + ny * ny;
  const float r2 = rx2 > ry2 ? rx2 : ry2;
  const float lambda = 0.5f * orc_log2_canonical(r2);
  const uint32_t filter = lambda > 0.0f ? s.min : s.mag;
  const float q = (float)(levels - 1);
  const float lc = !(lambda > 0.0f) ? 0.0f : (lambda > q ? q : lambda);
  if (s.mip == OXC_MIPMAP_NEAREST) {
    uint32_t d = lc <= 0.5f ? 0u : (uint32_t)ceilf(lc + 0.5f) - 1u;
    if (d > levels - 1) d = levels - 1;
    gb_sample_level(im, s, d, filter, u, v, out);
    return;
  }
  const uint32_t d = (uint32_t)floorf(lc), dn = d + 1u > levels - 1 ? levels - 1 : d + 1u;
  const float f = lc - (float)d;
  float lo[4], hi[4];
  gb_sample_level(im, s, d, filter, u, v, lo);
  gb_sample_level(im, s, dn, filter, u, v, hi);
  for (int c = 0; c < 4; c++) out[c] = (1.0f - f) * lo[c] + f * hi[c];
}

void orc_gbuffer_sample_level(const OxcAlphaImage* image, const OxcSamplerDesc* sampler, uint32_t level, uint32_t filter, float u, float v,
                              float out[4]) {
  gb_sample_level(image, gb_sampler(sampler), level, filter, u, v, out);
}

void orc_gbuffer_sample_grad(const OxcAlphaImage* image, const OxcSamplerDesc* sampler, float u, float v, float ddx_u, float ddx_v, float ddy_u,
                             float ddy_v, float out[4]) {
  gb_sample_grad(image, gb_sampler(sampler), u, v, ddx_u, ddx_v, ddy_u, ddy_v, out);
}

static float gb_sign(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); } /* HLSL sign, NaN -> 0 */

/* :150-161: T and B from the position derivatives, the world normal and the uv gradients */
static void gb_tangent_frame(const float pdx[3], const float pdy[3], const float n[3], float dxu, float dxv, float dyu, float dyv, float t[3],
                             float b[3]) {
  const float dxn = (pdx[0] * n[0] + pdx[1] * n[1]) + pdx[2] * n[2], dyn = (pdy[0] * n[0] + pdy[1] * n[1]) + pdy[2] * n[2];
  float sx[3], sy[3], cr[3];
  for (int k = 0; k < 3; k++) { sx[k] = pdx[k] - dxn * n[k]; sy[k] = pdy[k] - dyn * n[k]; }
  const float js = gb_sign(dxu * dyv - dxv * dyu);
  for (int k = 0; k < 3; k++) t[k] = js * (dyv * sx[k] - dxv * sy[k]);
  if (js != 0.0f) {
    const float len = sqrtf((t[0] * t[0] + t[1] * t[1]) + t[2] * t[2]);
    for (int k = 0; k < 3; k++) t[k] = t[k] / len;
  }
  cr[0] = n[1] * pdx[2] - n[2] * pdx[1]; cr[1] = n[2] * pdx[0] - n[0] * pdx[2]; cr[2] = n[0] * pdx[1] - n[1] * pdx[0]; /* cross(n, pos_ddx) */
  const float w = js * gb_sign((pdy[0] * cr[0] + pdy[1] * cr[1]) + pdy[2] * cr[2]);
  b[0] = -w * (n[1] * t[2] - n[2] * t[1]); b[1] = -w * (n[2] * t[0] - n[0] * t[2]); b[2] = -w * (n[0] * t[1] - n[1] * t[0]);
}

/* pos_ddx / pos_ddy of a pixel record: camera-relative positions weighted by the lambda derivatives */
static void gb_position_derivatives(const float px[24], const float cam[3], float pdx[3], float pdy[3]) {
  float p[3][3];
  for (int c = 0; c < 3; c++)
    for (int k = 0; k < 3; k++) p[c][k] = px[6 + c * 3 + k] - cam[k];
  for (int k = 0; k < 3; k++) {
    pdx[k] = (px[0] * p[0][k] + px[1] * p[1][k]) + px[2] * p[2][k];
    pdy[k] = (px[3] * p[0][k] + px[4] * p[1][k]) + px[5] * p[2][k];
  }
}

void orc_gbuffer_tangent_frame(const float px[24], const float cam[3], float out[6]) {
  float pdx[3], pdy[3];
  gb_position_derivatives(px, cam, pdx, pdy);
  gb_tangent_frame(pdx, pdy, px + 21, px[17], px[18], px[19], px[20], out, out + 3);
}

static void gb_oct(float x, float y, float z, float out[2]) {
  Vec3_f32 v = {x, y, z};
  vec3_to_oct_f32(v, out);
}

int orc_gbuffer_shade(const OxcMaterialTable* table, uint32_t material_index, const float px[24], const float cam[3], uint32_t want, float out[16]) {
  if (!table || material_index >= table->material_count) return 0;
  const OxcMaterial* m = &table->materials[material_index];
  const float n[3] = {px[21], px[22], px[23]};
  const GbSampler smp = gb_sampler(table->samplers && m->sampler_index < table->sampler_count ? &table->samplers[m->sampler_index] : NULL);
  /* :117-122 */
  const float us = orc_dequantize_half(m->uv_size[0]), vs = orc_dequantize_half(m->uv_size[1]);
  const float u = px[15] * us + orc_dequantize_half(m->uv_offset[0]), v = px[16] * vs + orc_dequantize_half(m->uv_offset[1]);
  const float dxu = px[17] * us, dxv = px[18] * vs, dyu = px[19] * us, dyv = px[20] * vs;
  float s[4];
#define GB_SAMPLE(index) gb_sample_grad(&table->images[index], smp, u, v, dxu, dxv, dyu, dyv, s)
  memset(out, 0, 16 * sizeof(float));
  if (want & 1u) { /* scene.slang:110-119 */
    for (int c = 0; c < 4; c++) out[c] = orc_dequantize_half(m->albedo_color[c]);
    if (m->flags & OXC_MATERIAL_HAS_ALBEDO_IMAGE) {
      GB_SAMPLE(m->albedo_image_index);
      for (int c = 0; c < 4; c++) out[c] = out[c] * s[c];
    }
  }
  if (want & 2u) { /* :127-170 */
    float pdx[3], pdy[3];
    gb_position_derivatives(px, cam, pdx, pdy);
    const float dxn = (pdx[0] * n[0] + pdx[1] * n[1]) + pdx[2] * n[2], dyn = (pdy[0] * n[0] + pdy[1] * n[1]) + pdy[2] * n[2];
    float t[3], b[3];
    gb_tangent_frame(pdx, pdy, n, dxu, dxv, dyu, dyv, t, b);
    float o[3] = {n[0], n[1], n[2]};
    if (m->flags & OXC_MATERIAL_HAS_NORMAL_IMAGE) {
      GB_SAMPLE(m->normal_image_index);
      float e[3] = {s[0] * 2.0f - 1.0f, s[1] * 2.0f - 1.0f, s[2] * 2.0f - 1.0f};
      if (m->flags & OXC_MATERIAL_NORMAL_FLIP_Y) e[1] = -e[1];
      if (m->flags & OXC_MATERIAL_NORMAL_TWO_COMPONENT) {
        const float q = 1.0f - (e[0] * e[0] + e[1] * e[1]);
        e[2] = sqrtf(q > 0.0f ? (q < 1.0f ? q : 1.0f) : 0.0f); /* saturate, NaN -> 0 */
      }
      for (int k = 0; k < 3; k++) o[k] = (e[0] * t[k] + e[1] * b[k]) + e[2] * n[k];
      const float len = sqrtf((o[0] * o[0] + o[1] * o[1]) + o[2] * o[2]);
      for (int k = 0; k < 3; k++) o[k] = o[k] / len;
    }
    gb_oct(o[0], o[1], o[2], out + 4);
    gb_oct(n[0], n[1], n[2], out + 6);
  }
  if (want & 4u) { /* scene.slang:130-139 */
    for (int c = 0; c < 3; c++) out[8 + c] = orc_dequantize_half(m->emissive_color[c]);
    if (m->flags & OXC_MATERIAL_HAS_EMISSIVE_IMAGE) {
      GB_SAMPLE(m->emissive_image_index);
      for (int c = 0; c < 3; c++) out[8 + c] = out[8 + c] * s[c];
    }
  }
  if (want & 8u) { /* scene.slang:141-159 */
    out[12] = orc_dequantize_half(m->metallic_factor); out[13] = orc_dequantize_half(m->roughness_factor); out[14] = 1.0f;
    if (m->flags & OXC_MATERIAL_HAS_METALLIC_ROUGHNESS_IMAGE) {
      GB_SAMPLE(m->metallic_roughness_image_index);
      out[12] = out[12] * s[2]; out[13] = out[13] * s[1];
    }
    if (m->flags & OXC_MATERIAL_HAS_OCCLUSION_IMAGE) { GB_SAMPLE(m->occlusion_image_index); out[14] = s[0]; }
  }
#undef GB_SAMPLE
  return 1;
}

void orc_decode_gbuffer_pixels(const OrcScene* scene, const OxcMeshletInstance* meshlet_instances, uint32_t total, const OxcCullCamera* cam,
                               const uint32_t* vis32, uint32_t width, uint32_t height, float* records, int32_t* material) {
  const size_t n_px = (size_t)width * height;
  float* planes = (float*)malloc(n_px * 4 * sizeof(float) * 5);
  float *lam = planes, *dx = planes + n_px * 4, *dy = planes + n_px * 8, *un = planes + n_px * 12, *ug = planes + n_px * 16;
  orc_decode_visbuffer(scene, meshlet_instances, total, cam, vis32, width, height, lam, dx, dy, un, ug);
  for (size_t pix = 0; pix < n_px; pix++) {
    const float status = lam[pix * 4 + 3];
    float* px = records + pix * 24;
    memset(px, 0, 24 * sizeof(float));
    material[pix] = status == 0.0f ? -1 : -2;
    if (status != 1.0f) continue;
    const uint32_t mii = (vis32[pix] >> OXC_VIS_PRIMITIVE_BITS) & 0xFFFFFFu, tri = vis32[pix] & OXC_VIS_PRIMITIVE_MASK;
    const OxcMeshletInstance mi = meshlet_instances[mii];
    const OxcMeshInstance inst = scene->mesh_instances[mi.mesh_instance_index];
    const OxcMesh* mesh = &scene->meshes[inst.mesh_index];
    const float* world = scene->transforms[inst.transform_index].world;
    const OxcMeshLOD* lod = mesh_lod(scene, mesh, inst.lod_index);
    const OxcMeshlet meshlet = ((const OxcMeshlet*)(scene->blob + lod->meshlets))[mi.meshlet_index];
    const uint32_t* micro = (const uint32_t*)(scene->blob + lod->local_triangle_indices);
    const uint32_t* vidx = (const uint32_t*)(scene->blob + lod->indirect_vertex_indices);
    const uint16_t* pos = (const uint16_t*)(scene->blob + mesh->vertex_positions);
    const uint32_t base = meshlet.local_triangle_index_offset + tri * 3;
    Vec3_f32 nrm[3];
    for (int c = 0; c < 3; c++) {
      const uint32_t i = vidx[meshlet.indirect_vertex_index_offset + micro_index(micro, base + (uint32_t)c)];
      Vec4_f32 p = {orc_dequantize_half(pos[i * 4 + 0]), orc_dequantize_half(pos[i * 4 + 1]), orc_dequantize_half(pos[i * 4 + 2]), 1.0f};
      const Vec4_f32 w = mul_mv_f32(world, p);
      px[6 + c * 3 + 0] = w.x; px[6 + c * 3 + 1] = w.y; px[6 + c * 3 + 2] = w.z;
      if (mesh->vertex_normals) nrm[c] = decode_normal_f32(((const uint32_t*)(scene->blob + mesh->vertex_normals))[i]);
      else { nrm[c].x = 0; nrm[c].y = 0; nrm[c].z = 0; }
    }
    for (int c = 0; c < 3; c++) { px[c] = dx[pix * 4 + c]; px[3 + c] = dy[pix * 4 + c]; }
    px[15] = un[pix * 4 + 0]; px[16] = un[pix * 4 + 1];
    for (int c = 0; c < 4; c++) px[17 + c] = ug[pix * 4 + c];
    /* orc_decode_visbuffer's world normal, :146-147 */
    const float* l = lam + pix * 4;
    Vec3_f32 b0 = {world[0], world[1], world[2]}, b1 = {world[4], world[5], world[6]}, b2 = {world[8], world[9], world[10]};
    Vec3_f32 r0 = cross3_f32(b1, b2), r1 = cross3_f32(b2, b0), r2 = cross3_f32(b0, b1);
    Vec3_f32 wn[3];
    for (int c = 0; c < 3; c++) {
      wn[c].x = (r0.x * nrm[c].x + r1.x * nrm[c].y) + r2.x * nrm[c].z;
      wn[c].y = (r0.y * nrm[c].x + r1.y * nrm[c].y) + r2.y * nrm[c].z;
      wn[c].z = (r0.z * nrm[c].x + r1.z * nrm[c].y) + r2.z * nrm[c].z;
    }
    Vec3_f32 nn = {(l[0] * wn[0].x + l[1] * wn[1].x) + l[2] * wn[2].x, (l[0] * wn[0].y + l[1] * wn[1].y) + l[2] * wn[2].y,
                   (l[0] * wn[0].z + l[1] * wn[1].z) + l[2] * wn[2].z};
    const float len = length3_f32(nn);
    px[21] = nn.x / len; px[22] = nn.y / len; px[23] = nn.z / len;
    material[pix] = (int32_t)inst.material_index;
  }
  free(planes);
}

uint64_t orc_decode_gbuffer(const OrcScene* scene, const OxcMeshletInstance* meshlet_instances, uint32_t total, const OxcCullCamera* cam,
                            const uint32_t* vis32, uint32_t width, uint32_t height, const OxcMaterialTable* table, float* albedo, float* normal,
                            float* emissive, float* mro) {
  const size_t n_px = (size_t)width * height;
  float* records = (float*)malloc(n_px * 24 * sizeof(float));
  int32_t* material = (int32_t*)malloc(n_px * sizeof(int32_t));
  orc_decode_gbuffer_pixels(scene, meshlet_instances, total, cam, vis32, width, height, records, material);
  float* const outs[4] = {albedo, normal, emissive, mro};
  const uint32_t want = (albedo ? 1u : 0u) | (normal ? 2u : 0u) | (emissive ? 4u : 0u) | (mro ? 8u : 0u);
  uint64_t bad = 0;
  for (size_t pix = 0; pix < n_px; pix++) {
    if (material[pix] == -1) continue; /* discard: not written */
    float out[16] = {0};
    if (material[pix] >= 0 && !orc_gbuffer_shade(table, (uint32_t)material[pix], records + pix * 24, cam->position, want, out)) bad++;
    for (int k = 0; k < 4; k++)
      if (outs[k]) memcpy(outs[k] + pix * 4, out + k * 4, 4 * sizeof(float));
  }
  free(records);
  free(material);
  return bad;
}
