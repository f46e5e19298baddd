// oxc_raster_core.cuh — the per-triangle core of the software visibility-buffer raster: snap to the 24.8 grid, set-up, edge
// functions, depth interpolation, the packed 64-bit max.  Pure per-thread functions (no warp intrinsics, no shared memory), so
// tests/raster_core_vs_oracle.cpp can compile exactly this source for the HOST and compare it with the oracle's specification
// (oracle/oxc_oracle.c, comment above raster_triangle) pixel for pixel without a GPU.  The kernels that schedule these
// functions over warps live in kernels_tri.cuh.
#pragma once
#include <climits>

#include "oxc_exact.cuh"

namespace oxc {

// Per-vertex screen record (computed once per vertex, not per corner): 24.8 fixed-point position + NDC depth.
// valid = w > 0 and |fx|,|fy| <= 2^22 (raster spec steps 2-3); invalid is flagged with fx == INT_MIN.
struct __align__(16) ScreenVert {
  int fx, fy;
  float z;
  int pad;
};

OXC_DI ScreenVert to_screen(float4 c, float fW, float fH) {
  ScreenVert v;
  v.fx = INT_MIN; v.fy = 0; v.z = 0.f; v.pad = 0;
  if (!(c.w > 0.0f)) return v;
  const float rw = fd(1.0f, c.w);
  const float nx = fm(c.x, rw), ny = fm(c.y, rw);
  const float sx = fm(fa(fm(nx, 0.5f), 0.5f), fW), sy = fm(fa(fm(ny, 0.5f), 0.5f), fH);
  const float qx = floorf(fa(fm(sx, 256.0f), 0.5f)), qy = floorf(fa(fm(sy, 256.0f), 0.5f));
  if (!(fabsf(qx) <= 4194304.0f && fabsf(qy) <= 4194304.0f)) return v;
  v.fx = (int)qx; v.fy = (int)qy; v.z = fm(c.z, rw);
  return v;
}

// oracle: orc_triangle_covers_no_sample
OXC_DI bool tri_covers_no_sample(float4 c0, float4 c1, float4 c2, float fW, float fH, uint32_t W, uint32_t H) {
  const ScreenVert v0 = to_screen(c0, fW, fH), v1 = to_screen(c1, fW, fH), v2 = to_screen(c2, fW, fH);
  if (v0.fx == INT_MIN || v1.fx == INT_MIN || v2.fx == INT_MIN) return false;
  const int minx = min(v0.fx, min(v1.fx, v2.fx)), maxx = max(v0.fx, max(v1.fx, v2.fx));
  const int miny = min(v0.fy, min(v1.fy, v2.fy)), maxy = max(v0.fy, max(v1.fy, v2.fy));
  const int px0 = max(0, (minx - 128 + 255) >> 8), px1 = min((int)W - 1, (maxx - 128) >> 8);
  const int py0 = max(0, (miny - 128 + 255) >> 8), py1 = min((int)H - 1, (maxy - 128) >> 8);
  return px1 < px0 || py1 < py0;
}

struct TriSetup {
  int ax, ay, bx, by, cx, cy;   // 24.8 fixed point, a/b/c positively oriented (b,c swapped)
  float za, dzb, dzc;           // depth at a, per-triangle gradients w.r.t. the edge functions of b and c
  int px0, px1, py0, py1;
  int bias;                     // bit0..2: edge biases (1 = -1)
  bool narrow;                  // all edge functions fit 32 bits (extent < 2^14 sub-pixels)
};

OXC_DI long long orient2d(int ax, int ay, int bx, int by, int cx, int cy) {
  return (long long)(bx - ax) * (long long)(cy - ay) - (long long)(by - ay) * (long long)(cx - ax);
}
OXC_DI int edge_bias_bit(int ax, int ay, int bx, int by) {
  const int dx = bx - ax, dy = by - ay;
  return ((dy > 0) || (dy == 0 && dx < 0)) ? 0 : 1;
}

// steps 2-4 of the raster spec; anything but TRI_DRAW = nothing to draw.  Rejections commute, so the cheapest go first:
// the bounding box (most sub-pixel triangles cover no sample centre) before the signed area.
enum : int { TRI_DRAW = 0, TRI_INVALID_VERTEX = 1, TRI_NO_SAMPLE = 2, TRI_BACK_OR_DEGENERATE = 3 };
OXC_DI int tri_setup(const ScreenVert v0, const ScreenVert v1, const ScreenVert v2, uint32_t W, uint32_t H, TriSetup& s) {
  if (v0.fx == INT_MIN || v1.fx == INT_MIN || v2.fx == INT_MIN) return TRI_INVALID_VERTEX;
  const int minx = min(v0.fx, min(v1.fx, v2.fx)), maxx = max(v0.fx, max(v1.fx, v2.fx));
  const int miny = min(v0.fy, min(v1.fy, v2.fy)), maxy = max(v0.fy, max(v1.fy, v2.fy));
  s.px0 = max(0, (minx - 128 + 255) >> 8);
  s.px1 = min((int)W - 1, (maxx - 128) >> 8);
  s.py0 = max(0, (miny - 128 + 255) >> 8);
  s.py1 = min((int)H - 1, (maxy - 128) >> 8);
  if (s.px1 < s.px0 || s.py1 < s.py0) return TRI_NO_SAMPLE; // the snapped bounding box holds no sample centre
  // extent < 2^14 sub-pixels per axis: every edge-function value inside the bbox fits 32 bits
  s.narrow = (maxx - minx) < 16384 && (maxy - miny) < 16384;
  long long area2;
  if (s.narrow) area2 = (long long)((v1.fx - v0.fx) * (v2.fy - v0.fy) - (v1.fy - v0.fy) * (v2.fx - v0.fx));
  else area2 = orient2d(v0.fx, v0.fy, v1.fx, v1.fy, v2.fx, v2.fy);
  if (area2 >= 0) return TRI_BACK_OR_DEGENERATE;
  s.ax = v0.fx; s.ay = v0.fy; s.bx = v2.fx; s.by = v2.fy; s.cx = v1.fx; s.cy = v1.fy;
  const float fa_ = (float)(-area2);
  s.za = v0.z;
  s.dzb = fd(fs(v2.z, v0.z), fa_);
  s.dzc = fd(fs(v1.z, v0.z), fa_);
  s.bias = edge_bias_bit(s.bx, s.by, s.cx, s.cy) | (edge_bias_bit(s.cx, s.cy, s.ax, s.ay) << 1) |
           (edge_bias_bit(s.ax, s.ay, s.bx, s.by) << 2);
  return TRI_DRAW;
}

// tri_setup for a raster that draws both windings (the VSM shadow draw, cullMode None): area2 < 0 is set up exactly as tri_setup;
// area2 > 0 keeps the submitted order (a, b, c = vertices 0, 1, 2) instead of being rejected; area2 == 0 draws nothing.
// kept_order = the area2 > 0 case (the caller's per-vertex attributes follow the same order).
OXC_DI int tri_setup_two_sided(const ScreenVert v0, const ScreenVert v1, const ScreenVert v2, uint32_t W, uint32_t H, TriSetup& s,
                               bool& kept_order) {
  if (v0.fx == INT_MIN || v1.fx == INT_MIN || v2.fx == INT_MIN) return TRI_INVALID_VERTEX;
  const int minx = min(v0.fx, min(v1.fx, v2.fx)), maxx = max(v0.fx, max(v1.fx, v2.fx));
  const int miny = min(v0.fy, min(v1.fy, v2.fy)), maxy = max(v0.fy, max(v1.fy, v2.fy));
  s.px0 = max(0, (minx - 128 + 255) >> 8);
  s.px1 = min((int)W - 1, (maxx - 128) >> 8);
  s.py0 = max(0, (miny - 128 + 255) >> 8);
  s.py1 = min((int)H - 1, (maxy - 128) >> 8);
  if (s.px1 < s.px0 || s.py1 < s.py0) return TRI_NO_SAMPLE;
  s.narrow = (maxx - minx) < 16384 && (maxy - miny) < 16384;
  const long long area2 = orient2d(v0.fx, v0.fy, v1.fx, v1.fy, v2.fx, v2.fy);
  if (area2 == 0) return TRI_BACK_OR_DEGENERATE;
  kept_order = area2 > 0;
  const ScreenVert b = kept_order ? v1 : v2, c = kept_order ? v2 : v1;
  s.ax = v0.fx; s.ay = v0.fy; s.bx = b.fx; s.by = b.fy; s.cx = c.fx; s.cy = c.fy;
  const float fa_ = (float)(kept_order ? area2 : -area2);
  s.za = v0.z;
  s.dzb = fd(fs(b.z, v0.z), fa_);
  s.dzc = fd(fs(c.z, v0.z), fa_);
  s.bias = edge_bias_bit(s.bx, s.by, s.cx, s.cy) | (edge_bias_bit(s.cx, s.cy, s.ax, s.ay) << 1) |
           (edge_bias_bit(s.ax, s.ay, s.bx, s.by) << 2);
  return TRI_DRAW;
}

// coverage (step 5) and depth (step 6) of one sample given its three edge-function values: false = not covered or z outside [0, 1]
OXC_DI bool sample_depth(const TriSetup& s, long long e0, long long e1, long long e2, float& z) {
  if ((e0 - (s.bias & 1)) < 0 || (e1 - ((s.bias >> 1) & 1)) < 0 || (e2 - ((s.bias >> 2) & 1)) < 0) return false;
  z = fa(fa(s.za, fm((float)e1, s.dzb)), fm((float)e2, s.dzc));
  return z >= 0.0f && z <= 1.0f;
}

// steps 5-6 given the three edge-function values at the pixel centre
OXC_DI void shade_pixel(const TriSetup& s, long long e0, long long e1, long long e2, int px, int py, uint32_t data,
                        unsigned long long* vis, uint32_t W) {
  if ((e0 - (s.bias & 1)) < 0 || (e1 - ((s.bias >> 1) & 1)) < 0 || (e2 - ((s.bias >> 2) & 1)) < 0) return;
  const float zz = fa(fa(s.za, fm((float)e1, s.dzb)), fm((float)e2, s.dzc));
  if (!(zz >= 0.0f && zz <= 1.0f)) return;
  uint32_t zb = __float_as_uint(zz);
  zb = zb == 0x80000000u ? 0u : zb; // -0.0 -> +0.0 so unsigned order == depth order
  const unsigned long long v = ((unsigned long long)zb << 32) | data;
  unsigned long long* ptr = vis + (size_t)py * W + px;
  // reverse-Z GreaterOrEqual == max (visbuffer.slang:72-74 packing).  No "if (v > *ptr)" pre-test: the result is unused, so this
  // is a fire-and-forget RED.MAX.64, while the pre-test's load stalled the whole warp on an L2 round trip from inside the
  // divergent pixel loop
  atomicMax(ptr, v);
}

OXC_DI void raster_pixel(const TriSetup& s, int px, int py, uint32_t data, unsigned long long* vis, uint32_t W) {
  const int sx = px * 256 + 128, sy = py * 256 + 128;
  shade_pixel(s, orient2d(s.bx, s.by, s.cx, s.cy, sx, sy), orient2d(s.cx, s.cy, s.ax, s.ay, sx, sy),
              orient2d(s.ax, s.ay, s.bx, s.by, sx, sy), px, py, data, vis, W);
}

OXC_DI int orient2d_32(int ax, int ay, int bx, int by, int cx, int cy) { return (bx - ax) * (cy - ay) - (by - ay) * (cx - ax); }

// raster_small for a narrow triangle (32-bit edge functions), the per-lane loop of k_raster_visbuffer.  Each edge's bias is
// folded into its start value, so a sample is covered when no stepped value is negative (one test of the three values' OR);
// e1 and e2 get their bias back for the depth, which converts the same values as shade_pixel ((float)int32 == (float)int64 of
// the same value).  The image pointer is stepped with the pixel instead of recomputed from (px, py).
OXC_DI void raster_narrow(const TriSetup& s, uint32_t data, unsigned long long* vis, uint32_t W) {
  const int sx0 = s.px0 * 256 + 128, sy0 = s.py0 * 256 + 128;
  const int b1 = (s.bias >> 1) & 1, b2 = (s.bias >> 2) & 1;
  int r0 = orient2d_32(s.bx, s.by, s.cx, s.cy, sx0, sy0) - (s.bias & 1), r1 = orient2d_32(s.cx, s.cy, s.ax, s.ay, sx0, sy0) - b1,
      r2 = orient2d_32(s.ax, s.ay, s.bx, s.by, sx0, sy0) - b2;
  const int dx0 = -(s.cy - s.by) * 256, dy0 = (s.cx - s.bx) * 256, dx1 = -(s.ay - s.cy) * 256, dy1 = (s.ax - s.cx) * 256,
            dx2 = -(s.by - s.ay) * 256, dy2 = (s.bx - s.ax) * 256;
  const int nx = s.px1 - s.px0;
  unsigned long long* row = vis + (size_t)s.py0 * W + s.px0;
  for (int py = s.py0; py <= s.py1; py++, row += W) {
    int e0 = r0, e1 = r1, e2 = r2;
    for (int i = 0; i <= nx; i++) {
      if ((e0 | e1 | e2) >= 0) {
        const float zz = fa(fa(s.za, fm((float)(e1 + b1), s.dzb)), fm((float)(e2 + b2), s.dzc));
        if (zz >= 0.0f && zz <= 1.0f) {
          uint32_t zb = __float_as_uint(zz);
          zb = zb == 0x80000000u ? 0u : zb;
          atomicMax(row + i, ((unsigned long long)zb << 32) | data); // fire-and-forget RED (see shade_pixel)
        }
      }
      e0 += dx0; e1 += dx1; e2 += dx2;
    }
    r0 += dy0; r1 += dy1; r2 += dy2;
  }
}

// one lane walks the (small) bounding box with incrementally stepped edge functions (adds only)
OXC_DI void raster_small(const TriSetup& s, uint32_t data, unsigned long long* vis, uint32_t W) {
  if (s.narrow) {
    raster_narrow(s, data, vis, W);
    return;
  }
  const int sx0 = s.px0 * 256 + 128, sy0 = s.py0 * 256 + 128;
  long long r0 = orient2d(s.bx, s.by, s.cx, s.cy, sx0, sy0);
  long long r1 = orient2d(s.cx, s.cy, s.ax, s.ay, sx0, sy0);
  long long r2 = orient2d(s.ax, s.ay, s.bx, s.by, sx0, sy0);
  // orient2d(a,b,p) = (bx-ax)*(py-ay) - (by-ay)*(px-ax):  d/dpx = -(by-ay), d/dpy = (bx-ax)   (x256 per pixel)
  const long long dx0 = -(long long)(s.cy - s.by) * 256, dy0 = (long long)(s.cx - s.bx) * 256;
  const long long dx1 = -(long long)(s.ay - s.cy) * 256, dy1 = (long long)(s.ax - s.cx) * 256;
  const long long dx2 = -(long long)(s.by - s.ay) * 256, dy2 = (long long)(s.bx - s.ax) * 256;
  for (int py = s.py0; py <= s.py1; py++) {
    long long e0 = r0, e1 = r1, e2 = r2;
    for (int px = s.px0; px <= s.px1; px++) {
      shade_pixel(s, e0, e1, e2, px, py, data, vis, W);
      e0 += dx0; e1 += dx1; e2 += dx2;
    }
    r0 += dy0; r1 += dy1; r2 += dy2;
  }
}

// ---- clip-space planes of the triangles the plain rules drop (specification: oracle/oxc_oracle.c raster_triangle_clipped):
//      near (w - z), left (w + x), right (w - x), bottom (w + y), top (w - y) ----
OXC_DI float clip_plane_distance(const float4 v, int plane) {
  switch (plane) {
    case 0: return fs(v.w, v.z);
    case 1: return fa(v.w, v.x);
    case 2: return fs(v.w, v.x);
    case 3: return fa(v.w, v.y);
    default: return fs(v.w, v.y);
  }
}

// Sutherland-Hodgman against the five planes; cut points evaluated from the inside vertex to the outside vertex with the canonical
// f32 operation order.  Result: poly[cur][0..n), n in {0, 3..8}; the caller draws the fan (P0, Pi, Pi+1) with the plain rules.
OXC_DI int clip_polygon(float4 c0, float4 c1, float4 c2, float4 (*poly)[12], int& cur) {
  int n = 3;
  cur = 0;
  poly[0][0] = c0; poly[0][1] = c1; poly[0][2] = c2;
  for (int plane = 0; plane < 5 && n >= 3; plane++) {
    const float4* in = poly[cur];
    float4* out = poly[cur ^ 1];
    int m = 0;
    for (int i = 0; i < n; i++) {
      const float4 A = in[i], B = in[(i + 1) % n];
      const float dA = clip_plane_distance(A, plane), dB = clip_plane_distance(B, plane);
      const bool inA = dA >= 0.0f, inB = dB >= 0.0f;
      if (inA) out[m++] = A;
      if (inA != inB) {
        const float4 I = inA ? A : B, O = inA ? B : A;
        const float dI = inA ? dA : dB, dO = inA ? dB : dA;
        const float tt = fd(dI, fs(dI, dO));
        out[m++] = make_float4(fa(I.x, fm(tt, fs(O.x, I.x))), fa(I.y, fm(tt, fs(O.y, I.y))), fa(I.z, fm(tt, fs(O.z, I.z))),
                               fa(I.w, fm(tt, fs(O.w, I.w))));
      }
    }
    n = m;
    cur ^= 1;
  }
  return n;
}

} // namespace oxc
