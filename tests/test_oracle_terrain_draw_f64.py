"""An independent binary64 restatement of passes/terrain_visbuffer.slang (vs_main, hs_constants with edge_tessellation, the fractional_odd
quad tessellator as include/oxcull.h oxc_draw_terrain items 2-3 commit to it, ds_main, fs_main) and of the rasteriser's coverage and
depth, written from the shader text in numpy, against the oracle (oracle/oxc_oracle_terrain_draw.c) per pixel.

The restatement shares no code with the oracle: tan is numpy's, the heights are a binary64 bilinear tap, the tessellator is a plain merge
walk over binary64 edge points, and a triangle is drawn when the face whose normal points up (+y) faces the camera, the rule item 6
derives for the raster's one winding; a pixel is covered when its centre lies inside the projected triangle, and its depth is the
screen-space affine interpolation of z / w, kept by the maximum (GreaterOrEqual on reverse-Z).  The cameras keep every triangle in
front of them, so the restatement has no clip path.

Decisions within their margin are counted, bounded and not compared: a patch whose binary64 factor lies within 1e-5 (relative) of a
rounding step of item 2 (odd integers, the pins at 1 and 63), or one of whose stitch walks compares two different coordinates within
1e-6, is drawn by neither side; a pixel whose centre lies within 1/128 pixel (twice
the 24.8 snap of a vertex) of
an edge of a triangle covering it (the top-left rule and the 24.8 snapping decide it), within 1e-4 of another triangle's depth, or
under a triangle seen nearly edge-on (|cos| < 1e-3 between its normal and the view: the raster's winding is the snapped area's sign)
is not compared.  Every other pixel has the same coverage, and its depth agrees within 2e-4 relative plus the tilt that snapping
each vertex by up to 1/512 pixel per axis can give the front triangle's plane: its depth range times 2 / 512 over its least altitude
in pixels."""
import numpy as np
import pytest

from tests import helpers_terrain as ht

CLEAR = np.uint64(0xFFFFFFFF)
FACTOR_MARGIN, WALK_MARGIN, EDGE_MARGIN_PX, FACING_MARGIN, DEPTH_RTOL = 1e-5, 1e-6, 1.0 / 128.0, 1e-3, 2e-4


@pytest.fixture(scope="module")
def so():
    import pyoracle_terrain_draw

    pyoracle_terrain_draw.build()
    return pyoracle_terrain_draw


def _height(hm, t, inv, x, z):
    """sample_height: base + bilinear(R16 / 65535, ClampToEdge, texel centres) * scale, binary64"""
    ry, rx = hm.shape
    u = (x - float(t["world_min"][0][0])) * inv[0] * rx - 0.5
    v = (z - float(t["world_min"][0][1])) * inv[1] * ry - 0.5
    x0, y0 = np.floor(u), np.floor(v)
    fx, fy = u - x0, v - y0
    ix0, iy0 = int(np.clip(x0, 0, rx - 1)), int(np.clip(y0, 0, ry - 1))
    ix1, iy1 = int(np.clip(x0 + 1, 0, rx - 1)), int(np.clip(y0 + 1, 0, ry - 1))
    a = hm.astype(np.float64) / 65535.0
    top = a[iy0, ix0] * (1 - fx) + a[iy0, ix1] * fx
    bot = a[iy1, ix0] * (1 - fx) + a[iy1, ix1] * fx
    return float(t["base_height"][0]) + (top * (1 - fy) + bot * fy) * float(t["height_scale"][0])


def _edge(a, b, cam, scale, target, max_tess):
    """edge_tessellation"""
    c = (a + b) * 0.5
    radius = np.linalg.norm(a - b) * 0.5
    vd = max(np.linalg.norm(c - cam["position"][0].astype(np.float64)) - radius, float(cam["near_clip"][0]))
    return min(max(2.0 * radius * scale / vd / target, 1.0), max_tess)


def _round(f):
    """item 2: pin to [1, 63], next odd integer; and whether f lies within the margin of a step"""
    c = min(max(f, 1.0), 63.0)
    n = 2 * int(np.ceil((c - 1.0) / 2.0)) + 1
    steps = np.arange(1, 64, 2, dtype=np.float64)
    return n, bool(np.any(np.abs(f - steps) <= FACTOR_MARGIN * steps))


def _points(f, n):
    if n == 1:
        return np.array([0.0, 1.0])
    L, s = 1.0 / f, (f - (n - 2)) / (2.0 * f)
    t = np.zeros(n + 1)
    t[n] = 1.0
    for k in range(1, (n + 1) // 2):
        t[k] = s + (k - 1) * L
        t[n - k] = 1.0 - t[k]
    return t


def _walk(outer, inner):
    """merge walk of two rows by coordinate, ties to the outer row: a list of (kind, i, j) steps"""
    i = j = 0
    out = []
    while i < len(outer) - 1 or j < len(inner) - 1:
        if j < len(inner) - 1 and i < len(outer) - 1 and 0.0 < abs(outer[i + 1] - inner[j + 1]) <= WALK_MARGIN:
            return None  # binary32 may order the two points the other way
        if j == len(inner) - 1 or (i < len(outer) - 1 and outer[i + 1] <= inner[j + 1]):
            out.append(((outer[i], 0), (outer[i + 1], 0), (inner[j], 1)))
            i += 1
        else:
            out.append(((outer[i], 0), (inner[j + 1], 1), (inner[j], 1)))
            j += 1
    return out


def _patch_triangles(hm, t, st, cam, idx):
    """vs_main + hs_constants + the tessellator: the patch's domain triangles (unordered) and its corners, or None when a factor lies
    within its margin"""
    pc = t["patch_count"][0]
    px, pz = idx % int(pc[0]), idx // int(pc[0])
    inv = st["inv_world_size"][0].astype(np.float64)
    wmin, wsize = t["world_min"][0].astype(np.float64), t["world_size"][0].astype(np.float64)
    corners = []
    for dx, dz in ((0, 0), (1, 0), (1, 1), (0, 1)):
        x = wmin[0] + (px + dx) / float(pc[0]) * wsize[0]
        z = wmin[1] + (pz + dz) / float(pc[1]) * wsize[1]
        corners.append(np.array([x, _height(hm, t, inv, x, z), z]))
    scale = float(cam["resolution"][0][1]) * 0.5 / np.tan(np.radians(float(st["fov"][0])) * 0.5)
    target, mt = float(st["target_edge_pixels"][0]), float(st["max_tessellation"][0])
    e = [_edge(corners[0], corners[3], cam, scale, target, mt), _edge(corners[0], corners[1], cam, scale, target, mt),
         _edge(corners[1], corners[2], cam, scale, target, mt), _edge(corners[3], corners[2], cam, scale, target, mt)]
    f = e + [max(e[1], e[3]), max(e[0], e[2])]
    rounded = [_round(x) for x in f]
    if any(r[1] for r in rounded):
        return None, corners
    n = [r[0] for r in rounded]
    if all(k == 1 for k in n):
        return [((0, 0), (1, 0), (1, 1)), ((0, 0), (1, 1), (0, 1))], corners
    fi = [min(max(x, 1.0), 63.0) for x in f[4:]]  # item 2: the pin applies to the points as to the rounding
    for k in range(2):
        if n[4 + k] == 1:
            n[4 + k], fi[k] = 3, 1.0 + 2.0**-23
    a, b = _points(fi[0], n[4]), _points(fi[1], n[5])
    tris = []
    # bottom (v0, v = 0), top (v1, v = 1) along u; left (u0, u = 0), right (u1, u = 1) along v
    for e_idx, along_u, fixed_o, fixed_i in ((1, True, 0.0, b[1]), (3, True, 1.0, b[-2]), (0, False, 0.0, a[1]), (2, False, 1.0, a[-2])):
        outer = _points(min(max(f[e_idx], 1.0), 63.0), n[e_idx])
        inner = (a if along_u else b)[1:-1]
        steps = _walk(outer, inner)
        if steps is None:
            return None, corners
        for tri in steps:
            tris.append(tuple((c, fixed_o if row == 0 else fixed_i) if along_u else (fixed_o if row == 0 else fixed_i, c) for c, row in tri))
    for j in range(1, n[5] - 1):
        for i in range(1, n[4] - 1):
            tris.append(((a[i], b[j]), (a[i + 1], b[j]), (a[i + 1], b[j + 1])))
            tris.append(((a[i], b[j]), (a[i + 1], b[j + 1]), (a[i], b[j + 1])))
    return tris, corners


def _raster(hm, t, st, cam, patches, w, h):
    """ds_main + fs_main + coverage and depth in binary64: (depth image with -inf where empty, ambiguous-pixel mask, the depth
    tolerance of each pixel's front triangle)"""
    inv = st["inv_world_size"][0].astype(np.float64)
    M = cam["projection_view"][0].reshape(4, 4).T.astype(np.float64)
    eye = cam["position"][0].astype(np.float64)
    depth = np.full((h, w), -np.inf)
    ambiguous = np.zeros((h, w), bool)
    tol = np.zeros((h, w))
    for tris, corners in patches:
        p0, p1, p2, p3 = corners
        for tri in tris:
            P = []
            for u, v in tri:
                e0, e1 = p0 * (1 - u) + p1 * u, p3 * (1 - u) + p2 * u
                q = e0 * (1 - v) + e1 * v
                P.append(np.array([q[0], _height(hm, t, inv, q[0], q[2]), q[2]]))
            nrm = np.cross(P[1] - P[0], P[2] - P[0])
            if nrm[1] < 0:
                nrm = -nrm
            facing = np.dot(nrm, eye - P[0]) / max(np.linalg.norm(nrm) * np.linalg.norm(eye - P[0]), 1e-300)
            if facing <= -FACING_MARGIN:  # the face seen from +y must face the camera
                continue
            C = np.array([M @ np.append(p, 1.0) for p in P])
            if (C[:, 3] <= 0).any():
                continue
            sx = (C[:, 0] / C[:, 3] * 0.5 + 0.5) * w
            sy = (C[:, 1] / C[:, 3] * 0.5 + 0.5) * h
            z = C[:, 2] / C[:, 3]
            x0, x1 = max(0, int(np.floor(sx.min() - 0.5))), min(w - 1, int(np.ceil(sx.max() - 0.5)))
            y0, y1 = max(0, int(np.floor(sy.min() - 0.5))), min(h - 1, int(np.ceil(sy.max() - 0.5)))
            if x1 < x0 or y1 < y0:
                continue
            ys, xs = np.mgrid[y0:y1 + 1, x0:x1 + 1] + 0.5
            area = (sx[1] - sx[0]) * (sy[2] - sy[0]) - (sy[1] - sy[0]) * (sx[2] - sx[0])
            if area == 0:
                continue
            lam = []
            for k in range(3):
                a_, b_ = (k + 1) % 3, (k + 2) % 3
                ek = (sx[b_] - sx[a_]) * (ys - sy[a_]) - (sy[b_] - sy[a_]) * (xs - sx[a_])
                lam.append(ek / area)
            lam = np.array(lam)
            lens = [np.hypot(sx[(k + 2) % 3] - sx[(k + 1) % 3], sy[(k + 2) % 3] - sy[(k + 1) % 3]) for k in range(3)]
            dist = np.array([lam[k] * abs(area) / max(lens[k], 1e-300) for k in range(3)])  # pixels from each edge
            inside = (dist > EDGE_MARGIN_PX).all(0)
            near = (dist > -EDGE_MARGIN_PX).all(0) & ~inside
            zz = lam[0] * z[0] + lam[1] * z[1] + lam[2] * z[2]
            sub_d, sub_a, sub_t = depth[y0:y1 + 1, x0:x1 + 1], ambiguous[y0:y1 + 1, x0:x1 + 1], tol[y0:y1 + 1, x0:x1 + 1]
            if facing < FACING_MARGIN:  # nearly edge-on: the raster's winding decision is the snapped area's sign
                sub_a |= inside | near
                continue
            win = inside & (zz >= 0) & (zz <= 1)
            sub_a |= near
            close = win & np.isfinite(sub_d) & (np.abs(zz - sub_d) <= 1e-4 * np.abs(zz))
            sub_a |= close
            # moving a vertex by the snap (1/512 pixel per axis) tilts the plane by about its depth range over its least altitude
            t_snap = DEPTH_RTOL * np.abs(zz) + (z.max() - z.min()) * (2.0 / 512.0) / max(abs(area) / max(lens), 1e-9)
            upd = win & (zz > sub_d)
            sub_d[upd] = zz[upd]
            sub_t[upd] = t_snap[upd] if np.ndim(t_snap) else t_snap
    return depth, ambiguous, tol


CASES = [("aerial", 4.0, (4, 4), 24, "noise"), ("grazing", 2.0, (3, 5), 32, "noise"), ("aerial", 1.0, (2, 2), 16, "rough"),
         ("grazing", 8.0, (6, 6), 48, "noise")]


@pytest.mark.parametrize("view,target,grid,res,kind", CASES, ids=[f"{c[0]}-{c[1]}-{c[4]}" for c in CASES])
def test_oracle_against_binary64_restatement(so, view, target, grid, res, kind):
    w, h = 96, 64
    hm = ht.heightmap(res, res, grid[0] * 7 + grid[1], kind, texel_noise=0.02)
    t = ht.terrain(grid, (80.0, 60.0), (0.0, 10.0))
    st = ht.settings(t, target)
    if view == "aerial":
        cam = ht.views(hm, t, w, h)["aerial"]
    else:  # low over the terrain's near edge, looking across it: no triangle reaches behind the camera (the restatement does not clip)
        cx, cz = float(t["world_min"][0][0]) + 40.0, float(t["world_min"][0][1]) + 60.0
        cam = ht.camera(w, h, (cx, 14.0, cz + 4.0), (cx, 0.0, cz - 60.0))
    n = grid[0] * grid[1]
    kept, patches, skipped = [], [], 0
    for idx in range(n):
        tris, corners = _patch_triangles(hm, t, st, cam, idx)
        if tris is None:
            skipped += 1
            continue
        assert len(tris) == so.patch(hm, st, cam, idx).triangles, idx
        kept.append(idx)
        patches.append((tris, corners))
    assert skipped <= n // 4
    vis = np.full((h, w), CLEAR, np.uint64)
    so.draw_terrain(hm, st, np.array(kept, np.uint32), len(kept), cam, vis)
    got_cov = vis != CLEAR
    got = (vis >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)
    want, ambiguous, tol = _raster(hm, t, st, cam, patches, w, h)
    want_cov = np.isfinite(want)
    compared = ~ambiguous
    assert ambiguous.mean() <= 0.15, ambiguous.mean()
    assert (got_cov[compared] == want_cov[compared]).all(), np.argwhere(compared & (got_cov != want_cov))[:5].tolist()
    both = compared & got_cov
    assert both.sum() > 500
    bad = both & ~(np.abs(got - want) <= tol)
    assert not bad.any(), [(tuple(i), got[tuple(i)], want[tuple(i)]) for i in np.argwhere(bad)[:5]]
