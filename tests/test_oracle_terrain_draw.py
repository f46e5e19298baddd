"""Properties of the terrain-draw oracle (oracle/oxc_oracle_terrain_draw.c, include/oxcull.h oxc_draw_terrain items 1-7): the edge factors
at known distances, the odd rounding, the domain points of an edge, the exact tiling of the unit square in rationals, a flat terrain's
depth against the plane's closed form, the winding seen from above and below, the tie with a meshlet word, and watertightness across
patch borders with different factors on a noisy heightmap."""
from fractions import Fraction

import numpy as np
import pytest

from oxylus_b200 import abi
from tests import helpers_terrain as ht

CLEAR = np.uint64(0xFFFFFFFF)


@pytest.fixture(scope="module")
def so():
    import pyoracle_terrain_draw

    pyoracle_terrain_draw.build()
    return pyoracle_terrain_draw


def test_factors_at_known_distances(so):
    """one flat 16 m patch seen along -z from distance d of its near edge's centre: an edge of radius 8 whose centre lies r from the
    camera projects to 16 * scale / (r - 8) pixels — the near edge v1 at r = d, the far edge v0 at d + 16, the side edges u0, u1 at
    hypot(d + 8, 8); scale = 540 / tan(30 degrees) at 1080 rows"""
    hm = ht.heightmap(4, 4, 0, "flat")
    t = ht.terrain((1, 1), (16.0, 16.0), (0.0, 10.0))
    scale = 540.0 / np.tan(np.radians(30.0))
    assert abs(float(so.projection_scale(60.0, 1080.0)) - scale) < 1e-4 * scale
    for d in (20.0, 100.0, 700.0):
        cam = ht.camera(1920, 1080, (0.0, 0.0, 8.0 + d), (0.0, 0.0, 0.0))
        p = so.patch(hm, ht.settings(t), cam, 0)
        near = 16.0 * scale / (d - 8.0) / 16.0
        side = 16.0 * scale / (np.hypot(d + 8.0, 8.0) - 8.0) / 16.0
        far = 16.0 * scale / (d + 8.0) / 16.0
        want = [min(max(x, 1.0), 64.0) for x in (side, far, side, near)]
        np.testing.assert_allclose(list(p.factor)[:4], want, rtol=1e-5)
        assert p.factor[4] == max(p.factor[1], p.factor[3]) and p.factor[5] == max(p.factor[0], p.factor[2])


def test_odd_rounding(so):
    cases = {1.0: 1, 1.0 + 2.0**-23: 3, 3.0: 3, 3.5: 5, 63.0: 63, 64.0: 63, float("nan"): 1, 0.0: 1, -5.0: 1, float("inf"): 63}
    for f, n in cases.items():
        assert so.round_odd(f) == n, f
    assert so.factor_clamp(float("nan")) == 1.0 and so.factor_clamp(1e9) == 63.0


@pytest.mark.parametrize("f", [1.0, 1.0 + 2.0**-23, 2.5, 3.0, 3.0001, 4.9999, 7.3, 33.1, 62.5, 63.0])
def test_edge_points(so, f):
    """n + 1 points, 0 and 1 at the ends, strictly increasing, mirror images bit for bit, n - 2 equal inner segments of 1 / f and two
    equal end segments of (f - (n - 2)) / (2 f)"""
    n = so.round_odd(f)
    t = so.edge_points(so.factor_clamp(f), n)
    assert len(t) == n + 1 and t[0] == 0 and t[-1] == 1
    assert (np.diff(t) > 0).all()
    for k in range(1, n):
        assert t[k] == np.float32(1) - t[n - k] or t[n - k] == np.float32(1) - t[k]
    if n > 1:
        seg = np.diff(t.astype(np.float64))
        fc = float(so.factor_clamp(f))
        np.testing.assert_allclose(seg[1:-1], 1.0 / fc, rtol=1e-5)
        np.testing.assert_allclose([seg[0], seg[-1]], (fc - (n - 2)) / (2 * fc), rtol=1e-4, atol=1e-7)


def _tiling(tris, outer):
    """tris [k, 3, 2] float32 in the raster's order; outer = the four edges' point lists (u0, v0, u1, v1)"""
    F = [[(Fraction(float(a)), Fraction(float(b))) for a, b in tri] for tri in tris]
    area = Fraction(0)
    edges = {}
    for a, b, c in F:
        s = (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])
        assert s < 0, "every triangle reaches the raster clockwise in (u, v)"
        area += -s / 2
        for e in ((a, b), (b, c), (c, a)):
            assert e not in edges, "a directed edge used twice: overlap"
            edges[e] = 1
    assert area == 1
    boundary = {e for e in edges if (e[1], e[0]) not in edges}
    want = set()
    u0, v0, u1, v1 = [[Fraction(float(x)) for x in pts] for pts in outer]
    # clockwise around the square in (u, v): along u = 0 upwards, v = 1 rightwards, u = 1 downwards, v = 0 leftwards
    want |= {((Fraction(0), u0[k]), (Fraction(0), u0[k + 1])) for k in range(len(u0) - 1)}
    want |= {((v1[k], Fraction(1)), (v1[k + 1], Fraction(1))) for k in range(len(v1) - 1)}
    want |= {((Fraction(1), u1[k + 1]), (Fraction(1), u1[k])) for k in range(len(u1) - 1)}
    want |= {((v0[k + 1], Fraction(0)), (v0[k], Fraction(0))) for k in range(len(v0) - 1)}
    assert boundary == want


def test_domain_tiles_the_square_exactly(so):
    """patches of a noisy terrain seen from several cameras (every factor mix from the quad to 63 on all sides): the domain triangles
    tile the unit square in exact rationals — area 1, each interior edge once in each direction, the boundary edges exactly the outer
    subdivisions — with one winding, and their count is item 3's formula"""
    hm = ht.heightmap(64, 64, 4)
    t = ht.terrain((8, 8), (64.0, 64.0), (0.0, 12.0))
    seen = set()
    for target in (1.0, 4.0, 16.0, 64.0):
        for name, cam in ht.views(hm, t, 640, 360).items():
            for idx in (0, 9, 27, 36, 63):
                p = so.patch(hm, ht.settings(t, target), cam, idx)
                tris = so.patch_domain(p)
                assert len(tris) == p.triangles
                outer = [so.edge_points(p.pinned[k], p.n[k]) for k in range(4)]
                _tiling(tris, outer)
                seen.add(tuple(p.n))
    ns = {n for key in seen for n in key}
    assert 1 in ns and 3 in ns and 63 in ns and len(seen) > 10


def test_flat_terrain_depth_and_winding(so):
    """a flat terrain at height 3 seen from above: straight down every pixel is written, obliquely most are; each written pixel holds
    the terrain's word and the plane's depth (the ray through the pixel centre meets y = 3) within binary32 error; seen from below
    nothing is written"""
    w, h = 96, 64
    hm = ht.heightmap(8, 8, 0, "flat")
    t = ht.terrain((4, 4), (400.0, 400.0), (3.0, 10.0))
    st = ht.settings(t, 4.0)
    vis_all = np.arange(16, dtype=np.uint32)
    for eye, center in (((0.0, 60.0, 5.0), (0.0, 3.0, 0.0)), ((10.0, 40.0, 30.0), (-5.0, 3.0, -20.0))):
        cam = ht.camera(w, h, eye, center)
        vis = np.full((h, w), CLEAR, np.uint64)
        so.draw_terrain(hm, st, vis_all, 16, cam, vis)
        drawn = (vis != CLEAR).ravel()
        assert drawn.all() if eye[0] == 0.0 else drawn.mean() > 0.5
        assert ((vis.ravel()[drawn] & CLEAR) == 0xFFFFFE00).all()
        M = cam["projection_view"][0].reshape(4, 4).T.astype(np.float64)
        inv = np.linalg.inv(M)
        ys, xs = np.mgrid[0:h, 0:w]
        xn, yn = (xs + 0.5) / w * 2 - 1, (ys + 0.5) / h * 2 - 1
        A = inv @ np.stack([xn.ravel(), yn.ravel(), np.zeros(xn.size), np.ones(xn.size)])
        B = inv[:, 2:3]
        z = (3.0 * A[3] - A[1]) / (B[1] - 3.0 * B[3])
        got = (vis >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64).ravel()
        np.testing.assert_allclose(got[drawn], z[drawn], rtol=2e-4, atol=1e-7)
    below = ht.camera(w, h, (0.0, -50.0, 5.0), (0.0, 3.0, 0.0))
    vis = np.full((h, w), CLEAR, np.uint64)
    assert so.draw_terrain(hm, st, vis_all, 16, below, vis) > 0
    assert (vis == CLEAR).all()


def test_terrain_wins_depth_ties(so):
    """over a meshlet word of the same depth the terrain's word wins (the packed max), nearer meshlet words stay, in both packings"""
    w, h = 64, 48
    hm = ht.heightmap(16, 16, 2)
    t = ht.terrain((2, 2), (64.0, 64.0), (0.0, 8.0))
    cam = ht.views(hm, t, w, h)["aerial"]
    alone = np.full((h, w), CLEAR, np.uint64)
    so.draw_terrain(hm, ht.settings(t, 4.0), np.arange(4, dtype=np.uint32), 4, cam, alone)
    drawn = alone != CLEAR
    assert drawn.sum() > 100
    for bits, word in ((8, 0xFFFFFE00), (6, 0xFFFFFF80)):
        depth = alone >> np.uint64(32)
        start = np.where(drawn, (depth << np.uint64(32)) | np.uint64(((0xFFFFFFFF >> bits) - 2) << bits), CLEAR).astype(np.uint64)
        start[::2] = np.where(drawn[::2], ((depth[::2] + np.uint64(1)) << np.uint64(32)) | np.uint64(5 << bits), CLEAR)
        vis = start.copy()
        so.draw_terrain(hm, ht.settings(t, 4.0), np.arange(4, dtype=np.uint32), 4, cam, vis, bits)
        assert ((vis[1::2][drawn[1::2]] & CLEAR) == word).all()
        assert (vis[::2] == start[::2]).all()


@pytest.mark.parametrize("target", [1.0, 6.0, 24.0])
def test_watertight(so, target):
    """a noisy heightfield seen from above, straight down and obliquely, with patch factors that differ across every border: every pixel
    whose ray passes through the prism of the (slightly shrunk) terrain rectangle between its highest and lowest height is written"""
    w, h = 200, 150
    hm = ht.heightmap(48, 48, 8)
    t = ht.terrain((6, 6), (60.0, 60.0), (0.0, 6.0))
    st = ht.settings(t, target)
    lo, hi = float(hm.min()) / 65535 * 6.0, float(hm.max()) / 65535 * 6.0
    written_total, factors = 0, set()
    for eye, center in (((0.0, 55.0, 0.1), (0.0, 0.0, 0.0)), ((8.0, 30.0, 35.0), (0.0, 0.0, -2.0)), ((-20.0, 18.0, 20.0), (2.0, 0.0, -3.0))):
        cam = ht.camera(w, h, eye, center)
        vis = np.full((h, w), CLEAR, np.uint64)
        so.draw_terrain(hm, st, np.arange(36, dtype=np.uint32), 36, cam, vis)
        factors |= {so.patch(hm, st, cam, i).n[k] for i in range(36) for k in range(4)}
        M = cam["projection_view"][0].reshape(4, 4).T.astype(np.float64)
        inv = np.linalg.inv(M)
        ys, xs = np.mgrid[0:h, 0:w]
        xn, yn = (xs + 0.5) / w * 2 - 1, (ys + 0.5) / h * 2 - 1
        inside = np.ones((h, w), bool)
        for y in (lo, hi):
            A = inv @ np.stack([xn.ravel(), yn.ravel(), np.zeros(xn.size), np.ones(xn.size)])
            B = inv[:, 2:3]
            z = (y * A[3] - A[1]) / (B[1] - y * B[3])
            P = A + z * B
            px, pz = (P[0] / P[3]).reshape(h, w), (P[2] / P[3]).reshape(h, w)
            inside &= (np.abs(px) < 29.5) & (np.abs(pz) < 29.5) & (z.reshape(h, w) > 0)
        assert inside.sum() > 1000
        holes = inside & (vis == CLEAR)
        assert not holes.any(), f"{holes.sum()} holes, first at {np.argwhere(holes)[:3].tolist()}"
        written_total += int((vis != CLEAR).sum())
    assert written_total > 0 and len(factors) > 1


def test_instance_count_and_bad_indices(so):
    """the count is clamped to the patch total; slots holding an index past it draw nothing"""
    w, h = 64, 48
    hm = ht.heightmap(16, 16, 3)
    t = ht.terrain((2, 2), (32.0, 32.0), (0.0, 4.0))
    cam = ht.views(hm, t, w, h)["aerial"]
    st = ht.settings(t, 2.0)
    ref = np.full((h, w), CLEAR, np.uint64)
    n_ref = so.draw_terrain(hm, st, np.arange(4, dtype=np.uint32), 4, cam, ref)
    two = np.full((h, w), CLEAR, np.uint64)
    n_two = so.draw_terrain(hm, st, np.array([0, 1], np.uint32), 2, cam, two)
    vis = np.full((h, w), CLEAR, np.uint64)
    n = so.draw_terrain(hm, st, np.array([0, 4, 1, 0xFFFFFFFF, 2, 3], np.uint32), 6, cam, vis)  # slots 4 and 5 lie past the total
    assert n == n_two and (vis == two).all() and n_two < n_ref
    vis = np.full((h, w), CLEAR, np.uint64)
    assert so.draw_terrain(hm, st, np.arange(4, dtype=np.uint32), 1 << 30, cam, vis) == n_ref and (vis == ref).all()
    assert abi.TERRAIN_DRAW_SETTINGS_DT.itemsize == 52
