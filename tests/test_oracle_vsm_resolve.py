"""The VSM shadow-resolve specification (oracle/oxc_oracle_vsm_resolve.c) pinned by hand: sky, misses, cleared atlas, a blocker, the
clipmap fall-back order, an out-of-atlas read, the helpers' known answers, the PCSS penumbra, and the canonical sin / cos bound."""
import os
import sys

import numpy as np
import pytest

from oxylus_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

B = abi.VSM_PAGE_BACKED
L = np.float32([0.0, -1.0, 0.0])  # straight down: the clipmaps below look along -y


@pytest.fixture(scope="module")
def vr():
    import pyoracle_vsm_resolve

    pyoracle_vsm_resolve.build()
    return pyoracle_vsm_resolve


def ortho_down(half_width, z_range=200.0):
    """column-major PV of a light looking straight down (-y) at the origin: x -> clip x, z -> clip y, depth = (100 - y) / z_range"""
    m = np.zeros((4, 4), np.float32)  # row-major rows
    m[0, 0] = 1.0 / half_width
    m[1, 2] = 1.0 / half_width
    m[2, 1] = -1.0 / z_range
    m[2, 3] = 100.0 / z_range
    m[3, 3] = 1.0
    return m.T.reshape(16)


def setup(size=4, page_size=8, atlas=32, layers=3, w=4, h=4, first_width=10.0):
    """a camera looking straight down at the ground y = 0 (orthographic, 4 x 4 pixels over [-2, 2]^2), clipmaps of half width
    first_width * 2^k, every page table entry Backed on physical page 0"""
    vsm = np.zeros(1, dtype=abi.VSM_CONTEXT_DT)
    vsm["page_size"], vsm["page_table_size"], vsm["physical_page_table_size"], vsm["clipmap_count"] = page_size, size, atlas, layers
    vsm["depth_extent"][0] = (w, h)
    vsm["first_clipmap_width"], vsm["clipmap_selection_bias"], vsm["virtual_extent"], vsm["z_length"] = first_width, 0.0, float(atlas), 200.0
    vsm["directional_light_dir"][0] = L
    cm = np.zeros(layers, dtype=abi.CLIPMAP_DT)
    for k in range(layers):
        cm["projection_view_mat"][k] = ortho_down(first_width * 2 ** k)
    # camera: ndc (x, y, z) -> world (2x, 100 - 100 z, 2y): inverse PV, column-major
    ipv = np.zeros((4, 4), np.float32)
    ipv[0, 0] = 2.0
    ipv[1, 2] = -100.0
    ipv[1, 3] = 100.0
    ipv[2, 1] = 2.0
    ipv[3, 3] = 1.0
    depth = np.ones((h, w), np.float32)  # y = 0
    normals = np.zeros((h, w, 4), np.float32)
    normals[..., 2:] = oct_encode(np.float32([0.0, 1.0, 0.0]))
    pt = np.full((layers, size, size), B, np.uint32)
    return vsm, ipv.T.reshape(16), np.float32([w, h]), cm, depth, normals, pt


def oct_encode(v):
    v = np.asarray(v, np.float64)
    p = v[:2] / np.abs(v).sum()
    if v[2] <= 0:
        return np.float32([(1 - abs(p[1])) * (1 if p[0] >= 0 else -1), (1 - abs(p[0])) * (1 if p[1] >= 0 else -1)])
    return np.float32(p)


def test_sky_is_lit(vr):
    vsm, ipv, res, cm, depth, normals, pt = setup()
    depth[:] = 0.0
    s, pcf = vr.vsm_resolve_shadows(vsm, ipv, res, cm, depth, normals, pt, np.zeros((32, 32), np.float32))
    assert (s == 1.0).all() and not pcf.any()


def test_no_backed_page_is_the_hard_shadow(vr):
    vsm, ipv, res, cm, depth, normals, pt = setup()
    pt[:] = 0
    s, _ = vr.vsm_resolve_shadows(vsm, ipv, res, cm, depth, normals, pt, np.zeros((32, 32), np.float32))
    assert (s == 1.0).all()


def test_cleared_atlas_is_lit(vr):
    vsm, ipv, res, cm, depth, normals, pt = setup()
    s, _ = vr.vsm_resolve_shadows(vsm, ipv, res, cm, depth, normals, pt, np.ones((32, 32), np.float32))
    assert (s == 1.0).all()


def test_uniform_blocker_above_is_shadowed(vr):
    vsm, ipv, res, cm, depth, normals, pt = setup()
    # receiver y = 0 at depth 0.5; a blocker at y = 50 has depth 0.25
    s, _ = vr.vsm_resolve_shadows(vsm, ipv, res, cm, depth, normals, pt, np.full((32, 32), 0.25, np.float32))
    assert (s == 0.0).all()


def test_unbacked_base_page_falls_back_below_then_above(vr):
    """with the base clipmap's pages unbacked, the taps read clipmap base - 1 first and base + 1 only when that misses too"""
    vsm, ipv, res, cm, depth, normals, pt = setup(layers=4, page_size=8, atlas=32)
    atlas = np.ones((32, 32), np.float32)
    atlas[:8, :8] = 0.25  # physical page 0: a blocker; page 1: lit
    base = 2  # the 1-unit pixel footprint over a 0.47-unit first texel: ceil(log2(2.13)) = 2
    pt[:] = B | (1 << 16)  # everything on the lit page
    s0, _ = vr.vsm_resolve_shadows(vsm, ipv, res, cm, depth, normals, pt, atlas)
    assert (s0 == 1.0).all()
    pt[base - 1] = B       # clipmap base - 1 on the blocker page
    pt[base] = 0
    s1, _ = vr.vsm_resolve_shadows(vsm, ipv, res, cm, depth, normals, pt, atlas)
    assert (s1 == 0.0).all()  # clipmap base - 1 is read: shadowed
    pt[base - 1] = 0
    pt[base + 1] = B
    s2, _ = vr.vsm_resolve_shadows(vsm, ipv, res, cm, depth, normals, pt, atlas)
    assert (s2 == 0.0).all()  # clipmap 2 is read only when clipmap 0 misses
    pt[base + 1] = B | (1 << 16)
    s3, _ = vr.vsm_resolve_shadows(vsm, ipv, res, cm, depth, normals, pt, atlas)
    assert (s3 == 1.0).all()


def test_out_of_atlas_address_reads_zero(vr):
    """a Backed entry whose physical page lies beyond the atlas reads 0.0: the receiver is shadowed (0 < its depth)"""
    vsm, ipv, res, cm, depth, normals, pt = setup()
    pt[:] = B | (40 << 16)  # 16 physical pages: page 40 is outside
    s, _ = vr.vsm_resolve_shadows(vsm, ipv, res, cm, depth, normals, pt, np.ones((32, 32), np.float32))
    assert (s == 0.0).all()


def test_helper_known_answers(vr):
    assert list(vr.hammersley2d(0, 16)) == [0.0, 0.0]
    assert list(vr.hammersley2d(1, 16)) == [0.0625, 0.5]
    assert list(vr.hammersley2d(3, 24)) == [np.float32(3) / np.float32(24), 0.75]
    assert list(vr.hammersley2d(6, 16)) == [0.375, 0.375]
    # hash2: fract(sin(dot) * 43758.5453) in binary32 with the canonical sin
    for px, py in ((0.5, 0.5), (1919.5, 1079.5), (3839.5, 2159.5)):
        d0 = np.float32(np.float32(px) * np.float32(127.1)) + np.float32(np.float32(py) * np.float32(311.7))
        s = np.float32(np.sin(np.float64(d0)))
        want = np.float32(s * np.float32(43758.5453))
        got = vr.hash2(px, py)
        assert abs(float(got[0]) - float(want - np.floor(want))) < 1e-2 or abs(abs(float(got[0]) - float(want - np.floor(want))) - 1) < 1e-2
        assert 0.0 <= got[0] <= 1.0 and 0.0 <= got[1] <= 1.0
    assert list(vr.hash2(0.5, 0.5)) == [np.float32(0.7050781), np.float32(0.63378906)]
    # perpendicular_basis: |L.y| < 0.999 crosses with +y, else with +x
    t, b = vr.perpendicular_basis([0.0, -1.0, 0.0])  # cross(+x, L) = (0, 0, -1), cross(L, t) = (1, 0, 0)
    np.testing.assert_array_equal(t, np.float32([0.0, 0.0, -1.0]))
    np.testing.assert_array_equal(b, np.float32([1.0, 0.0, 0.0]))
    t, b = vr.perpendicular_basis([1.0, 0.0, 0.0])
    np.testing.assert_array_equal(t, np.float32([0.0, 0.0, -1.0]))
    np.testing.assert_array_equal(b, np.float32([0.0, 1.0, 0.0]))
    # base_bias: (quantize + b) + term, b = sqrt2 * texel * 0.5; NoL >= 0.99 -> term = b
    vsm, *_ = setup()
    texel = np.float32(np.float32(np.float32(10.0) * (np.float32(3) / np.float32(4))) * np.float32(2.0)) / np.float32(32.0)
    cts = np.float32(2.0) * texel
    bb = np.float32(np.float32(np.float32(1.41421356) * cts) * np.float32(0.5))
    assert vr.base_bias(vsm, 0, [0.0, -1.0, 0.0]) == np.float32(np.float32(np.float32(2.0 ** -22) + bb) + bb)
    # NoL = 0.6 (normal (0.8, -0.6, 0)): term = b * |N x L| / NoL = b * 0.8 / 0.6
    n = np.float32([0.8, -0.6, 0.0])
    nol = np.float32(0.6)
    cr = np.float32(np.sqrt(np.float32(np.float32(0.8) * np.float32(0.8))))
    term = np.float32(np.float32(bb * cr) / nol)
    assert vr.base_bias(vsm, 0, n) == np.float32(np.float32(np.float32(2.0 ** -22) + bb) + term)
    assert vr.round_to_half(1.0 + 2.0 ** -11) == 1.0 and vr.round_to_half(1.0 + 3 * 2.0 ** -11) == np.float32(1.0 + 2.0 ** -9)
    assert vr.round_to_half(65520.0) == np.inf and vr.round_to_half(2.0 ** -25) == 0.0 and vr.round_to_half(3 * 2.0 ** -26) == np.float32(2.0 ** -24)


def test_pcss_penumbra_widens_with_blocker_distance(vr):
    """a half-plane blocker (x < 0 in light space) over the receiver: 0 deep in its shadow, 1 far outside, a band in (0, 1) across the
    edge, wider when the blocker is further from the receiver"""
    w = 256
    widths = []
    for blocker_y in (20.0, 90.0):
        vsm, ipv, res, cm, depth, normals, pt = setup(size=8, page_size=64, atlas=512, layers=1, w=w, h=1, first_width=4.0)
        ipv = ipv.reshape(4, 4).T.copy()
        ipv[0, 0] = 2.0  # x over [-2, 2]
        ipv[2, 1] = 0.0
        vsm["first_clipmap_width"], vsm["virtual_extent"] = 4.0, 512.0
        pt[0] = B | (np.arange(64, dtype=np.uint32).reshape(8, 8) << 16)  # virtual page (x, y) -> physical page y * 8 + x
        depth = np.ones((1, w), np.float32)
        normals = np.zeros((1, w, 4), np.float32)
        normals[..., 2:] = oct_encode([0.0, 1.0, 0.0])
        # atlas texel (tx, ty): world x = (tx + 0.5) / 512 * 8 - 4; blocker for x < 0 at depth (100 - blocker_y) / 200
        tx = np.arange(512)
        wx = (tx + 0.5) / 512 * 8 - 4
        atlas = np.ones((512, 512), np.float32)
        atlas[:, wx < 0] = np.float32((100.0 - blocker_y) / 200.0)
        s, pcf = vr.vsm_resolve_shadows(vsm, ipv.T.reshape(16), np.float32([w, 1]), cm, depth, normals, pt, atlas)
        s = s[0]
        assert s[0] == 0.0 and s[-1] == 1.0
        band = (s > 0) & (s < 1)
        assert band.sum() > 0 and pcf[0][band].all()
        widths.append(int(band.sum()))
    assert widths[1] > widths[0], widths


def test_canonical_sincos_error_bound(vr):
    """every binary32 in [0, 2 pi] within 1 ulp of binary64 sin / cos; 10^6 random arguments over the whole bounded range [0, 2^21]
    (hash2's arguments reach 1.43e6 at 3840 x 2160) and every 64th binary32 up to 2^21 within 2^-24 absolute"""
    two_pi = np.float32(2 * np.pi).view(np.uint32)
    err = vr.sincos_error_scan(0, int(two_pi))
    assert err[2] <= 1.0 and err[3] <= 1.0, err
    assert err[0] <= 2.0 ** -24 and err[1] <= 2.0 ** -24, err
    x = np.random.default_rng(3).uniform(0, 2.0 ** 21, 1000000).astype(np.float32)
    err = vr.sincos_error_list(x)
    assert err[0] <= 2.0 ** -24 and err[1] <= 2.0 ** -24, err
    s = np.array([vr.sincos(v)[0] for v in x[:2000]], np.float32)  # the wrapper against numpy directly
    assert np.abs(s.astype(np.float64) - np.sin(x[:2000].astype(np.float64))).max() <= 2.0 ** -24
    err = vr.sincos_error_scan(int(two_pi), int(np.float32(2.0 ** 21).view(np.uint32)), 64)
    assert err[0] <= 2.0 ** -24 and err[1] <= 2.0 ** -24, err
