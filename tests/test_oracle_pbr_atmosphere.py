"""The atmospheric PBR apply's oracle (oracle/oxc_oracle_pbr_atmosphere.c) pinned by hand: the constant bits and the near fade-out's
binary32 fold, the binary32 per_slice_depth, the sun disc on both sides of min_cos, cube face selection with ties, edge and corner
remaps, NaN and zero directions, the 3D tap, the early returns, the round trip of every cube texel through the IBL's face directions,
and the reduction to orc_apply_pbr under a unit transmittance, a clear aerial LUT and a constant cube."""
import numpy as np
import pytest

from oxylus_b200 import abi
from tests.test_gpu_pbr import mixed_lights, random_planes

F = np.float32


@pytest.fixture(scope="module")
def pa():
    import pyoracle_pbr_atmosphere

    pyoracle_pbr_atmosphere.build()
    return pyoracle_pbr_atmosphere


def bits(x):
    return int(np.float32(x).view(np.uint32))


def small_atmosphere(ap=(8, 6, 4)):
    return abi.atmosphere(transmittance_lut_size=(16, 8, 1), sky_view_lut_size=(12, 10, 1), aerial_perspective_lut_size=(*ap, 1)[:3]
                          if len(ap) == 2 else ap)


def random_sky(rng, at, hostile=False):
    """float16 transmittance, sky-view, aerial-perspective LUTs and a cube for the record's sizes; hostile ones carry NaN, Inf,
    subnormal and negative texels"""
    t, s, a = at.transmittance_lut_size, at.sky_view_lut_size, at.aerial_perspective_lut_size
    planes = [rng.uniform(0, 1, (t[1], t[0], 4)), rng.uniform(0, 2, (s[1], s[0], 4)), rng.uniform(0, 1, (a[2], a[1], a[0], 4)),
              rng.uniform(0, 1.5, (6, 32, 32, 4))]
    planes = [p.astype(np.float16) for p in planes]
    if hostile:
        bad = np.float16([np.nan, np.inf, -np.inf, 6e-8, -1.0, 65504.0])
        for p in planes:
            m = rng.random(p.shape) < 0.03
            p[m] = rng.choice(bad, int(m.sum()))
    return planes


def test_constant_bits(pa):
    """the bits of the constants the oracle's pass reads (tests/test_pbr_atmosphere_source_cpu.py pins the kernel's to the same), and
    that they are the binary32 folds of the shader's literals"""
    arg, min_cos, half_slice, fade = (int(b) for b in pa.pass_constants().view(np.uint32))
    assert arg == 0x3C8EFA35 == bits(F(F(1.0) * F(np.pi)) / F(180.0))
    assert min_cos == bits(np.cos(np.float64(np.uint32(arg).view(np.float32)))) == 0x3F7FF605
    assert half_slice == 0x3F3504F3 == bits(np.sqrt(0.5))
    assert fade == 0x4479FFFF == bits(F(1.0) / F(0.001))  # fl(1 / fl(0.001)): the binary32 fold
    assert bits(1.0 / 0.001) == 0x447A0000  # what a binary64 fold would give


def test_sun_disc_both_sides(pa):
    min_cos = pa.pass_constants()[1]
    assert pa.draw_sun(min_cos) == 1.0 and pa.draw_sun(1.0) == 1.0
    below = np.nextafter(min_cos, F(0))
    off = F(min_cos - below)
    want = F(F(np.exp(np.float64(F(-off * F(50000))))) * F(0.5)) + F(F(F(1) / F(F(0.02) + F(off * F(300)))) * F(0.01))
    assert abs(float(pa.draw_sun(below)) - float(want)) <= 2e-7
    assert pa.draw_sun(-1.0) < 0.02 and np.isnan(pa.draw_sun(np.nan))


def test_per_slice_depth_is_a_binary32_division(pa):
    """32 x 32 x 24: f32(32) / f32(24) = 1.3333334, where the LUT pass's integer division gives 1; the aerial sample's w follows it"""
    at = abi.atmosphere(aerial_perspective_lut_size=(32, 32, 24), aerial_perspective_start_km=0.0, aerial_perspective_exposure=1.0)
    lut = np.zeros((24, 32, 32, 4), np.float16)
    lut[..., 3] = 1.0
    lut[..., 0] = np.arange(24, dtype=np.float16)[:, None, None]  # slice index in red
    d = np.float32([0.0, 0.0, 6.0])
    out = pa.aerial(at, lut, 0.5, 0.5, d)
    psd = F(32) / F(24)
    w = np.sqrt(F(F(F(6) * F(F(1) / psd)) * F(F(1) / F(24))), dtype=np.float32)
    z = F(F(w * F(24)) - F(0.5))
    assert out[0] == pytest.approx(float(z), abs=2e-6)
    w_int = np.sqrt(F(F(6) / F(24)), dtype=np.float32)  # per_slice_depth 1
    assert abs(float(F(F(w_int * F(24)) - F(0.5))) - float(out[0])) > 0.3


def test_tap3_is_bilinear_then_z(pa):
    at = small_atmosphere()
    rng = np.random.default_rng(5)
    lut = rng.uniform(0, 1, (4, 6, 8, 4)).astype(np.float16)
    u, v, w = F(0.37), F(0.61), F(0.55)
    z = F(F(w * F(4)) - F(0.5))
    z0 = np.floor(z)
    wz = F(z - z0)

    def bil(sl):
        x, y = F(F(u * F(8)) - F(0.5)), F(F(v * F(6)) - F(0.5))
        x0, y0 = np.floor(x), np.floor(y)
        wx, wy = F(x - x0), F(y - y0)
        a = sl.astype(np.float32)
        t = lambda i, j: a[min(max(int(j), 0), 5), min(max(int(i), 0), 7)]
        top = t(x0, y0) + F(wx) * (t(x0 + 1, y0) - t(x0, y0))
        bot = t(x0, y0 + 1) + F(wx) * (t(x0 + 1, y0 + 1) - t(x0, y0 + 1))
        return (top + wy * (bot - top)).astype(np.float32)

    s0, s1 = bil(lut[int(z0)]), bil(lut[int(z0) + 1])
    want = (s0 + wz * (s1 - s0)).astype(np.float32)
    np.testing.assert_array_equal(pa.tap3(at, lut, u, v, w), want)


@pytest.mark.parametrize("r,face", [((1, 0.5, -0.2), 0), ((-1, 0.5, 0.2), 1), ((0.1, 1, 0.3), 2), ((0.1, -1, 0.3), 3), ((0.2, 0.1, 1), 4),
                                    ((0.2, 0.1, -1), 5), ((1, 1, 1), 0), ((-1, 1, 1), 1), ((0, 1, 1), 2), ((0, -1, -1), 3), ((0, 0, -0.0), 0),
                                    ((-0.0, 0, 0), 0), ((np.nan, 0, 0), 2), ((0, np.nan, 1), 4), ((1, np.nan, 0), 4),
                                    ((np.nan, np.nan, np.nan), 5)])
def test_face_selection_and_ties(pa, r, face):
    assert pa.cube_face(r)[0] == face


def test_edge_and_corner_remaps(pa):
    idx = lambda f, x, y: (f * 32 + y) * 32 + x
    # +X (face 0) left of x = 0 is +Z's right column; above y = 0 is +Y's right column
    assert pa.cube_remap(0, -1, 5) == idx(4, 31, 5)
    assert pa.cube_remap(0, 32, 5) == idx(5, 0, 5)
    assert pa.cube_remap(0, 7, -1) == idx(2, 31, 24)
    assert pa.cube_remap(2, 7, -1) == idx(5, 24, 0)
    assert pa.cube_remap(4, 32, 9) == idx(0, 0, 9)
    # every edge texel's remap is a true neighbour: its direction lies within two texels of the off-face texel's direction
    for f in range(6):
        for k in range(32):
            for (i, j) in ((-1, k), (32, k), (k, -1), (k, 32)):
                t = pa.cube_remap(f, i, j)
                nf, ny, nx = t // 1024, (t // 32) % 32, t % 32
                assert nf != f
                # the remap is an involution through the shared edge
                back = {(-1, ny), (32, ny), (nx, -1), (nx, 32)}
                assert any(pa.cube_remap(nf, a, b) == idx(f, min(max(i, 0), 31), min(max(j, 0), 31)) for a, b in back)
    # a corner: the mean of the three texels that meet there
    cube = np.zeros((6, 32, 32, 4), np.float16)
    cube[0, 0, 0] = (3, 3, 3, 1)
    cube.reshape(-1, 4)[pa.cube_remap(0, -1, 0)] = (6, 6, 6, 1)
    cube.reshape(-1, 4)[pa.cube_remap(0, 0, -1)] = (9, 9, 9, 1)
    corner_dir = np.float32([1.0, 1.0, 1.0])  # +X wins the tie; s = t = 0: x = y = -0.5, the corner texel at weight 1/4
    out = pa.cube_tap(cube, corner_dir)
    assert out[0] == pytest.approx((3 + 6 + 9 + 6) / 4, abs=1e-5)


def test_nan_and_zero_directions(pa):
    cube = np.ones((6, 32, 32, 4), np.float16)
    for r in ((0, 0, 0), (np.nan, np.nan, np.nan), (np.inf, np.inf, 0)):
        assert np.isnan(pa.cube_tap(cube, r)).all()


def test_round_trip_every_texel(pa):
    import pyoracle_sky_ibl

    rng = np.random.default_rng(11)
    cube = rng.uniform(0.0, 4.0, (6, 32, 32, 4)).astype(np.float16)
    worst = 0.0
    for f in range(6):
        for y in range(32):
            for x in range(32):
                d = pyoracle_sky_ibl.direction(f, x, y)
                assert pa.cube_face(d)[0] == f
                got = pa.cube_tap(cube, d)
                worst = max(worst, float(np.abs(got - cube[f, y, x].astype(np.float32)).max()))
    assert worst < 1e-4


def test_early_returns(pa):
    at = small_atmosphere()
    rng = np.random.default_rng(3)
    pcam, planes = random_planes(rng, 16, 8)
    sky = random_sky(rng, at)
    s = abi.pbr_settings(scene_flags=abi.SCENE_HAS_ATMOSPHERE | abi.SCENE_TRANSPARENT_BACKGROUND | abi.SCENE_HAS_SKY,
                         sun_direction=(0.3, 0.8, 0.5), light_count=0)
    out = pa.apply_pbr_atmosphere(pcam, s, at, None, *[planes[k] for k in abi.PBR_INPUTS], *sky)
    sky_px = planes["depth"] == 0
    assert sky_px.any() and (out[sky_px] == 0).all() and (out[~sky_px][:, 3] == 1).all()
    s.scene_flags = abi.SCENE_HAS_ATMOSPHERE | abi.SCENE_HAS_SKY  # no HasSky early return: the sky view, alpha 1
    out = pa.apply_pbr_atmosphere(pcam, s, at, None, *[planes[k] for k in abi.PBR_INPUTS], *sky)
    assert (out[sky_px][:, 3] == 1).all() and (out[sky_px][:, :3] > 0).any()


def test_reduction_to_apply_pbr(pa):
    """unit transmittance, a high sun (horizon_darkening 1), aerial (0, 0, 0, 1) and a cube of constant c: every non-sky pixel under
    HasDirectionalLight is orc_apply_pbr with HasSky and sky_ambient c, bit for bit, except a -0 sum that the +0 aerial term makes +0"""
    import pyoracle_pbr

    at = small_atmosphere()
    rng = np.random.default_rng(21)
    pcam, planes = random_planes(rng, 48, 32)
    lights = mixed_lights(rng, 17)
    t, s_, a = at.transmittance_lut_size, at.sky_view_lut_size, at.aerial_perspective_lut_size
    c = np.float16(0.375)
    sky = [np.ones((t[1], t[0], 4), np.float16), np.ones((s_[1], s_[0], 4), np.float16),
           np.tile(np.float16([0, 0, 0, 1]), (a[2], a[1], a[0], 1)), np.tile(np.float16([c, c, c, 1]), (6, 32, 32, 1))]
    flags = abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_CONTACT_SHADOWS
    st = abi.pbr_settings(scene_flags=flags | abi.SCENE_HAS_ATMOSPHERE, sun_direction=(0.3, 0.9, 0.3), sun_intensity=7.5, light_count=17)
    ref = abi.pbr_settings(scene_flags=flags | abi.SCENE_HAS_SKY, sun_direction=(0.3, 0.9, 0.3), sun_intensity=7.5,
                           sky_ambient_color=(float(c),) * 3, light_count=17)
    args = [planes[k] for k in abi.PBR_INPUTS]
    got = pa.apply_pbr_atmosphere(pcam, st, at, lights, *args, *sky)
    want = pyoracle_pbr.apply_pbr(pcam, ref, lights, *args)
    m = planes["depth"] != 0
    g, w = got[m], want[m]
    w = np.where(w == 0, np.float32(0), w)  # -0 + +0 = +0
    np.testing.assert_array_equal(g.view(np.uint32), w.view(np.uint32))
    assert m.sum() > 1000
