"""Properties of the tonemap's specification (oracle/oxc_oracle_tonemap.c, include/oxcull.h oxc_tonemap items 1-10), pinned by hand:
the identity, the ranges of ACES and GT7 (and that AgX has none), the vignette's centre and the identities at amount 0, the constant
table against a host binary32 recomputation written from tonemap.slang, the zero-divisor film grain at the component's 0.7, and the
Repeat wrap of the taps."""
import numpy as np
import pytest

from oxylus_b200 import abi
from tests.test_gpu_post import hdr_frame, hostile_frame

F = np.float32
EA, BL = abi.SCENE_HAS_EYE_ADAPTATION, abi.SCENE_HAS_BLOOM
CA, VG, FG, TB = abi.SCENE_HAS_CHROMATIC_ABERRATION, abi.SCENE_HAS_VIGNETTE, abi.SCENE_HAS_FILM_GRAIN, abi.SCENE_TRANSPARENT_BACKGROUND


@pytest.fixture(scope="module")
def so():
    import pyoracle_tonemap

    pyoracle_tonemap.build()
    return pyoracle_tonemap


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_none_is_the_identity(so):
    """NONE at exposure 1 without bloom or lens: the frame itself where u * W - 0.5 is exactly x (power-of-two extents), within one
    rounding of a neighbour blend elsewhere; alpha is 1, or the frame's under TransparentBackground"""
    rng = np.random.default_rng(1)
    frame = hdr_frame(rng, 64, 32)
    out = so.tonemap(frame, abi.tonemap_settings(0, abi.TONEMAP_NONE))
    np.testing.assert_array_equal(bits(out[..., :3]), bits(frame[..., :3]))
    assert (out[..., 3] == 1.0).all()
    out = so.tonemap(frame, abi.tonemap_settings(TB, abi.TONEMAP_NONE))
    np.testing.assert_array_equal(bits(out), bits(frame))
    frame = hdr_frame(rng, 17, 9)
    out = so.tonemap(frame, abi.tonemap_settings(0, abi.TONEMAP_NONE))
    np.testing.assert_allclose(out[..., :3], frame[..., :3], rtol=1e-6, atol=1e-30)


def test_curve_ranges(so):
    """ACES saturates into [0, 1]; GT7's Rec.2020 output lies in [0, 1] after the SDR correction, NaN included (min(NaN, 2.5) = 2.5);
    AgX applies its inverse matrix after the last clamp, so it has outputs outside [0, 1]"""
    rng = np.random.default_rng(2)
    c = np.concatenate([hdr_frame(rng, 64, 8)[..., :3].reshape(-1, 3), hostile_frame(rng, 16, 8)[..., :3].reshape(-1, 3)])
    aces = so.curve(abi.TONEMAP_ACES, c)
    assert ((aces >= 0) & (aces <= 1)).all()
    gt7 = so.gt7_rec2020(c)
    assert ((gt7 >= 0) & (gt7 <= 1)).all()
    agx = so.curve(abi.TONEMAP_AGX, c)
    assert np.isfinite(agx).all() and ((agx < 0) | (agx > 1)).any()
    np.testing.assert_array_equal(bits(so.curve(abi.TONEMAP_NONE, c)), bits(c))


def test_vignette_centre_and_zero_amounts(so):
    """the vignette is exactly 1 at the centre pixel; a vignette of amount 0 and a grain of amount 0 change nothing"""
    rng = np.random.default_rng(3)
    frame = rng.uniform(0.0, 1.0, (32, 64, 4)).astype(np.float32)
    base = so.tonemap(frame, abi.tonemap_settings(0, abi.TONEMAP_NONE))
    vig = so.tonemap(frame, abi.tonemap_settings(VG, abi.TONEMAP_NONE, vignette_amount=0.9))
    assert bits(vig[16, 32]).tolist() == bits(base[16, 32]).tolist()
    assert (vig[0, 0, :3] < base[0, 0, :3]).all()
    for flags, kw in ((VG, dict(vignette_amount=0.0)), (FG, dict(film_grain_amount=0.0)), (VG | FG, dict(vignette_amount=0.0, film_grain_amount=0.0))):
        np.testing.assert_array_equal(bits(so.tonemap(frame, abi.tonemap_settings(flags, abi.TONEMAP_NONE, **kw))), bits(base))


def _agx_constants():
    """tonemap.slang AgX_DS's matrices, recomputed in numpy binary32 in the shader's order"""
    def inverse(m):
        a, b, c, d, e, f, g, h, i = m.reshape(-1)
        A, B, C = e * i - f * h, -(d * i - f * g), d * h - e * g
        D, E, Fv = -(b * i - c * h), a * i - c * g, -(a * h - b * g)
        G, H, I = b * f - c * e, -(a * f - c * d), a * e - b * d
        inv = F(1) / (a * A + b * B + c * C)
        return np.array([[A * inv, D * inv, G * inv], [B * inv, E * inv, H * inv], [C * inv, Fv * inv, I * inv]], F)

    def mv(m, v):
        return np.array([(m[r, 0] * v[0] + m[r, 1] * v[1]) + m[r, 2] * v[2] for r in range(3)], F)

    def unproject(x, y):
        return np.array([(x * F(1)) / y, F(1), ((F(1) - x - y) * F(1)) / y], F)

    def primaries(r, g, b, w):
        R, G, B, W = (unproject(*p) for p in (r, g, b, w))
        s = mv(inverse(np.array([[R[0], G[0], B[0]], [1, 1, 1], [R[2], G[2], B[2]]], F)), W)
        return np.array([[R[k] * s[0], G[k] * s[1], B[k] * s[2]] for k in range(3)], F)

    xy = [(F(0.64), F(0.33)), (F(0.3), F(0.6)), (F(0.15), F(0.06))]
    w = (F(0.3127), F(0.3290))
    srgb = primaries(*xy, w)
    sf = F(1) / (F(1) - F(0.15))
    adj = primaries(*[tuple(w[k] + (p[k] - w[k]) * sf for k in range(2)) for p in xy], w)
    xyz_to_adj = inverse(adj)
    m = np.array([[(srgb[i, 0] * xyz_to_adj[0, j] + srgb[i, 1] * xyz_to_adj[1, j]) + srgb[i, 2] * xyz_to_adj[2, j] for j in range(3)]
                  for i in range(3)], F)
    return m, inverse(m)


def test_constant_table_equals_a_binary32_recomputation(so):
    k = so.constants()
    name = lambda n: k[so.CONSTANT_NAMES[n][0]: sum(so.CONSTANT_NAMES[n])]
    m, inv = _agx_constants()
    np.testing.assert_array_equal(bits(name("agx")), bits(m.reshape(-1)))
    np.testing.assert_array_equal(bits(name("agx_inv")), bits(inv.reshape(-1)))
    assert bits(name("agx_s")).tolist() == bits(F(1) * F(0.1)).reshape(1).tolist()
    assert name("agx_c")[0] == F(1) / (F(1) - F(0.1)) and name("agx_peak_s")[0] == F(1) - F(0.1)
    peak, alpha, lin = F(250) / F(100), F(0.25), F(0.444)
    kk = (lin - F(1)) / (alpha - F(1))
    assert name("gt7_ka")[0] == peak * lin + peak * kk and name("gt7_kc")[0] == F(-1) / (kk * peak)
    assert abs(float(name("gt7_kb")[0]) - float(-peak * kk) * np.exp(float(lin / kk))) < 4e-7  # canonical_exp: within 1 ulp
    assert name("gt7_linear_peak")[0] == lin * peak and name("gt7_target")[0] == peak and name("gt7_sdr")[0] == F(1) / (F(250) / F(100))
    assert name("gt7_one_minus_blend")[0] == F(1) - F(0.6)
    assert name("pq_inv_m1")[0] == F(1) / F(0.1593017578125) and name("pq_inv_m2")[0] == F(1) / F(78.84375)
    sq3 = np.sqrt(F(3))
    assert name("simplex_f2")[0] == (sq3 - F(1)) / F(2) and name("simplex_g2")[0] == (F(3) - sq3) / F(6)
    # the target's UCS intensity: ICtCp I of (2.5, 2.5, 2.5) (l = m = s = 2.5 exactly), against binary64 PQ
    y = 2.5 * 100 / 10000
    ym = y ** 0.1593017578125
    pq = 2 ** (78.84375 * (np.log2(0.8359375 + 18.8515625 * ym) - np.log2(1 + 18.6875 * ym)))
    assert abs(float(name("gt7_target_ucs")[0]) - pq) < 1e-5


def test_zero_divisor_film_grain(so):
    """scale 0.7 (the component's default): (i32)(0.7 / 8) = 0, so every pixel hashes the quotient -1 (all ones) with the seed: the
    grain then depends on the pixel only through coord / scale; equal to an explicit 0xFFFFFFFF quotient restated here"""
    frame = np.full((6, 10, 4), 0.5, np.float32)
    s = abi.tonemap_settings(FG, abi.TONEMAP_NONE, film_grain_scale=0.7, film_grain_amount=0.6, film_grain_seed=5)
    out = so.tonemap(frame, s)
    k = so.constants()

    def pcg(v):
        v = [(x * 12829 + 47989) & 0xFFFFFFFF for x in v]
        for _ in range(2):
            v[0] = (v[0] + v[1] * v[2]) & 0xFFFFFFFF
            v[1] = (v[1] + v[2] * v[0]) & 0xFFFFFFFF
            v[2] = (v[2] + v[0] * v[1]) & 0xFFFFFFFF
        return [x >> 16 for x in v]

    h = pcg([0xFFFFFFFF, 0xFFFFFFFF, 5])
    r = [F(F(h[0]) * F(2.0 ** -16)) - F(0.5), F(F(h[1]) * F(2.0 ** -16)) - F(0.5)]
    for y in range(6):
        for x in range(10):
            p = [F(F(x) / F(0.7)) + r[0], F(F(y) / F(0.7)) + r[1]]
            u = (p[0] + p[1]) * k[31]
            pi = [np.rint(p[0] + u), np.rint(p[1] + u)]
            v = (pi[0] + pi[1]) * k[32]
            f = [p[0] - (pi[0] - v), p[1] - (pi[1] - v)]
            length = np.sqrt(f[0] * f[0] + f[1] * f[1])
            grain = F(1) - F(2) * F(2.0 ** (-float(length) * 3.0))
            want = F(0.5) + grain * F(0.5) * F(0.6)
            assert abs(float(out[y, x, 0]) - float(want)) < 1e-6
    # a negative divisor's quotient wraps to u32, a divisor from scale 16 is 2: both are finite
    for scale in (-16.0, 16.0, 1e30, float("nan")):
        assert np.isfinite(so.tonemap(frame, abi.tonemap_settings(FG, abi.TONEMAP_NONE, film_grain_scale=scale))[..., 3]).all()


def test_taps_wrap(so):
    """item 1: Repeat; the tap at u = 0 reads the first and last columns half and half"""
    plane = np.zeros((1, 4, 4), np.float32)
    plane[0, 0], plane[0, 3] = 2.0, 6.0
    np.testing.assert_array_equal(so.tap(plane, 0.0, 0.5), np.float32([4, 4, 4, 4]))
    np.testing.assert_array_equal(so.tap(plane, 1.0, 0.5), np.float32([4, 4, 4, 4]))
    np.testing.assert_array_equal(so.tap(plane, 0.125, 0.5), np.float32([2, 2, 2, 2]))
