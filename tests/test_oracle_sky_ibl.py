"""The sky IBL oracle's specification pinned by hand (oracle/oxc_oracle_sky_ibl.c, include/oxcull.h above oxc_atmosphere_sky_ibl): the
constants' bits, the face directions, radical_inverse_vdc and IGN, the history rules, the 0.02 lerp, the clamp at 65504, the sun term with
an unnormalized sun and a sun below the horizon, the view-zenith cosine that cannot round past 1 and a NaN acos, canonical_atan2's special cases and error bound,
and canonical_acos' coefficients.  The LUTs are uniform or hand-made, so every expected value is formed here in binary32.  No GPU."""
import math
import os
import re

import numpy as np
import pytest

from oxylus_b200 import abi
from tests.test_gpu_atmosphere import camera_for

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
SIZES = dict(transmittance_lut_size=(8, 4, 1), sky_view_lut_size=(6, 5, 1), aerial_perspective_lut_size=(1, 1, 1))


@pytest.fixture(scope="module")
def so():
    import pyoracle_sky_ibl

    pyoracle_sky_ibl.build()
    return pyoracle_sky_ibl


def bits(x):
    return int(np.array(x, np.float32).view(np.uint32))


def uniform(shape, rgba):
    return np.broadcast_to(np.float16(rgba), tuple(shape) + (4,)).copy()


def planes(a, sky=(0.5, 0.5, 0.5, 1.0), trans=(0.5, 0.25, 1.0, 1.0)):
    t = uniform((a.transmittance_lut_size[1], a.transmittance_lut_size[0]), trans)
    sv = uniform((a.sky_view_lut_size[1], a.sky_view_lut_size[0]), sky)
    return t, sv


CONSTANTS = {"SKY_IBL_UP_LIMIT": (0x3F7FBE77, "0.999"), "SKY_IBL_IGN_X": (0x3D897143, "0.06711056"), "SKY_IBL_IGN_Y": (0x3BBF4590, "0.00583715"),
             "SKY_IBL_IGN_Z": (0x4253EE82, "52.9829189"), "SKY_IBL_GOLDEN": (0x3F1E377A, "0.61803398875"),
             "SKY_IBL_VDC_SCALE": (0x2F800000, "2.3283064365386963e-10"), "SKY_IBL_ALPHA": (0x3CA3D70A, "0.02"),
             "SKY_IBL_SAFE_NORMALIZE_MIN": (0x1E3CE508, "1e-20"), "SKY_IBL_SIDE_MIN": (0x3727C5AC, "1e-5")}


def test_constants_bits():
    """each literal of the kernel header and of the oracle is the binary32 rounding of the shader's, with the bits the specification states"""
    src = open(os.path.join(ROOT, "oxylus_b200", "csrc", "oxc_sky_ibl.cuh")).read()
    orc = open(os.path.join(ROOT, "oracle", "oxc_oracle_sky_ibl.c")).read()
    hdr = open(os.path.join(ROOT, "include", "oxcull.h")).read()
    for name, (b, literal) in CONSTANTS.items():
        m = re.search(rf"constexpr float {name} = (0x[0-9a-fp.+-]+)f;", src)
        assert m, name
        assert bits(F(float.fromhex(m.group(1)))) == b == bits(F(float(literal))), name
        assert m.group(1) + "f" in orc, name
        assert f"0x{b:08X}" in hdr, name


def test_acos_coefficients_are_the_recurrence():
    """canonical_acos' written-out coefficients are the binary64 values of the oracle's recurrence"""
    src = open(os.path.join(ROOT, "oxylus_b200", "csrc", "oxc_exact.cuh")).read()
    body = src[src.index("OXC_HD float canonical_acos"):src.index("OXC_HD float canonical_atan2")]
    lits = [float.fromhex(x) for x in re.findall(r"(0x1\.[0-9a-f]+p[+-]\d+)", body)]
    c, central = [], 1.0
    for n in range(29):
        if n > 0:
            central = central * float(2 * n - 1) / float(2 * n)
        c.append(central / float(2 * n + 1))
    assert lits == c[28:0:-1]


@pytest.mark.parametrize("face", range(6))
def test_face_directions(so, face):
    """the four texels around each face's centre look along its axis (+X, -X, +Y, -Y, +Z, -Z), every direction is unit length, and the
    faces' edges meet: texel (0, y) of +X and texel (31, y) of +Z are mirror images across the x = z plane"""
    axis, sign = face // 2, 1.0 if face % 2 == 0 else -1.0
    for x, y in ((15, 15), (16, 16), (15, 16), (16, 15)):
        d = so.direction(face, x, y)
        assert np.argmax(np.abs(d)) == axis and np.sign(d[axis]) == sign and abs(d[axis]) > 0.998
    for x in range(32):
        for y in range(0, 32, 7):
            assert abs(float(np.linalg.norm(so.direction(face, x, y).astype(np.float64))) - 1.0) < 3e-7


def test_radical_inverse_and_ign(so):
    for i in range(64):
        assert so.radical_inverse(i) == F(int(f"{i:032b}"[::-1], 2) * 2.0 ** -32)
    for px, py in ((0.0, 0.0), (5.0, 9.0), (31.0 + 5 * 37.0, 31.0 + 5 * 17.0), (17.0, 3.0 + 17.0)):
        d = F(F(F(px) * F(0.06711056)) + F(F(py) * F(0.00583715)))
        inner = F(d - np.floor(d))
        v = F(F(52.9829189) * inner)
        assert so.ign(px, py) == F(v - np.floor(v)), (px, py)


def test_local_samples_are_cosine_weighted(so):
    """the 64 local directions have unit length, z = sqrt(1 - u1), and their mean z is near the cosine-weighted 2/3"""
    zs = []
    for i in range(64):
        s = so.local_sample(i, 0.3).astype(np.float64)
        assert abs(np.linalg.norm(s) - 1.0) < 1e-6
        zs.append(s[2])
    assert abs(np.mean(zs) - 2.0 / 3.0) < 2e-3


def _frame(so, a, cube, sky, strength=0.0, sun=(0.0, 0.70710677, -0.70710677), intensity=10.0, frame=3, trans=(0.5, 0.25, 1.0, 1.0)):
    t, sv = planes(a, sky, trans)
    return so.sky_ibl(a, camera_for(0.2), sun, intensity, strength, frame, t, sv, cube)


def test_history_rules_and_lerp(so):
    """a uniform sky (c, 1) with the sun term off gives c on every texel without history; a texel with a > 0 and finite rgb lerps toward c
    with alpha 0.02; a = 0, -0, a < 0, a NaN, a NaN or +-inf rgb channel all mean no history"""
    a = abi.atmosphere(**SIZES)
    c = F(0.5)
    cube = np.zeros(abi.SKY_IBL_CUBE_SHAPE, np.float16)
    hostile = {(0, 3, 4): (2.0, 2.0, 2.0, 0.0), (0, 3, 5): (2.0, 2.0, 2.0, -0.0), (0, 3, 6): (2.0, 2.0, 2.0, -1.0),
               (0, 3, 7): (2.0, 2.0, 2.0, np.nan), (0, 3, 8): (np.nan, 2.0, 2.0, 1.0), (0, 3, 9): (2.0, np.inf, 2.0, 1.0),
               (0, 3, 10): (2.0, 2.0, -np.inf, 1.0)}
    valid = {(1, 9, 9): (2.0, -3.0, 65504.0, 0.5), (4, 20, 2): (0.0, 6e-8, 1.0, 6e-8)}
    for (f, y, x), v in {**hostile, **valid}.items():
        cube[f, y, x] = np.float16(v)
    out = _frame(so, a, cube, (c, c, c, 1.0)).astype(np.float32)
    assert (out[..., 3] == 1).all()
    for key in hostile:
        np.testing.assert_array_equal(out[key][:3], [c, c, c])
    for key, v in valid.items():
        h = np.float16(v[:3]).astype(np.float32)
        want = np.float16(F(h + F(F(c - h) * F(0.02))))
        np.testing.assert_array_equal(np.float16(out[key][:3]).view(np.uint16), want.view(np.uint16))
    plain = np.ones(out.shape[:3], bool)
    for key in list(hostile) + list(valid):
        plain[key] = False
    assert (out[plain][:, :3] == c).all()


def test_clamp_at_half_max(so):
    """the estimate plus the sun term is clamped to 65504 before the store; an infinite sky reads 0 (sanitize), not inf"""
    a = abi.atmosphere(**SIZES)
    out = _frame(so, a, None, (60000.0, 60000.0, 60000.0, 1.0), strength=1.0, intensity=1e6, sun=(0.0, 1.0, 0.0)).astype(np.float32)
    assert out[2, 15, 15, 0] == 65504.0 and np.isfinite(out).all()
    assert (out[..., :3] <= 65504.0).all()
    inf_sky = _frame(so, a, None, (np.inf, 1.0, 1.0, 1.0)).astype(np.float32)
    assert (inf_sky[..., 0] == 0).all() and (inf_sky[..., 1] > 0).any()


@pytest.mark.parametrize("sun", [(0.0, 2.0, 0.0), (0.3, 1.5, -0.9), (0.0, -0.5, 0.0)])
def test_sun_term(so, sun):
    """with a black sky the texel is the sun term alone: (((0.15 * T) * I) * saturate(dot(dir, sun))) / PI with the sun as given (an
    unnormalized sun saturates at 1 early; a sun below the horizon still lights the faces it faces) and T the uniform transmittance"""
    a = abi.atmosphere(**SIZES)
    trans = (0.5, 0.25, 1.0, 1.0)
    out = _frame(so, a, None, (0.0, 0.0, 0.0, 1.0), strength=0.15, sun=sun, intensity=7.0, trans=trans)
    s = np.float32(sun)
    lit = 0
    for f in range(6):
        for y in (0, 9, 31):
            for x in (0, 14, 31):
                d = so.direction(f, x, y)
                dot = F(F(F(d[0] * s[0]) + F(d[1] * s[1])) + F(d[2] * s[2]))
                sat = F(min(max(dot, F(0)), F(1)))
                want = [np.float16(F(F(F(F(F(0.15) * F(tc)) * F(7.0)) * sat) / F(math.pi))) for tc in trans[:3]]
                np.testing.assert_array_equal(out[f, y, x, :3].view(np.uint16), np.float16(want).view(np.uint16))
                lit += sat > 0
    assert lit > 0


def test_zenith_acos_argument(so):
    """the view-zenith cosine cannot round past 1: up = (0, y / sqrt(fl(y * y)), 0) is exactly (0, 1, 0) for every finite height, so the
    cosine is the sample's y, at most 1 after normalize.  acos of an argument past +-1 or NaN is NaN; in sky_view_params_to_lut_uv the NaN
    reaches safe_sqrt, whose max(0, NaN) is 0, so v is 0.5 (the horizon row) in both branches: an infinite eye height (up = inf / inf =
    NaN) reads the sky there.  A NaN v would make the tap NaN in every channel"""
    a = abi.atmosphere(**SIZES)
    R = F(a.planet_radius)
    cy = np.linspace(-10.0, 30000.0, 200001, dtype=np.float32)
    ey = np.maximum(F(cy * F(0.01)) + F(R + F(0.001)), F(R + F(0.001))).astype(np.float32)
    assert (np.float32(ey / np.sqrt(np.float32(ey * ey))) == 1.0).all()
    assert np.isnan(so.acos(np.float32([1.0000001, -1.0000001, np.nan]))).all()
    _, sv = planes(a, (0.5, 0.5, 0.5, 1.0))
    assert np.isnan(so.tap4(sv, 0.5, np.nan)).all()
    sun = (0.0, 0.70710677, -0.70710677)
    assert (so.illuminance(a, 0.2, sun, sv, (0.0, 1.0, 0.0)) == F(0.5)).all()
    sky = np.zeros_like(sv)
    sky[2, :, :3], sky[..., 3] = np.float16(0.25), np.float16(1.0)  # only the rows around v = 0.5 are lit
    got = so.illuminance(a, np.inf, sun, sky, (0.0, 1.0, 0.0))
    assert (got > 0).all() and np.isfinite(got).all()


def _ulp_of_exact(e):
    e32 = np.abs(e).astype(np.float32)
    return np.where(np.abs(e) < 2.0 ** -126, 2.0 ** -149, np.spacing(e32).astype(np.float64))


def test_canonical_atan2_special_values(so):
    pi, nan, inf = F(math.pi), np.nan, np.inf
    cases = [((0.0, 1.0), 0.0), ((-0.0, 1.0), -0.0), ((0.0, 0.0), 0.0), ((-0.0, 0.0), -0.0), ((0.0, -0.0), pi), ((-0.0, -0.0), -pi),
             ((0.0, -1.0), pi), ((-0.0, -1.0), -pi), ((1.0, 0.0), F(math.pi / 2)), ((-1.0, -0.0), -F(math.pi / 2)),
             ((inf, inf), F(math.pi / 4)), ((-inf, inf), -F(math.pi / 4)), ((inf, -inf), F(3 * math.pi / 4)), ((-inf, -inf), -F(3 * math.pi / 4)),
             ((inf, 5.0), F(math.pi / 2)), ((-inf, -5.0), -F(math.pi / 2)), ((5.0, inf), 0.0), ((-5.0, inf), -0.0), ((5.0, -inf), pi),
             ((-5.0, -inf), -pi), ((1.0, 1.0), F(math.pi / 4)), ((1.0, -1.0), F(3 * math.pi / 4)), ((-1.0, -1.0), -F(3 * math.pi / 4))]
    for (y, x), want in cases:
        got = so.atan2(np.float32([y]), np.float32([x]))[0]
        assert bits(got) == bits(F(want)), (y, x, got, want)
    for y, x in ((nan, 1.0), (1.0, nan), (nan, nan), (inf, nan)):
        assert bits(so.atan2(np.float32([y]), np.float32([x]))[0]) == 0x7FC00000


def test_canonical_atan2_bound(so):
    """within 1 ulp of the exact atan2 over 10^7 inputs: 5 M random bit-pattern pairs (the whole binary32 domain) and 5 M normal pairs in
    all four quadrants; measured max 0.5 ulp"""
    rng = np.random.default_rng(3)
    n = 5_000_000
    y = np.concatenate([rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32), rng.normal(size=n).astype(np.float32)])
    x = np.concatenate([rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32), rng.normal(size=n).astype(np.float32)])
    got = so.atan2(y, x).astype(np.float64)
    e = np.arctan2(y.astype(np.float64), x.astype(np.float64))
    ok = np.isfinite(x) & np.isfinite(y)
    err = np.abs(got[ok] - e[ok]) / _ulp_of_exact(e[ok])
    assert ok.sum() > 9_000_000 and err.max() < 1.0, err.max()
    # the sign follows y, the quadrant x
    assert (np.signbit(got[ok]) == np.signbit(y[ok])).all()
    assert (np.abs(got[ok & (x < 0) & (y != 0)]) > math.pi / 2 - 1e-6).all()
