"""The atmosphere oracle's specification pinned by hand (oracle/oxc_oracle_atmosphere.c, include/oxcull.h above
oxc_atmosphere_transmittance): the constants' bits, canonical_exp's and canonical_acos' error bounds and special values, the ray-sphere
cases, the transmittance LUT's parametrisation round trip, the aerial perspective's integer per_slice_depth, and whole LUTs of
atmospheres whose answer is known exactly (zero scattering, zero extinction, a camera above the atmosphere) or in closed form (the
zenith transmittance from the ground).  No GPU."""
import math
import os
import re

import numpy as np
import pytest

from oxylus_b200 import abi
from tests.test_gpu_atmosphere import camera_for

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ao():
    import pyoracle_atmosphere

    pyoracle_atmosphere.build()
    return pyoracle_atmosphere


def f32(x):
    return np.float32(x)


def bits(x):
    return int(np.array(x, np.float32).view(np.uint32))


PI = f32(math.pi)
# name in oxc_atmosphere.cuh (PI: oxc_shader_math.cuh) -> (bits, how the shader's value is formed)
CONSTANTS = {
    "PI": (0x40490FDB, PI),
    "ATM_TAU": (0x40C90FDB, f32(2 * math.pi)),
    "ATM_INV_4PI": (0x3DA2F983, f32(1) / (f32(4) * PI)),          # 1.0 / (4.0 * PI), 4 * PI exact
    "ATM_RAYLEIGH_K": (0x3D747645, f32(3) / (f32(16) * PI)),      # 3.0 / (16.0 * PI), 16 * PI exact
    "ATM_THIRD": (0x3EAAAAAB, f32(1) / f32(3)),
    "ATM_CAMERA_SCALE_UNIT": (0x3C23D70A, f32(0.01)),
    "ATM_PLANET_RADIUS_OFFSET": (0x3A83126F, f32(0.001)),
    "ATM_HALF_MIN_NORMAL": (0x38800000, f32(6.103515625e-5)),
    "ATM_HALF_MAX": (0x477FE000, f32(65504.0)),
}


def test_constants_bits():
    """each constant of the kernel header and of the oracle is the binary32 value the shader forms, with the bits the specification
    states; the folded quotients give the same bits in binary32 and in binary64 rounded once"""
    src = "".join(open(os.path.join(ROOT, "oxylus_b200", "csrc", h)).read() for h in ("oxc_atmosphere.cuh", "oxc_shader_math.cuh"))
    orc = open(os.path.join(ROOT, "oracle", "oxc_oracle_atmosphere.c")).read()
    hdr = open(os.path.join(ROOT, "include", "oxcull.h")).read()
    for name, (b, value) in CONSTANTS.items():
        m = re.search(rf"constexpr float {name} = ([^;]+);", src)
        assert m, name
        lit = m.group(1).strip()
        got = f32(float.fromhex(lit[:-1])) if lit.startswith("0x") else f32(float(lit[:-1]))
        assert bits(got) == b == bits(value), (name, hex(bits(got)), hex(b), hex(bits(value)))
        assert f"0x{b:08X}" in hdr or name in ("ATM_THIRD",), name
    assert bits(f32(1.0 / (4.0 * float(PI)))) == 0x3DA2F983 and bits(f32(3.0 / (16.0 * float(PI)))) == 0x3D747645
    assert bits(f32(1.0 / 3.0)) == 0x3EAAAAAB
    for lit, name in (("0x1.45f306p-4f", "A_INV_4PI"), ("0x1.e8ec8ap-5f", "A_RAYLEIGH_K"), ("0x1.555556p-2f", "A_THIRD"),
                      ("0x1.47ae14p-7f", "A_CSU"), ("0x1.0624dep-10f", "A_PRO"), ("0x1.921fb6p+1f", "A_PI"), ("0x1.921fb6p+2f", "A_TAU")):
        assert f"{name} = {lit}" in orc, name


def test_rayleigh_phase_constant(ao):
    assert bits(ao.rayleigh_phase(0.0)) == 0x3D747645
    assert ao.rayleigh_phase(1.0) == CONSTANTS["ATM_RAYLEIGH_K"][1] * f32(2.0)


def _ulp_of_exact(e):
    e32 = np.abs(e).astype(np.float32)
    return np.where(np.abs(e) < 2.0 ** -126, 2.0 ** -149, np.spacing(e32).astype(np.float64))


def test_canonical_exp_bound_and_special_values(ao):
    """within 1 ulp of the exact exp over 10^7 inputs: 5 M random bit patterns (the whole binary32 domain) and 5 M uniform in the
    range where the result is neither 0 nor inf; measured max 0.945 ulp"""
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.integers(0, 2 ** 32, 5_000_000, dtype=np.uint64).astype(np.uint32).view(np.float32),
                        rng.uniform(-104.0, 89.0, 5_000_000).astype(np.float32)])
    y = ao.exp(x)
    with np.errstate(all="ignore"):
        e = np.exp(x.astype(np.float64))
    finite = np.isfinite(x)
    ok = finite & (e < float(np.finfo(np.float32).max))
    err = np.abs(y[ok].astype(np.float64) - e[ok]) / _ulp_of_exact(e[ok])
    assert ok.sum() > 8_000_000 and err.max() < 1.0, err.max()
    over = finite & ~ok
    assert np.isposinf(y[over]).all() and over.sum() > 1000
    # specials
    s = ao.exp(np.float32([0.0, -0.0, np.inf, -np.inf, np.nan, 88.72283, 88.7229, 89.0, -103.0, -103.97, -104.0, -104.1, -87.33655]))
    assert bits(s[0]) == bits(s[1]) == 0x3F800000
    assert np.isposinf(s[2]) and bits(s[3]) == 0 and np.isnan(s[4])
    assert np.isfinite(s[5]) and np.isposinf(s[6]) and np.isposinf(s[7])
    assert 0 < s[8] < 2 ** -126 and s[9] == 2.0 ** -149 and s[10] == 0 and s[11] == 0  # subnormals, then 0
    assert s[12] == f32(np.exp(np.float64(np.float32(-87.33655))))
    # monotone over a dense sweep
    sweep = np.linspace(-20, 20, 200001).astype(np.float32)
    ys = ao.exp(sweep)
    assert (np.diff(ys) >= 0).all()


def test_canonical_acos_bound(ao):
    """within 1 ulp (measured 0.5) of the exact acos on 2 M inputs of [-1, 1]; +-1, 0 and out-of-range / NaN inputs"""
    rng = np.random.default_rng(2)
    x = np.concatenate([rng.uniform(-1, 1, 2_000_000), rng.uniform(0.999, 1.0, 10000), rng.uniform(-0.5, 0.5, 10000)]).astype(np.float32)
    y = ao.acos(x).astype(np.float64)
    e = np.arccos(x.astype(np.float64))
    err = np.abs(y - e) / np.spacing(e.astype(np.float32)).astype(np.float64)
    assert err.max() < 1.0, err.max()
    s = ao.acos(np.float32([1.0, -1.0, 0.0, 1.0000001, -1.0000001, np.nan]))
    assert s[0] == 0 and s[1] == PI and s[2] == f32(math.pi / 2) and np.isnan(s[3:]).all()


def test_ray_sphere_cases(ao):
    r = 10.0
    # from inside: the exit
    assert ao.ray_sphere_nearest((0, 0, 0), (0, 1, 0), r) == f32(10.0)
    # from outside towards it: the near side
    assert ao.ray_sphere_nearest((0, 20, 0), (0, -1, 0), r) == f32(10.0)
    # outside, pointing away: behind, `none`
    assert ao.ray_sphere_nearest((0, 20, 0), (0, 1, 0), r) is None
    # a miss
    assert ao.ray_sphere_nearest((0, 20, 0), (1, 0, 0), r) is None
    # tangent: delta = 0, one touching point at distance 20
    t = ao.ray_sphere_nearest((-20, 10, 0), (1, 0, 0), r)
    assert t == f32(20.0)
    # starting on the sphere: the roots are 0 and +-20, so the nearest is 0 going out and going in
    assert ao.ray_sphere_nearest((0, 10, 0), (0, 1, 0), r) == 0.0
    assert ao.ray_sphere_nearest((0, 10, 0), (0, -1, 0), r) == 0.0
    # NaN: delta < 0 is false, the roots are NaN, max(0, min(NaN, NaN)) = 0
    assert ao.ray_sphere_nearest((0, np.nan, 0), (0, 1, 0), r) == 0.0


def test_transmittance_uv_round_trip(ao):
    """transmittance_params_to_lut_uv maps every bake texel's (height, cos theta) back to that texel's centre, within a tolerance (the
    binary32 steps of both directions lose a few ulps of the km-sized radii) of 2e-4 in u and v (measured 9.6e-5 and 8.7e-5)"""
    a = abi.atmosphere(transmittance_lut_size=(256, 64, 1))
    worst_u = worst_v = 0.0
    for y in range(64):
        for x in range(256):
            h, c = ao.transmittance_params(a, x, y)
            mu, r = ao.transmittance_uv(a.atmos_radius, a.planet_radius, h, c)
            worst_u = max(worst_u, abs(mu - (x + 0.5) / 256))
            worst_v = max(worst_v, abs(r - (y + 0.5) / 64))
    assert worst_u < 2e-4 and worst_v < 2e-4, (worst_u, worst_v)


def test_aerial_perspective_per_slice_depth_is_integer_division(ao):
    """per_slice_depth = f32(size.x / size.z) in integers: 0 when z > x, so every slice integrates over length 0 and stores (0, 0, 0,
    mean of 1); at 32^3 it is 1 and slice z reaches ((z + 0.5) / 32)^2 * 32 km, so the transmittance falls with depth"""
    cam = camera_for(0.2)
    one = f32(f32(f32(1.0 / 3.0) + f32(1.0 / 3.0)) + f32(1.0 / 3.0))
    a = abi.atmosphere(transmittance_lut_size=(32, 8, 1), sky_view_lut_size=(4, 4, 1), aerial_perspective_lut_size=(3, 2, 4))
    t = ao.transmittance(a)
    _, ap = ao.sky_luts(a, cam, (0.0, 1.0, 0.0), 10.0, t)
    assert (ap[..., :3] == 0).all() and (ap[..., 3] == np.float16(one)).all()
    a = abi.atmosphere(transmittance_lut_size=(32, 8, 1), sky_view_lut_size=(4, 4, 1), aerial_perspective_lut_size=(4, 4, 4))
    _, ap = ao.sky_luts(a, cam, (0.0, 1.0, 0.0), 10.0, ao.transmittance(a))
    mean_t = ap[..., 3].astype(np.float32).mean(axis=(1, 2))
    assert (np.diff(mean_t) < 0).all() and (ap[1:, :2, :, :3] > 0).all()  # the rays above the horizon (rows 0 and 1)


def test_zero_scattering_gives_zero_luminance(ao):
    a = abi.atmosphere(rayleigh_scatter=(0, 0, 0), mie_scatter=(0, 0, 0), transmittance_lut_size=(32, 8, 1), sky_view_lut_size=(24, 16, 1),
                       aerial_perspective_lut_size=(8, 8, 8))
    t = ao.transmittance(a)
    sv, ap = ao.sky_luts(a, camera_for(1000.0), (0.3, 0.8, 0.5), 10.0, t)
    assert (sv[..., :3].view(np.uint16) == 0).all() and (sv[..., 3] == np.float16(6.103515625e-5)).all()
    assert (ap[..., :3].view(np.uint16) == 0).all() and (ap[..., 3] > 0).all()


def test_zero_extinction(ao):
    """no extinction: transmittance exactly 1; the aerial perspective's integral is 0 / 0 and stores the pinned NaN 0x7FFF; the sky
    view's max(NaN, 0) = 0 gives (0, 0, 0, HALF_MIN_NORMAL)"""
    a = abi.atmosphere(rayleigh_scatter=(0, 0, 0), mie_extinction=0.0, ozone_absorption=(0, 0, 0), transmittance_lut_size=(32, 8, 1),
                       sky_view_lut_size=(24, 16, 1), aerial_perspective_lut_size=(8, 8, 8))
    t = ao.transmittance(a)
    assert (t.view(np.uint16) == 0x3C00).all()
    sv, ap = ao.sky_luts(a, camera_for(0.2), (0.3, 0.8, 0.5), 10.0, t)
    assert (ap[..., :3].view(np.uint16) == 0x7FFF).all() and (ap[..., 3] == np.float16(1.0)).all()
    assert (sv[..., :3].view(np.uint16) == 0).all() and (sv[..., 3] == np.float16(6.103515625e-5)).all()
    assert ao.half(float("nan")) == 0x7FFF and ao.half(-float("nan")) == 0x7FFF


def test_camera_above_the_atmosphere(ao):
    """at 150 km the sky-view texels whose rays miss the atmosphere (binary64 test from the eye) store exactly 0; the aerial
    perspective's slices (at most 32 km deep) end before the atmosphere (50 km below) and are all 0"""
    a = abi.atmosphere(transmittance_lut_size=(64, 16, 1), sky_view_lut_size=(48, 32, 1), aerial_perspective_lut_size=(8, 8, 8))
    t = ao.transmittance(a)
    sv, ap = ao.sky_luts(a, camera_for(15000.0), (0.0, 0.70710677, -0.70710677), 10.0, t)
    assert (ap.view(np.uint16) == 0).all()
    eye_y = float(ao.eye_y(a, 15000.0))
    miss = hit = 0
    for y in range(32):
        for x in range(48):
            d = ao.sky_view_dir(a, (x + 0.5) / 48, (y + 0.5) / 32, eye_y).astype(np.float64)
            b = 2 * d[1] * eye_y
            delta = b * b - 4 * (d @ d) * (eye_y ** 2 - float(a.atmos_radius) ** 2)
            if delta < -1.0 or (delta > 1.0 and -b + math.sqrt(delta) < 0):
                miss += 1
                assert (sv[y, x].view(np.uint16) == 0).all(), (x, y)
            elif delta > 1.0:
                hit += 1
                assert sv[y, x, 3] > 0
    assert miss > 300 and hit > 300


def test_zenith_transmittance_from_the_ground(ao):
    """the bake's march straight up from the ground (height R, cos theta 1) against the closed-form optical depth of the exponential
    Rayleigh / Mie profiles and the ozone tent.  The bake is the right Riemann sum with 1000 steps of L / 1000: its error is at most
    the step times the total variation of the integrand (exponentials: f(0) - f(L); tent: twice its peak); the binary32 sum of 1000
    terms adds at most 1000 * 2^-24 relative."""
    a = abi.atmosphere()
    R, A = float(a.planet_radius), float(a.atmos_radius)
    L = A - R
    step = L / 1000.0
    hr, hm = float(a.rayleigh_density), float(a.mie_density)
    oh, ot = float(a.ozone_height), float(a.ozone_thickness)

    def tent_integral(lo, hi):  # integral of max(0, 1 - |z - oh| / ot) over [lo, hi]
        zs = np.linspace(lo, hi, 2_000_001)
        return np.trapezoid(np.maximum(0.0, 1.0 - np.abs(zs - oh) / ot), zs)

    got = ao.transmittance_ray(a, R, 1.0).astype(np.float64)
    for c in range(3):
        rs, ms, me, oz = float(a.rayleigh_scatter[c]), float(a.mie_scatter[c]), float(a.mie_extinction), float(a.ozone_absorption[c])
        od = rs * hr * (1 - math.exp(-L / hr)) + me * hm * (1 - math.exp(-L / hm)) + oz * tent_integral(0.0, L)
        tv = rs * (1 - math.exp(-L / hr)) + me * (1 - math.exp(-L / hm)) + oz * 2.0
        bound = step * tv + od * 1000 * 2.0 ** -24 + 1e-6
        od_bake = -math.log(got[c])
        assert abs(od_bake - od) <= bound, (c, od_bake, od, bound)
        assert abs(od_bake - od) > 0  # the Riemann sum is not the integral
