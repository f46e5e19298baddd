"""The PBR apply oracle (oracle/oxc_oracle_pbr.c) pinned by hand: the new structs' layout, canonical_pow5 against the exact power, the
split-sum fit against binary64, the point window, the spot smoothstep, the early returns, flag gating, hostile inputs, and an
independent binary64 numpy restatement of the shader over random frames."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_pbr import mixed_lights, random_planes, settings_for

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


@pytest.fixture(scope="module")
def po():
    import pyoracle_pbr

    pyoracle_pbr.build()
    return pyoracle_pbr


def run(po, pcam, s, lights, planes, omit=()):
    p = {k: (None if k in omit else v) for k, v in planes.items()}
    return po.apply_pbr(pcam, s, lights, p["depth"], p["albedo"], p["normal"], p["emissive"], p["metallic_roughness_occlusion"],
                        p["ambient_occlusion"], p["shadow"], p["contact_shadow"])


def test_struct_layout():
    assert C.sizeof(abi.Light) == 64 and C.sizeof(abi.PbrSettings) == 68 and C.sizeof(abi.PbrCamera) == 76 and C.sizeof(abi.PbrInputs) == 64
    off = {k: getattr(abi.Light, k).offset for k in ("position", "intensity", "color", "range", "direction", "inner_cone_angle",
                                                      "outer_cone_angle", "kind", "pad")}
    assert off == dict(position=0, intensity=12, color=16, range=28, direction=32, inner_cone_angle=44, outer_cone_angle=48, kind=52, pad=56)
    off = {k: getattr(abi.PbrSettings, k).offset for k, _ in abi.PbrSettings._fields_}
    assert off == dict(scene_flags=0, sun_direction=4, sun_intensity=16, base_ambient_color=20, sky_solid_color=32, sky_ambient_color=48,
                       sky_has_texture=60, light_count=64)
    assert abi.PbrCamera.position.offset == 64
    assert [getattr(abi.PbrInputs, k).offset for k in abi.PBR_INPUTS] == list(range(0, 64, 8))
    assert (abi.SCENE_HAS_GTAO, abi.SCENE_HAS_CONTACT_SHADOWS, abi.SCENE_HAS_SKY, abi.SCENE_TRANSPARENT_BACKGROUND) == (32, 512, 1024, 2048)


def _within_one_ulp(x, r):
    """exact check, in Python integers (every binary32 is a multiple of 2^-149): the exact x^5 lies strictly between the binary32
    neighbours of r, i.e. r is within 1 ulp of it"""
    S = 2.0 ** 149
    lo = np.nextafter(r, np.float32(-np.inf)).astype(np.float64) * S
    hi = np.nextafter(r, np.float32(np.inf)).astype(np.float64) * S
    xm = (x.astype(np.float64) * S).tolist()
    bad = []
    for i, (m, a, b) in enumerate(zip(xm, lo.tolist(), hi.tolist())):
        p = int(m) ** 5
        if not (int(a) << 596 < p < int(b) << 596):
            bad.append(i)
    return bad


def test_pow5_within_one_ulp(po):
    """canonical_pow5 against the exact power on 10^6 random binary32 values in [0, 1] and every 256th binary32 in [0, 1]"""
    rng = np.random.default_rng(0)
    xs = [rng.random(10**6, dtype=np.float32), np.arange(0, 0x3F800001, 256, dtype=np.uint32).view(np.float32)]
    for x in xs:
        r = po.pow5(x)
        assert _within_one_ulp(x, r) == []
    # correctly rounded almost everywhere: the binary64 error is far below half a binary32 ulp
    x = xs[0]
    exact = (x.astype(np.float64) ** 2) ** 2 * x.astype(np.float64)
    assert (po.pow5(x) == exact.astype(np.float32)).mean() > 0.999999
    assert po.pow5(np.float32([0.0, 1.0, -0.0]))[[0, 1]].tolist() == [0.0, 1.0]
    assert np.isnan(po.pow5(np.float32([np.nan])))[0]


def test_ggx_directional_albedo_against_binary64(po):
    c = np.float64([[0.1003, 0.9345, 1.0, 1.0], [-0.6303, -2.323, -1.765, 0.2281], [9.748, 2.229, 8.263, 15.94], [-2.038, -3.748, 11.53, -55.83],
                    [29.34, 1.424, 28.96, 13.08], [-8.245, -0.7684, -7.507, 41.26], [-26.44, 1.436, -36.11, 54.9], [19.99, 0.2913, 15.86, 300.2],
                    [-5.448, 0.6286, 33.37, -285.1]])
    rng = np.random.default_rng(1)
    for NoV, alpha in zip(rng.uniform(1e-5, 1.0, 2000), rng.uniform(0.0025, 1.0, 2000)):
        x, y = float(np.float32(NoV)), float(np.float32(alpha))
        t = np.float64([1.0, x, y, x * y, x * x, y * y, x * x * y, x * y * y, x * x * y * y]) @ c
        want = np.clip(t[:2] / t[2:], 0.0, 1.0)
        got = po.ggx_directional_albedo(x, y)
        np.testing.assert_allclose(got, want, rtol=2e-5, atol=2e-6)


def test_point_attenuation(po):
    f32 = np.float32
    assert po.attenuate_point(2.0, 0.0) == f32(1.0) / (f32(4.0) + f32(0.1))
    assert po.attenuate_point(3.0, -1.0) == f32(1.0) / (f32(9.0) + f32(0.1))
    assert po.attenuate_point(0.0, 5.0) == f32(1.0) / f32(0.1)
    for r in (0.5, 1.0, 7.25, 100.0):
        assert po.attenuate_point(r, r) == 0.0
        assert po.attenuate_point(np.nextafter(f32(r), f32(np.inf)), r) == 0.0
        assert po.attenuate_point(r * 1.5, r) == 0.0 and po.attenuate_point(1e30, r) == 0.0
        assert po.attenuate_point(r * 0.999, r) > 0.0
        d = f32(r * 0.5)
        w = f32(1.0) - ((d / f32(r)) ** 2) ** 2
        assert po.attenuate_point(d, r) == np.float32(w * w / (d * d + f32(0.1)))
    assert po.attenuate_point(1.0, float("nan")) == 0.0


def test_spot_smoothstep(po):
    down = np.float32([0.0, -1.0, 0.0])
    L_axis = np.float32([0.0, 1.0, 0.0])  # to the light: the pixel lies on the spot's axis
    assert po.spot_attenuation(L_axis, down, 0.3, 0.5) == 1.0
    off = np.float32([np.sin(0.8), np.cos(0.8), 0.0])  # 0.8 rad off the axis: outside the outer cone
    assert po.spot_attenuation(off, down, 0.3, 0.5) == 0.0
    mid = np.float32([np.sin(0.4), np.cos(0.4), 0.0])
    assert 0.0 < po.spot_attenuation(mid, down, 0.3, 0.5) < 1.0
    # inner == outer: a step, x == e gives 0 / 0 -> saturate(NaN) = 0
    assert po.spot_attenuation(L_axis, down, 0.4, 0.4) == 1.0 and po.spot_attenuation(off, down, 0.4, 0.4) == 0.0
    assert po.smoothstep(0.5, 0.5, 0.5) == 0.0 and po.smoothstep(0.5, 0.5, 0.6) == 1.0 and po.smoothstep(0.5, 0.5, 0.4) == 0.0
    assert po.smoothstep(0.0, 1.0, 0.5) == 0.5 and po.smoothstep(0.0, 1.0, float("nan")) == 0.0
    # the spot direction is normalized: its length does not matter
    assert po.spot_attenuation(mid, down * 7, 0.3, 0.5) == po.spot_attenuation(mid, down, 0.3, 0.5)


def test_early_returns(po):
    rng = np.random.default_rng(2)
    pcam, planes = random_planes(rng, 40, 30)
    sky = planes["depth"] == 0
    lights = mixed_lights(rng, 5)
    s = settings_for(abi.SCENE_TRANSPARENT_BACKGROUND | abi.SCENE_HAS_SKY | abi.SCENE_HAS_DIRECTIONAL_LIGHT, 5)
    out = run(po, pcam, s, lights, planes)
    assert (out[sky] == 0).all() and (out[~sky][:, 3] == 1).all()
    s = settings_for(abi.SCENE_HAS_SKY, 5)
    out = run(po, pcam, s, lights, planes)
    assert (out[sky] == np.float32([0.2, 0.4, 0.9, 1.0])).all()
    s.sky_has_texture = 1
    assert (run(po, pcam, s, lights, planes)[sky] == 1.0).all()
    # without HasSky the sky pixels run the full computation (at the far plane): lit, alpha 1
    s = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT, 5)
    out = run(po, pcam, s, lights, planes)
    assert (out[sky][:, 3] == 1).all() and (out[sky][:, :3] > 0).any() and not (out[sky] == np.float32([0.2, 0.4, 0.9, 1.0])).all(-1).any()


def test_flag_gating(po):
    """a NaN-filled shadow or contact plane changes nothing while its flag is off; NULL ambient occlusion and shadow read as 1"""
    rng = np.random.default_rng(3)
    pcam, planes = random_planes(rng, 48, 32)
    lights = mixed_lights(rng, 12)
    nan = np.full_like(planes["shadow"], np.nan)
    s = settings_for(abi.SCENE_HAS_SKY, 12)
    base = run(po, pcam, s, lights, planes, omit=("shadow", "contact_shadow"))
    np.testing.assert_array_equal(run(po, pcam, s, lights, dict(planes, shadow=nan, contact_shadow=nan)).view(np.uint32), base.view(np.uint32))
    s = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT, 12)
    base = run(po, pcam, s, lights, planes, omit=("contact_shadow",))
    np.testing.assert_array_equal(run(po, pcam, s, lights, dict(planes, contact_shadow=nan)).view(np.uint32), base.view(np.uint32))
    ones = np.ones_like(nan)
    np.testing.assert_array_equal(run(po, pcam, s, lights, planes, omit=("shadow", "ambient_occlusion")).view(np.uint32),
                                  run(po, pcam, s, lights, dict(planes, shadow=ones, ambient_occlusion=ones)).view(np.uint32))
    # and the planes are read when their flag is on
    s = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_CONTACT_SHADOWS, 12)
    assert np.isnan(run(po, pcam, s, lights, dict(planes, contact_shadow=nan))[planes["depth"] != 0][:, :3]).any()


def test_hostile_inputs_give_defined_bits(po):
    rng = np.random.default_rng(4)
    pcam, planes = random_planes(rng, 64, 40, hostile=True)
    lights = mixed_lights(rng, 40, hostile=True)
    s = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_CONTACT_SHADOWS, 40, rng)
    a, b = run(po, pcam, s, lights, planes), run(po, pcam, s, lights, {k: v.copy() for k, v in planes.items()})
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))
    nan = a.view(np.uint32)[np.isnan(a)]
    assert nan.size > 0 and (nan == 0x7FFFFFFF).all()


# ---- an independent binary64 restatement of pbr_apply_no_atmos.slang:23-127 and pbr.slang, vectorized over pixels ----------------

def _oct(e):
    v = np.stack([e[..., 0], e[..., 1], 1.0 - np.abs(e[..., 0]) - np.abs(e[..., 1])], -1)
    sgn = np.where(v[..., :2] >= 0, 1.0, -1.0)
    folded = (1.0 - np.abs(v[..., 1::-1])) * sgn
    v[..., :2] = np.where(v[..., 2:3] < 0, folded, v[..., :2])
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _dot(a, b):
    return (a * b).sum(-1)


def _ggx_albedo(x, y):
    c = np.float64([[0.1003, 0.9345, 1.0, 1.0], [-0.6303, -2.323, -1.765, 0.2281], [9.748, 2.229, 8.263, 15.94], [-2.038, -3.748, 11.53, -55.83],
                    [29.34, 1.424, 28.96, 13.08], [-8.245, -0.7684, -7.507, 41.26], [-26.44, 1.436, -36.11, 54.9], [19.99, 0.2913, 15.86, 300.2],
                    [-5.448, 0.6286, 33.37, -285.1]])
    t = np.stack([np.ones_like(x), x, y, x * y, x * x, y * y, x * x * y, x * y * y, x * x * y * y], -1) @ c
    return np.clip(t[..., 0] / t[..., 2], 0, 1), np.clip(t[..., 1] / t[..., 3], 0, 1)


def _brdf(V, N, L, albedo, rough, metal):
    VL = V + L
    H = VL / np.linalg.norm(VL, axis=-1, keepdims=True)
    NoV = np.abs(_dot(N, V)) + 1e-5
    NoL, NoH, LoH = (np.clip(_dot(a, b), 0, 1) for a, b in ((N, L), (N, H), (L, H)))
    F0 = 0.04 + (albedo - 0.04) * metal[..., None]
    alpha = np.maximum(rough * rough, 0.0025)
    a2 = alpha * alpha
    f = (NoH * a2 - NoH) * NoH + 1.0
    D = a2 / (np.pi * f * f + 1e-7)
    Vis = np.clip(0.5 / (NoL * np.sqrt(NoV * NoV * (1 - a2) + a2) + NoV * np.sqrt(NoL * NoL * (1 - a2) + a2) + 1e-7), 0, 1)
    F = F0 + (1 - F0) * (np.clip(1 - LoH, 0, 1) ** 5)[..., None]
    A, B = _ggx_albedo(NoV, alpha)
    Ess = np.clip(A + B, 0, 1)
    energy = 1 + F0 * ((1 - Ess) / np.maximum(Ess, 1e-4))[..., None]
    spec = (D * Vis)[..., None] * F * energy
    diff = (1 - metal)[..., None] * (1 - F) * albedo / np.pi
    return diff, spec


def restated(pcam, s, lights, planes):
    f64 = np.float64
    depth = planes["depth"].astype(f64)
    h, w = depth.shape
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    half = lambda a: a.astype(np.float16).astype(f64)  # noqa: E731
    albedo = planes["albedo"][..., :3].astype(f64)
    nrm = half(planes["normal"])
    N, smooth = _oct(nrm[..., :2]), _oct(nrm[..., 2:])
    mro = planes["metallic_roughness_occlusion"].astype(f64)
    metal, rough = np.clip(mro[..., 0], 0, 1), np.clip(mro[..., 1], 0.045, 1)
    occ = mro[..., 2] * half(planes["ambient_occlusion"])
    inv = np.asarray(pcam.inv_projection_view, f64).reshape(4, 4).T
    ndc = np.stack([(xs + 0.5) / w * 2 - 1, (ys + 0.5) / h * 2 - 1, depth, np.ones_like(depth)], -1) @ inv.T
    world = ndc[..., :3] / ndc[..., 3:]
    V = np.asarray(pcam.position, f64) - world
    V /= np.linalg.norm(V, axis=-1, keepdims=True)
    N = N / np.linalg.norm(N, axis=-1, keepdims=True)
    R = -V - 2 * N * _dot(-V, N)[..., None]
    NoV = np.abs(_dot(N, V)) + 1e-5
    Ls = np.asarray(s.sun_direction, f64)
    NoL = np.maximum(_dot(N, np.broadcast_to(Ls, N.shape)), 0)
    vis = planes["shadow"].astype(f64)
    env = np.asarray(s.base_ambient_color, f64)
    F0 = 0.04 + (albedo - 0.04) * metal[..., None]
    alpha = np.maximum(rough * rough, 0.0025)
    A, B = _ggx_albedo(NoV, alpha)
    kS = F0 * A[..., None] + B[..., None]
    kD = (1 - metal)[..., None] * (1 - kS)
    spec_occ = np.clip((NoV + occ) ** (2.0 ** (-16 * rough - 1)) - 1 + occ, 0, 1)
    indirect = kD * env * albedo / np.pi * occ[..., None] + kS * env * spec_occ[..., None]
    total = np.zeros_like(world)
    degenerate = np.zeros(depth.shape, bool)  # next to a light's range, cone edge or horizon, where binary32 rounding is amplified
    for L in lights:
        lv = np.asarray(L.position, f64) - world
        dist = np.linalg.norm(lv, axis=-1)
        Ld = lv / dist[..., None]
        att = np.maximum(0, 1 - (dist / L.range) ** 4) ** 2 / (dist * dist + 0.1)
        degenerate |= np.abs(1 - (dist / L.range) ** 4) < 1e-2
        if L.kind == abi.LIGHT_SPOT:
            sd = np.asarray(L.direction, f64)
            ca = _dot(-Ld, sd / np.linalg.norm(sd))
            ci, co = np.cos(f64(np.float32(L.inner_cone_angle))), np.cos(f64(np.float32(L.outer_cone_angle)))
            t = np.clip((ca - co) / (ci - co), 0, 1)
            att = att * t * t * (3 - 2 * t)
            degenerate |= (t > 0) & (t < 1e-2)
        elif L.kind != abi.LIGHT_POINT:
            continue
        NdotL = np.clip(_dot(N, Ld), 0, 1)
        degenerate |= np.abs(_dot(N, Ld)) < 1e-3
        d, sp = _brdf(V, N, Ld, albedo, rough, metal)
        c = (d + sp) * np.asarray(L.color, f64) * (att * L.intensity * NdotL)[..., None]
        total += np.where(((att > 0) & (NdotL > 0))[..., None], c, 0.0)
    horizon = np.clip(1 + 1.3 * _dot(R, smooth), 0, 1) ** 2
    d, sp = _brdf(V, N, np.broadcast_to(Ls, N.shape), albedo, rough, metal)
    surf = np.where((NoL > 0)[..., None], (d + sp * horizon[..., None]) * (s.sun_intensity * NoL * vis)[..., None], 0.0)
    return surf + total + indirect + planes["emissive"][..., :3].astype(f64), degenerate


@pytest.mark.parametrize("seed", range(3))
def test_binary64_restatement_agrees(po, seed):
    """the oracle agrees with an independent binary64 restatement on the finite, non-degenerate pixels holding depth (not next to a
    light's range, a cone edge or a light's horizon): 99 % of them to 1e-5 relative and every one to 3e-4 (binary32 rounding in the
    written order, amplified by D_GGX at small alpha, reaches a few 1e-5); a transcription error that the oracle and the kernel could
    share moves whole pixels by far more"""
    rng = np.random.default_rng(40 + seed)
    pcam, planes = random_planes(rng, 96, 64, yaw=9.0 * seed)
    planes["metallic_roughness_occlusion"] = np.clip(planes["metallic_roughness_occlusion"], 0.05, 1.0)
    # roughness >= 0.2: below it D_GGX's (NoH * alpha^2 - NoH) * NoH + 1 cancels at the highlight and binary32 keeps few digits
    planes["metallic_roughness_occlusion"][..., 1] = np.maximum(planes["metallic_roughness_occlusion"][..., 1], 0.2)
    lights = synth.make_lights(rng, (1, 16, 64)[seed], spot_fraction=0.5)
    s = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT, len(lights), rng)
    s.sun_direction[:] = [float(v) for v in np.float32(np.asarray(s.sun_direction) / np.linalg.norm(s.sun_direction))]
    got = run(po, pcam, s, lights, planes, omit=("contact_shadow",))[..., :3].astype(np.float64)
    want, degenerate = restated(pcam, s, lights, planes)
    held = (planes["depth"] != 0) & np.isfinite(want).all(-1) & ~degenerate
    assert held.sum() > 3000
    err = np.abs(got - want) / np.maximum(np.abs(want), 1e-3)
    assert np.isfinite(got[held]).all()
    assert np.quantile(err[held], 0.99) < 1e-5 and err[held].max() < 3e-4, np.quantile(err[held], [0.5, 0.99, 0.999, 1.0])
