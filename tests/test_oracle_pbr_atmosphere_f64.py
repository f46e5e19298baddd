"""An independent binary64 restatement of passes/pbr_apply.slang:26-184 and the functions it calls, in numpy, over LUTs the atmosphere
oracle makes at the reference's sizes and a cube the sky IBL oracle makes from them, against the atmospheric PBR oracle
(oracle/oxc_oracle_pbr_atmosphere.c).  It calls no function of that oracle.  Written from the shader text:
  pbr_apply.slang:57-83   the G-buffer reads (the normal plane and the AO rounded to binary16, as the R16 attachments hold them),
                          oct_to_vec3 (common/encoding.slang:7-15), the world position, V, N, R = reflect(-V, N), NoV, NoL
  :85-87                  visibility; :99-106 the sun's transmittance at get_eye_pos(world).y, horizon_darkening
  :108-124                the sky pixels: right / forward, light_on_plane, the planet hit from the camera's eye, sky.slang:39-67's uv
                          (altitude = eye.y), the sky-view tap, draw_sun (:26-38) without a planet hit, rgb * a
  :126-141                sample_aerial_perspective (sky.slang:258-293, per_slice_depth = size.x / size.z, near fade 1 / 0.001);
                          the cube taps at normalize(lerp(N, R, 1 - roughness)) and N
  :143-183                the indirect term, the sun's BRDF (pbr.slang:6-87) with the horizon term, the sum
The cube is sampled the way a seamless linear TextureCube filter does it, derived here from the geometry and not from the oracle's
integer table: a footprint texel off the face is the texel of the face its extended-plane centre projects onto, a corner texel the mean
of the three texels around it.  The taps are bilinear (trilinear for the aerial LUT) over the binary16 texels.  No point or spot lights:
those terms are the merged PBR oracle's (the reduction test of tests/test_oracle_pbr_atmosphere.py ties the two).
Comparison: a pixel away from every discrete decision must agree to REL of its value plus ABS of the frame's largest value; pixels near
a decision (the planet hit, the sun disc's edge, a cube face boundary, the aerial weight's knees) are counted and their share bounded,
and they are held to LOOSE.  Cameras at 2 m, 10 km and 200 km (above the atmosphere); suns above, at and below the horizon; the sun disc
in view."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_pbr import random_planes

REL, ABS, LOOSE = 2e-3, 2e-4, 0.05
NEAR_SHARE = 0.1
HEIGHTS = {"2m": 0.2, "10km": 1000.0, "200km": 20000.0}
SUNS = {"high": (0.3, 0.8, 0.52), "horizon": (0.9, 0.0, 0.43), "below": (0.5, -0.3, 0.81)}


def dot(a, b):
    return (a * b).sum(-1)


def normalize(v):
    return v / np.sqrt(dot(v, v))[..., None]


def cross(a, b):
    return np.cross(a, b)


def sat(x):
    return np.clip(np.nan_to_num(x, nan=0.0), 0.0, 1.0)


def smoothstep(e0, e1, x):
    t = sat((x - e0) / (e1 - e0))
    return t * t * (3 - 2 * t)


def tap2(lut, u, v):
    """linear-clamp bilinear of a float16 [H, W, 4] plane"""
    h, w = lut.shape[:2]
    a = lut.astype(np.float64)
    x, y = u * w - 0.5, v * h - 0.5
    x0, y0 = np.floor(x), np.floor(y)
    wx, wy = (x - x0)[..., None], (y - y0)[..., None]
    ix, iy = x0.astype(np.int64), y0.astype(np.int64)
    t = lambda i, j: a[np.clip(j, 0, h - 1), np.clip(i, 0, w - 1)]
    top = t(ix, iy) * (1 - wx) + t(ix + 1, iy) * wx
    bot = t(ix, iy + 1) * (1 - wx) + t(ix + 1, iy + 1) * wx
    return top * (1 - wy) + bot * wy


def tap3(lut, u, v, w):
    d = lut.shape[0]
    z = w * d - 0.5
    z0 = np.floor(z)
    wz = (z - z0)[..., None]
    iz = z0.astype(np.int64)
    s0 = np.stack([tap2(lut[k], u, v) for k in range(d)])  # [D, ..., 4]
    n = np.arange(s0.shape[1])
    a, b = s0[np.clip(iz, 0, d - 1), n], s0[np.clip(iz + 1, 0, d - 1), n]
    return a * (1 - wz) + b * wz


# the Vulkan cube face table: (sc, tc, ma) axes and signs per face
FACE_AXES = {0: ((2, -1), (1, -1), (0, 1)), 1: ((2, 1), (1, -1), (0, -1)), 2: ((0, 1), (2, 1), (1, 1)), 3: ((0, 1), (2, -1), (1, -1)),
             4: ((0, 1), (1, -1), (2, 1)), 5: ((0, -1), (1, -1), (2, -1))}


def select_face(r):
    ax, ay, az = np.abs(r[0]), np.abs(r[1]), np.abs(r[2])
    if ax >= ay and ax >= az:
        return 0 if r[0] >= 0 else 1
    if ay >= az:
        return 2 if r[1] >= 0 else 3
    return 4 if r[2] >= 0 else 5


def face_st(f, r):
    (si, ss), (ti, ts), (mi, _) = FACE_AXES[f]
    ma = abs(r[mi])
    return 0.5 * (ss * r[si] / ma) + 0.5, 0.5 * (ts * r[ti] / ma) + 0.5


def face_point(f, sc, tc):
    """the 3D point of (sc, tc) on face f's plane (extended past its edges)"""
    (si, ss), (ti, ts), (mi, ms) = FACE_AXES[f]
    p = np.zeros(3)
    p[si], p[ti], p[mi] = ss * sc, ts * tc, ms * 1.0
    return p


def cube_texel(cube, f, i, j):
    n = 32
    if 0 <= i < n and 0 <= j < n:
        return cube[f, j, i].astype(np.float64)
    if not (0 <= i < n) and not (0 <= j < n):
        ci, cj = min(max(i, 0), n - 1), min(max(j, 0), n - 1)
        return (cube_texel(cube, f, ci, cj) + cube_texel(cube, f, i, cj) + cube_texel(cube, f, ci, j)) / 3.0
    p = face_point(f, (2 * i + 1) / n - 1, (2 * j + 1) / n - 1)
    g = select_face(p)
    s, t = face_st(g, p)
    return cube[g, min(int(np.floor(t * n)), n - 1), min(int(np.floor(s * n)), n - 1)].astype(np.float64)


def cube_tap(cube, r):
    """seamless linear TextureCube sampling at direction r; also returns whether r lies near a face boundary"""
    if not np.all(np.isfinite(r)) or not np.any(r):
        return np.full(4, np.nan), True
    f = select_face(r)
    s, t = face_st(f, r)
    x, y = s * 32 - 0.5, t * 32 - 0.5
    x0, y0 = int(np.floor(x)), int(np.floor(y))
    wx, wy = x - x0, y - y0
    top = cube_texel(cube, f, x0, y0) * (1 - wx) + cube_texel(cube, f, x0 + 1, y0) * wx
    bot = cube_texel(cube, f, x0, y0 + 1) * (1 - wx) + cube_texel(cube, f, x0 + 1, y0 + 1) * wx
    m = np.sort(np.abs(r))
    return top * (1 - wy) + bot * wy, m[2] - m[1] <= 1e-5 * m[2]  # near a face boundary: binary32 may pick the other face


def oct_to_vec3(e):
    x, y = e[..., 0], e[..., 1]
    z = 1 - np.abs(x) - np.abs(y)
    sx, sy = np.where(x >= 0, 1.0, -1.0), np.where(y >= 0, 1.0, -1.0)
    nx = np.where(z < 0, (1 - np.abs(y)) * sx, x)
    ny = np.where(z < 0, (1 - np.abs(x)) * sy, y)
    return normalize(np.stack([nx, ny, z], -1))


def ggx_albedo(x, y):
    c = np.array([[0.1003, 0.9345, 1.0, 1.0], [-0.6303, -2.323, -1.765, 0.2281], [9.748, 2.229, 8.263, 15.94], [-2.038, -3.748, 11.53, -55.83],
                  [29.34, 1.424, 28.96, 13.08], [-8.245, -0.7684, -7.507, 41.26], [-26.44, 1.436, -36.11, 54.9], [19.99, 0.2913, 15.86, 300.2],
                  [-5.448, 0.6286, 33.37, -285.1]])
    x, y = x[..., None], y[..., None]
    r = c[0] + c[1] * x + c[2] * y + c[3] * x * y + c[4] * x * x + c[5] * y * y + c[6] * x * x * y + c[7] * x * y * y + c[8] * x * x * y * y
    return np.clip(r[..., 0] / r[..., 2], 0, 1), np.clip(r[..., 1] / r[..., 3], 0, 1)


def ray_sphere_hit(o, d, radius):
    a, b, c = dot(d, d), 2 * dot(d, o), dot(o, o) - radius * radius
    delta = b * b - 4 * a * c
    sq = np.sqrt(np.maximum(delta, 0))
    s0, s1 = (-b - sq) / (2 * a), (-b + sq) / (2 * a)
    return (delta >= 0) & ~((s0 < 0) & (s1 < 0)), delta / np.maximum(b * b, 1e-30)


def restate(pcam, s, at, planes, sky):
    """(rgb [H, W, 3], near-decision mask)"""
    tl, sv, ap, cube = sky
    h, w = planes["depth"].shape
    depth = planes["depth"].astype(np.float64)
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    u, v = (xs + 0.5) / w, (ys + 0.5) / h
    nrm = planes["normal"].astype(np.float16).astype(np.float64)
    mapped, smooth = oct_to_vec3(nrm[..., :2]), oct_to_vec3(nrm[..., 2:])
    alb = planes["albedo"][..., :3].astype(np.float64)
    em = planes["emissive"][..., :3].astype(np.float64)
    mro = planes["metallic_roughness_occlusion"].astype(np.float64)
    metallic, rough = np.clip(mro[..., 0], 0, 1), np.clip(mro[..., 1], 0.045, 1)
    occlusion = mro[..., 2] * planes["ambient_occlusion"].astype(np.float16).astype(np.float64)
    M = np.array(pcam.inv_projection_view[:], np.float64).reshape(4, 4).T
    hp = np.stack([2 * u - 1, 2 * v - 1, depth, np.ones_like(u)], -1) @ M.T
    world = hp[..., :3] / hp[..., 3:]
    cam = np.array(pcam.position[:], np.float64)
    V = normalize(cam - world)
    N = normalize(mapped)
    I = -V
    R = I - 2 * N * dot(I, N)[..., None]
    NoV = np.abs(dot(N, V)) + 1e-5
    L = np.array(s.sun_direction[:], np.float64)
    Li = float(s.sun_intensity)
    NoL = np.maximum(dot(N, L), 0)
    has_dir = bool(s.scene_flags & abi.SCENE_HAS_DIRECTIONAL_LIGHT)
    visibility = (planes["shadow"].astype(np.float64) if has_dir else 1.0) * (
        planes["contact_shadow"].astype(np.float64) if s.scene_flags & abi.SCENE_HAS_CONTACT_SHADOWS else 1.0)
    Rp, Ra = float(at.planet_radius), float(at.atmos_radius)
    min_alt = Rp + 0.001
    sun_cos = L[1]
    hd = smoothstep(-0.1, 0.3, sun_cos)
    # get_direct_sun_lighting at get_eye_pos(world).y (sky.slang:15-29 uv)
    px = np.maximum(world[..., 1] * 0.01 + min_alt, min_alt)
    py = sun_cos
    H_ = np.sqrt(max(Ra * Ra - Rp * Rp, 0))
    rho = np.sqrt(np.maximum(px * px - Rp * Rp, 0))
    d = np.maximum(0, -px * py + np.sqrt(np.maximum(px * px * (py * py - 1) + Ra * Ra, 0)))
    d_min, d_max = Ra - px, rho + H_
    T = tap2(tl, (d - d_min) / (d_max - d_min), rho / H_)[..., :3]
    direct = T * Li * hd
    out = np.zeros((h, w, 3))
    near = np.zeros((h, w), bool)
    sky_px = depth == 0
    # the sky pixels
    eye_y = max(float(pcam.position[1]) * 0.01 + min_alt, min_alt)
    eye = np.array([0.0, eye_y, 0.0])
    up = np.array([0.0, 1.0, 0.0])
    mv = -V[sky_px]
    right = normalize(cross(up, mv))
    fwd = normalize(cross(right, up))
    lop = np.stack([dot(fwd, L), dot(right, L)], -1)
    lop = lop / np.sqrt(dot(lop, lop))[..., None]
    vzc = mv[:, 1]
    hit, disc = ray_sphere_hit(eye, mv, Rp)
    horizon = np.sqrt(max(eye_y * eye_y - Rp * Rp, 0))
    beta = np.arccos(horizon / eye_y)
    zh = np.pi - beta
    vza = np.arccos(np.clip(vzc, -1, 1))
    vv = np.where(hit, np.sqrt(np.maximum((vza - zh) / beta, 0)) * 0.5 + 0.5, (1 - np.sqrt(np.maximum(1 - vza / zh, 0))) * 0.5)
    uu = (np.arctan2(-lop[:, 1], -lop[:, 0]) + np.pi) / (2 * np.pi)
    rw, rh = at.sky_view_lut_size[0], at.sky_view_lut_size[1]
    sv4 = tap2(sv, (uu + 0.5 / rw) * (rw / (rw + 1)), (vv + 0.5 / rh) * (rh / (rh + 1)))
    min_cos = np.cos(np.pi / 180)
    cth = dot(mv, L)
    off = min_cos - cth
    sun = np.where(cth >= min_cos, 1.0, np.exp(-off * 50000) * 0.5 + 1 / (0.02 + off * 300) * 0.01)
    rgb = sv4[:, :3] + np.where(hit, 0.0, sun * Li)[:, None] * T[sky_px]
    out[sky_px] = rgb * sv4[:, 3:]
    near[sky_px] = (np.abs(disc) < 1e-3) | (np.abs(cth - min_cos) < 1e-5) | (np.abs(np.abs(vzc) - 1) < 1e-6)
    # the surface pixels
    g = ~sky_px
    crp = (world[g] - cam) * 0.01
    lut = np.array(at.aerial_perspective_lut_size[:], np.float64)
    psd = lut[0] / lut[2]
    rel = np.maximum(0, np.sqrt(dot(crp, crp)) - float(at.aerial_perspective_start_km))
    lw = rel * (1 / psd) * (1 / lut[2])
    nlw = np.sqrt(lw)
    nls = nlw * lut[2]
    weight = np.where(nls < np.sqrt(0.5), sat(nls * nls * 2), 1.0) * sat(rel * (1 / 0.001))
    a4 = tap3(ap, u[g], v[g], nlw)
    a4[:, :3] *= weight[:, None]
    a4[:, 3] = 1 - weight * (1 - a4[:, 3])
    a4[:, :3] *= float(at.aerial_perspective_exposure)
    aerial = a4[:, :3] * a4[:, 3:]
    Ng, Rg = N[g], R[g]
    rd = normalize(Ng + (Rg - Ng) * (1 - rough[g])[:, None])
    spec, diff, edge = np.zeros((g.sum(), 4)), np.zeros((g.sum(), 4)), np.zeros(g.sum(), bool)
    for k in range(g.sum()):
        spec[k], e1 = cube_tap(cube, rd[k])
        diff[k], e2 = cube_tap(cube, Ng[k])
        edge[k] = e1 or e2
    spec_sky = spec[:, :3] * spec[:, 3:] * hd
    diff_sky = diff[:, :3] * diff[:, 3:] * hd
    albg, met, rgh, occ, nov = alb[g], metallic[g][:, None], rough[g], occlusion[g][:, None], NoV[g]
    F0 = 0.04 + (albg - 0.04) * met
    alpha = np.maximum(rgh * rgh, 0.0025)
    A, B = ggx_albedo(nov, alpha)
    kS = F0 * A[:, None] + B[:, None]
    kD = (1 - met) * (1 - kS)
    spec_occ = sat((nov + occ[:, 0]) ** (2.0 ** (-16 * rgh - 1)) - 1 + occ[:, 0])[:, None]
    indirect = kD * diff_sky * albg / np.pi * occ + kS * spec_sky * spec_occ
    hz = sat(1 + 1.3 * dot(Rg, smooth[g])) ** 2
    Vg = V[g]
    VL = Vg + L
    Hv = np.where((dot(VL, VL) > 1e-8)[:, None], normalize(VL), Ng)
    nol = sat(dot(Ng, L))
    noh, loh = sat(dot(Ng, Hv)), sat(dot(L, Hv))
    a2 = alpha * alpha
    f = (noh * a2 - noh) * noh + 1
    D = a2 / (np.pi * f * f + 1e-7)
    vis = sat(0.5 / (nol * np.sqrt(nov * nov * (1 - a2) + a2) + nov * np.sqrt(nol * nol * (1 - a2) + a2) + 1e-7))
    F = F0 + (1 - F0) * (sat(1 - loh) ** 5)[:, None]
    Ess = sat(A + B)
    energy = 1 + F0 * ((1 - Ess) / np.maximum(Ess, 1e-4))[:, None]
    specular = (D * vis)[:, None] * F * energy
    diffuse = (1 - met) * (1 - F) * albg / np.pi
    surf = np.where((NoL[g] > 0)[:, None], (diffuse + specular * hz[:, None]) * direct[g] * (NoL[g] * visibility[g] if np.ndim(visibility)
                                                                                            else NoL[g] * visibility)[:, None], 0.0)
    out[g] = surf + indirect + em[g] + aerial
    knee = (np.abs(nls - np.sqrt(0.5)) < 1e-4) | (np.abs(rel * 1000 - 1) < 1e-3) | (np.abs(dot(N[g], L)) < 1e-6)
    near[g] = edge | knee
    return out, near


_SKIES = {}


def oracle_sky(camera_y, sun):
    import pyoracle_atmosphere
    import pyoracle_sky_ibl

    key = (camera_y, tuple(sun))
    if key not in _SKIES:
        at = abi.atmosphere()
        cam = synth.pbr_camera(synth.make_camera(64, 64, 1))
        cam.position[1] = camera_y
        t = pyoracle_atmosphere.transmittance(at)
        sv, ap = pyoracle_atmosphere.sky_luts(at, cam, sun, 10.0, t)
        cube = None
        for f in range(2):
            cube = pyoracle_sky_ibl.sky_ibl(at, cam, sun, 10.0, abi.SKY_IBL_SUN_AMBIENT_STRENGTH, f, t, sv, cube)
        _SKIES[key] = (at, [t, sv, ap, cube])
    return _SKIES[key]


@pytest.fixture(scope="module")
def pa():
    import pyoracle_pbr_atmosphere

    pyoracle_pbr_atmosphere.build()
    return pyoracle_pbr_atmosphere


CASES = [(hk, sk) for hk in HEIGHTS for sk in SUNS] + [("2m", "in_view")]


@pytest.mark.parametrize("height,sun", CASES, ids=[f"{h}_{s}" for h, s in CASES])
def test_restatement_agrees(pa, height, sun):
    sdir = SUNS.get(sun)
    if sun == "in_view":  # the sun a little above the horizon straight ahead (the camera looks along -z): the disc on the sky pixels
        sdir = tuple(float(x) for x in np.float32([0.0, 0.12, -0.99]))
    at, sky = oracle_sky(HEIGHTS[height], sdir)
    rng = np.random.default_rng(31)
    pcam, planes = random_planes(rng, 160, 90)
    pcam.position[1] = HEIGHTS[height]
    s = abi.pbr_settings(scene_flags=abi.SCENE_HAS_ATMOSPHERE | abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_CONTACT_SHADOWS,
                         sun_direction=sdir, sun_intensity=10.0, light_count=0)
    got = pa.apply_pbr_atmosphere(pcam, s, at, None, *[planes[k] for k in abi.PBR_INPUTS], *sky)[..., :3].astype(np.float64)
    want, near = restate(pcam, s, at, planes, sky)
    scale = np.abs(want).max()
    err = np.abs(got - want).max(-1)
    ok = err <= REL * np.abs(want).max(-1) + ABS * scale
    assert np.isfinite(want).all() and np.isfinite(got).all()
    assert near.mean() <= NEAR_SHARE, near.mean()
    bad = ~ok & ~near
    assert bad.sum() == 0, (int(bad.sum()), float(err[bad].max()) if bad.any() else 0.0, float(scale))
    assert (err[near] <= LOOSE * scale).all()
    if sun == "in_view":
        sky_px = planes["depth"] == 0
        assert (want[sky_px].max(-1) > 0.5 * 10.0 * 0.02).any()  # some sky pixel shows the disc's glow
