"""An independent binary64 restatement of passes/sky_transmittance.slang, sky_view.slang and sky_aerial_perspective.slang with the
sky.slang / common/math.slang functions they call, written from the shader text in numpy, against the oracle
(oracle/oxc_oracle_atmosphere.c).  It bakes and taps its own transmittance LUT.  It stays below binary64 only where the reference does:
every LUT texel is stored as binary16 (RGBA16F), and the per-frame passes tap the binary16 transmittance texels.

The oracle runs binary32 with a binary32 exp, so the two agree within binary16 and accumulated-binary32 tolerances (below), except on
texels where a discrete decision goes the other way: a ray grazing the planet (planet intersection or not) or a march step on the
terminator (earth shadow or not).  Those texels are counted and bounded."""
import math

import numpy as np
import pytest

from oxylus_b200 import abi
from tests.test_gpu_atmosphere import SUNS, camera_for

PRO = 0.001   # PLANET_RADIUS_OFFSET
CSU = 0.01    # CAMERA_SCALE_UNIT


@pytest.fixture(scope="module")
def ao():
    import pyoracle_atmosphere

    pyoracle_atmosphere.build()
    return pyoracle_atmosphere


class Atm:
    def __init__(self, a):
        self.rs = np.float64(a.rayleigh_scatter[:])
        self.rd = float(a.rayleigh_density)
        self.ms = np.float64(a.mie_scatter[:])
        self.md, self.me, self.g = float(a.mie_density), float(a.mie_extinction), float(a.mie_asymmetry)
        self.oz = np.float64(a.ozone_absorption[:])
        self.oh, self.ot = float(a.ozone_height), float(a.ozone_thickness)
        self.R, self.A = float(a.planet_radius), float(a.atmos_radius)
        self.t_size = tuple(a.transmittance_lut_size[:2])
        self.sv_size = tuple(a.sky_view_lut_size[:2])
        self.ap_size = tuple(a.aerial_perspective_lut_size[:])

    def medium(self, alt):
        """(rayleigh scattering, mie scattering, extinction sum), each [..., 3]"""
        alt = alt[..., None]
        rs = self.rs * np.exp(-alt / self.rd)
        md = np.exp(-alt / self.md)
        ms = self.ms * md
        oz = self.oz * np.maximum(0.0, 1.0 - np.abs(alt - self.oh) / self.ot)
        return rs, ms, rs + self.me * md + oz


def ray_sphere_nearest(o, d, r):
    """(hit, t) of common/math.slang's ray_sphere_intersect_nearest, vectorised"""
    a = (d * d).sum(-1)
    b = 2.0 * (d * o).sum(-1)
    c = (o * o).sum(-1) - r * r
    delta = b * b - 4.0 * a * c
    sq = np.sqrt(np.maximum(delta, 0.0))
    s0, s1 = (-b - sq) / (2 * a), (-b + sq) / (2 * a)
    hit = (delta >= 0) & ~((s0 < 0) & (s1 < 0))
    t = np.where(s0 < 0, np.maximum(0, s1), np.where(s1 < 0, np.maximum(0, s0), np.maximum(0, np.minimum(s0, s1))))
    return hit, t


def bake(at):
    """sky_transmittance.slang: the LUT as the reference stores it, binary16 [H, W, 3]"""
    W, H = at.t_size
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    u, v = (xs + 0.5) / W, (ys + 0.5) / H
    h = math.sqrt(max(0.0, at.A ** 2 - at.R ** 2))
    rho = h * v
    lut_x = np.sqrt(rho * rho + at.R ** 2)
    d_min, d_max = at.A - lut_x, rho + h
    d = d_min + u * (d_max - d_min)
    with np.errstate(divide="ignore", invalid="ignore"):
        lut_y = np.clip(np.where(d == 0, 1.0, (h * h - rho * rho - d * d) / (2 * lut_x * d)), -1, 1)
    sun = np.stack([np.zeros_like(lut_y), np.sqrt(1 - lut_y ** 2), lut_y], -1)
    pos = np.stack([np.zeros_like(lut_x), np.zeros_like(lut_x), lut_x], -1)
    _, dist = ray_sphere_nearest(pos, sun, at.A)
    step = dist / 1000.0
    od = np.zeros(pos.shape)
    for _ in range(1000):
        pos = pos + sun * step[..., None]
        od += at.medium(np.linalg.norm(pos, axis=-1) - at.R)[2] * step[..., None]
    return np.exp(-od).astype(np.float16)


def tap(lut, u, v):
    H, W = lut.shape[:2]
    x, y = u * W - 0.5, v * H - 0.5
    x0, y0 = np.floor(x), np.floor(y)
    wx, wy = (x - x0)[..., None], (y - y0)[..., None]
    xa, xb = np.clip(x0, 0, W - 1).astype(int), np.clip(x0 + 1, 0, W - 1).astype(int)
    ya, yb = np.clip(y0, 0, H - 1).astype(int), np.clip(y0 + 1, 0, H - 1).astype(int)
    L = lut.astype(np.float64)
    top = L[ya, xa] + wx * (L[ya, xb] - L[ya, xa])
    bot = L[yb, xa] + wx * (L[yb, xb] - L[yb, xa])
    return top + wy * (bot - top)


def transmittance_uv(at, hh, c):
    H = math.sqrt(at.A ** 2 - at.R ** 2)
    rho = np.sqrt(np.maximum(0, hh * hh - at.R ** 2))
    d = np.maximum(0, -hh * c + np.sqrt(np.maximum(0, hh * hh * (c * c - 1) + at.A ** 2)))
    d_min, d_max = at.A - hh, rho + H
    return (d - d_min) / (d_max - d_min), rho / H


def draine(alpha, g, c):
    return (1 / (4 * math.pi)) * ((1 - g * g) / (1 + g * g - 2 * g * c) ** 1.5) * ((1 + alpha * c * c) / (1 + alpha / 3 * (1 + 2 * g * g)))


def mie_phase(g, c):
    g_hg = math.exp(-(0.0990567 / (g - 1.67154)))
    g_d = math.exp(-(2.20679 / (g + 3.91029)) - 0.428934)
    alpha = math.exp(3.62489 - (8.29288 / (g + 5.52825)))
    w_d = math.exp(-(0.599085 / (g - 0.641583)) - 0.665888)
    a, b = draine(0, g_hg, c), draine(alpha, g_d, c)
    return a + (b - a) * w_d


def integrate(at, lut, eye, d, sun, steps, t_max):
    """integrate_single_scattered_luminance for rays [N, 3] with one step count; also returns how many steps sat in the earth's
    shadow within 1e-4 km of its edge (the terminator decisions) and whether the planet test was within 1e-3 of tangent"""
    n = eye.shape[0]
    lum, T = np.zeros((n, 3)), np.ones((n, 3))
    inside = (eye * eye).sum(-1) > at.R ** 2
    ph, pt = ray_sphere_nearest(eye, d, at.R)
    if t_max is None:
        ah, atv = ray_sphere_nearest(eye, d, at.A)
        length = np.where(ph, np.maximum(0, pt), atv)
        active = inside & ah
    else:
        length = np.broadcast_to(t_max, (n,)).astype(np.float64)
        active = inside
    c = (sun * d).sum(-1)
    rp, mp = 3 / (16 * math.pi) * (1 + c * c), mie_phase(at.g, c)
    old = np.zeros(n)
    near_edge = np.zeros(n, bool)
    for s in range(steps):
        new = length * (s + 0.3) / steps
        sl = new - old
        old = new
        pos = eye + new[:, None] * d
        h = np.linalg.norm(pos, axis=-1)
        rs, ms, es = at.medium(h - at.R)
        up = pos / h[:, None]
        u, v = transmittance_uv(at, h, (sun * up).sum(-1))
        st = tap(lut, u, v)
        sp = ms * mp[:, None] + rs * rp[:, None]
        o = pos - PRO * up
        sh, _ = ray_sphere_nearest(o, sun, at.R)
        # the earth-shadow test's margin: distance of the sun ray's closest approach from the planet's surface
        tc = -(o * sun).sum(-1) / (sun * sun).sum(-1)
        closest = np.linalg.norm(o + np.maximum(tc, 0)[:, None] * sun, axis=-1) - at.R
        near_edge |= np.abs(closest) < 0.05
        sl_ = np.where(sh, 0.0, 1.0)[:, None] * st * sp
        stt = np.exp(-sl[:, None] * es)
        with np.errstate(divide="ignore", invalid="ignore"):
            integ = (sl_ - sl_ * stt) / es
        lum += np.where(active[:, None], 10.0 * integ * T, 0)
        T = np.where(active[:, None], T * stt, T)
    # grazing the planet: the closest approach of the view ray within 0.05 km of the surface
    tc = -(eye * d).sum(-1)
    graze = np.abs(np.linalg.norm(eye + np.maximum(tc, 0)[:, None] * d, axis=-1) - at.R) < 0.05
    return lum, T, near_edge | graze


def move_to_top(at, pos, d):
    h = np.linalg.norm(pos, axis=-1)
    hit, t = ray_sphere_nearest(pos, d, at.A)
    above = h > at.A
    moved = pos + d * t[:, None] - PRO * pos / h[:, None]
    return np.where(above[:, None], moved, pos), ~(above & ~hit)


def sky_view(at, lut, cam_y, sun):
    W, H = at.sv_size
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    u, v = ((xs + 0.5) / W).ravel(), ((ys + 0.5) / H).ravel()
    eye_y = max(cam_y * CSU + at.R + PRO, at.R + PRO)
    h = eye_y
    u, v = (u - 0.5 / W) * (W / (W - 1)), (v - 0.5 / H) * (H / (H - 1))
    beta = math.acos(math.sqrt(max(0, h * h - at.R ** 2)) / h)
    zha = math.pi - beta
    vza = np.where(v < 0.5, zha * (1 - (1 - 2 * v) ** 2), zha + beta * (2 * v - 1) ** 2)
    lon = u * 2 * math.pi
    d = np.stack([np.sin(vza) * np.cos(lon), np.cos(vza), np.sin(vza) * np.sin(lon)], -1)
    # the shader's sin from sqrt(1 - cos^2) with the sign of the angle: sin for vza in (0, pi], the sign of sin(lon) by lon <= pi
    eye = np.tile([0.0, eye_y, 0.0], (len(u), 1))
    eye, ok = move_to_top(at, eye, d)
    up = eye / h
    szc = (up * np.float64(sun)).sum(-1)
    sd = np.stack([np.sqrt(np.maximum(0, 1 - szc * szc)), szc, np.zeros_like(szc)], -1)
    sd /= np.linalg.norm(sd, axis=-1, keepdims=True)
    lum, _, flip = integrate(at, lut, eye, d, sd, 48, None)
    lum = np.where(ok[:, None], np.maximum(lum, 0), 0)
    return lum.reshape(H, W, 3), flip.reshape(H, W)


def aerial(at, lut, cam, sun):
    X, Y, Z = at.ap_size
    ys, xs = np.meshgrid(np.arange(Y), np.arange(X), indexing="ij")
    u, v = ((xs + 0.5) / X).ravel(), ((ys + 0.5) / Y).ravel()
    m = np.float64(cam.inv_projection_view[:]).reshape(4, 4).T
    ws = m @ np.stack([2 * u - 1, 2 * v - 1, np.ones_like(u), np.ones_like(u)])
    wp = (ws[:3] / ws[3]).T - np.float64(cam.position[:])
    d = wp / np.linalg.norm(wp, axis=-1, keepdims=True)
    eye_y = max(float(cam.position[1]) * CSU + at.R + PRO, at.R + PRO)
    out, T, flips = np.zeros((Z, Y * X, 3)), np.zeros((Z, Y * X)), np.zeros((Z, Y * X), bool)
    for z in range(Z):
        slice_ = ((z + 0.5) / Z) ** 2 * Z
        t_max = slice_ * float(X // Z)
        eye = np.tile([0.0, eye_y, 0.0], (len(u), 1))
        assert eye_y < at.A  # the restatement covers cameras inside the atmosphere
        lum, tr, flip = integrate(at, lut, eye, d, np.float64(sun), 2 * (z + 1), t_max)
        out[z], T[z], flips[z] = lum, tr.mean(-1), flip
    return out.reshape(Z, Y, X, 3), T.reshape(Z, Y, X), flips.reshape(Z, Y, X)


SIZES = dict(transmittance_lut_size=(64, 16, 1), sky_view_lut_size=(40, 24, 1), aerial_perspective_lut_size=(16, 8, 16))
# (camera height, sun, relative tolerance above the horizon, largest share of below-horizon texels off by more than 30 %)
CASES = [(0.2, "45deg", 2e-3, 0.35), (1000.0, "horizon", 2e-2, 0.0), (0.2, "zenith", 2e-3, 0.35)]


@pytest.mark.parametrize("height,sun,tol,decided", CASES, ids=["2m-45deg", "10km-horizon", "2m-zenith"])
def test_restatement_agrees(ao, height, sun, tol, decided):
    """Above the horizon the oracle's sky view and aerial perspective equal the restatement within `tol` relative (2e-3 at 2 m, the
    binary16 store and the binary32 march; 2e-2 with the sun on the horizon, whose march steps sit on the earth's shadow edge).  Rays
    into the ground from 2 m are decided in binary32 at a planet radius whose ulp is 0.49 m, so their few-metre paths and their
    earth-shadow tests differ from binary64: they are counted, and at most `decided` of them differ by more than 30 %."""
    a = abi.atmosphere(**SIZES)
    at = Atm(a)
    cam = camera_for(height, yaw=20.0)
    t_orc = ao.transmittance(a)
    sv_orc, ap_orc = ao.sky_luts(a, cam, SUNS[sun], 10.0, t_orc)
    lut = bake(at)
    # the transmittance LUTs: binary16 texels of a binary32 and a binary64 march.  The binary32 march adds the same step to a position of
    # about 6400 km 1000 times, each add rounding by up to ulp(6400) / 2 = 2.4e-4 km, so its sample altitudes drift by up to about
    # 0.1 km against the binary64 march (the reference's own binary32 behaviour): within 8e-3 (measured 5.4e-3)
    diff = np.abs(lut.astype(np.float64) - t_orc[..., :3].astype(np.float64))
    assert diff.max() <= 8e-3, diff.max()
    assert (t_orc[..., 3] == 1).all()
    # sky view: the decoded luminance rgb * m; rows v < 0.5 look above the horizon (uv_to_sky_view_lut_params puts it at v = 0.5)
    want, _ = sky_view(at, lut, cam.position[1], SUNS[sun])
    got = sv_orc[..., :3].astype(np.float64) * sv_orc[..., 3:].astype(np.float64)
    rel = (np.abs(got - want) / np.maximum(want, 1e-12)).max(-1)
    H = rel.shape[0]
    assert rel[: H // 2].max() <= tol, rel[: H // 2].max()
    assert want.max() > 1e-3 and np.isfinite(got).all() and (got >= 0).all()
    below = rel[H // 2:]
    assert (below > 0.3).mean() <= decided, (below > 0.3).mean()
    # aerial perspective: luminance and mean transmittance; its rows y < Y / 2 look above the horizon (the camera looks level)
    lum, T, _ = aerial(at, lut, cam, SUNS[sun])
    got = ap_orc[..., :3].astype(np.float64)
    rel = (np.abs(got - lum) / np.maximum(lum, 1e-12)).max(-1)
    Y = rel.shape[1]
    assert rel[:, : Y // 2].max() <= tol, rel[:, : Y // 2].max()
    assert np.abs(ap_orc[..., 3].astype(np.float64) - T).max() <= 1e-3
    below = rel[:, Y // 2:]
    assert (below > 0.3).mean() <= decided, (below > 0.3).mean()
