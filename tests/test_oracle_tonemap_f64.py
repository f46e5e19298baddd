"""An independent binary64 restatement of the tonemap pass, written from passes/tonemap.slang (fs_main, ACES_Fitted, AgX_DS with
color_PrimariesToMatrix / color_ComputeCompressionMatrix / inverse, GT7ToneMapping with the ICtCp UCS), passes/lens.slang and
common/color.slang, not from the oracle: vectorised numpy, binary64 throughout with numpy's exp / log2 / power / cos, except two
kinds of position, formed in binary32 in the shader's order: the texture coordinates the sampler receives (with the chromatic
aberration's magnitudes that place them) and the sampler's texel
position and bilinear weights (a last-bit shift of a coordinate moves the weights, and on an HDR frame neighbours differ by 2^16, so
such a shift changes the sampled value itself, not only the arithmetic after it) and the film grain's simplex point, which the shader's round() makes discontinuous (the hash is
integer arithmetic either way).  It is compared with the oracle (oracle/oxc_oracle_tonemap.c) per curve on random HDR frames with
every flag group and on the component defaults.  Tolerances are absolute plus relative, per curve, and stated below, the relative part
of the larger of the value and the 3 x 3 texels around it; they hold the binary32 rounding of the oracle's chain and its canonical
transcendentals (within 1 ulp each), amplified by the PQ exponents in GT7.  The worst pixel reaches about 0.25 (none), 0.15 (ACES),
0.03 (AgX) and 0.65 (GT7) of its tolerance."""
import numpy as np
import pytest

from oxylus_b200 import abi
from tests.test_gpu_post import hdr_frame

EA, BL = abi.SCENE_HAS_EYE_ADAPTATION, abi.SCENE_HAS_BLOOM
CA, VG, FG, TB = abi.SCENE_HAS_CHROMATIC_ABERRATION, abi.SCENE_HAS_VIGNETTE, abi.SCENE_HAS_FILM_GRAIN, abi.SCENE_TRANSPARENT_BACKGROUND
F = np.float32
# (absolute, relative) tolerance of |oracle - restatement| per curve
TOLERANCE = {abi.TONEMAP_NONE: (1e-6, 2e-6), abi.TONEMAP_ACES: (2e-6, 1e-5), abi.TONEMAP_AGX: (5e-6, 2e-5), abi.TONEMAP_GT7: (3e-5, 2e-4)}


@pytest.fixture(scope="module")
def so():
    import pyoracle_tonemap

    pyoracle_tonemap.build()
    return pyoracle_tonemap


# ---------------------------------------------------------------- binary64 restatement

def tap(plane, u, v):
    """SampleLevel with linear filtering and Repeat: [..., 4] at binary32 coordinates u, v (arrays); the texel position and the
    weights are the sampler's, binary32, the blend binary64"""
    H, W = plane.shape[:2]
    x, y = np.asarray(u, F) * F(W) - F(0.5), np.asarray(v, F) * F(H) - F(0.5)
    x0, y0 = np.floor(x), np.floor(y)
    wx, wy = (x - x0).astype(np.float64)[..., None], (y - y0).astype(np.float64)[..., None]
    x0, y0 = x0.astype(np.float64), y0.astype(np.float64)
    c0, c1 = np.mod(x0, W).astype(np.int64), np.mod(x0 + 1, W).astype(np.int64)
    r0, r1 = np.mod(y0, H).astype(np.int64), np.mod(y0 + 1, H).astype(np.int64)
    top = plane[r0, c0] * (1 - wx) + plane[r0, c1] * wx
    bot = plane[r1, c0] * (1 - wx) + plane[r1, c1] * wx
    return top * (1 - wy) + bot * wy


def mv(m, c):
    return np.einsum("ij,...j->...i", m, c)


def aces(c):
    c = mv(np.array([[0.59719, 0.35458, 0.04823], [0.07600, 0.90834, 0.01566], [0.02840, 0.13383, 0.83777]]), c)
    c = (c * (c + 0.0245786) - 0.000090537) / (c * (0.983729 * c + 0.4329510) + 0.238081)
    c = mv(np.array([[1.60475, -0.53108, -0.07367], [-0.10208, 1.10813, -0.00605], [-0.00327, -0.07276, 1.07602]]), c)
    return np.clip(c, 0, 1)


def primaries(r, g, b, w):
    un = lambda p: np.array([p[0] / p[1], 1.0, (1 - p[0] - p[1]) / p[1]])
    R, G, B, Wt = un(r), un(g), un(b), un(w)
    s = np.linalg.inv(np.array([[R[0], G[0], B[0]], [1, 1, 1], [R[2], G[2], B[2]]])) @ Wt
    return np.column_stack([R * s[0], G * s[1], B * s[2]])


def agx(c):
    xy = [np.array([0.64, 0.33]), np.array([0.3, 0.6]), np.array([0.15, 0.06])]
    w = np.array([0.3127, 0.3290])
    srgb_to_xyz = primaries(*xy, w)
    sf = 1 / (1 - 0.15)
    adjusted_to_xyz = primaries(*[w + (p - w) * sf for p in xy], w)
    m = srgb_to_xyz @ np.linalg.inv(adjusted_to_xyz)  # mul(sRGB_to_XYZ, XYZ_to_adjusted), as written
    c = mv(m, np.maximum(c, 0))
    S = 0.1
    c = np.clip(np.where(c < S, c, 1 - (1 - S) * np.exp(-(1 / (1 - S)) * (c - S))), 0, 1)
    d = (c @ np.array([0.2126729, 0.7151522, 0.0721750]))[..., None]
    c = np.clip(d + (c - d) * 1.3, 0, 1)
    return mv(np.linalg.inv(m), c)


M1, M2, C1, C2, C3 = 0.1593017578125, 78.84375, 0.8359375, 18.8515625, 18.6875


def inv_eotf(v):
    with np.errstate(invalid="ignore", divide="ignore"):
        ym = np.power(v * 100 / 10000, M1)
        return 2 ** (M2 * (np.log2(C1 + C2 * ym) - np.log2(1 + C3 * ym)))


def eotf(n):
    n = np.clip(n, 0, 1)
    np_ = np.power(n, 1 / M2)
    l = np.maximum(np_ - C1, 0) / (C2 - C3 * np_)
    return np.power(l, 1 / M1) * 10000 / 100


def to_ictcp(c):
    lms = mv(np.array([[1688, 2146, 262], [683, 2951, 462], [99, 309, 3688]]) / 4096, c)
    pq = inv_eotf(lms)
    return mv(np.array([[2048, 2048, 0], [6610, -13613, 7003], [17933, -17390, -543]]) / 4096, pq)


def from_ictcp(u):
    lms = eotf(mv(np.array([[1, 0.00860904, 0.11103], [1, -0.00860904, -0.11103], [1, 0.560031, -0.320627]]), u))
    return np.maximum(mv(np.array([[3.43661, -2.50645, 0.0698454], [-0.79133, 1.9836, -0.192271], [-0.0259499, -0.0989137, 1.12486]]), lms), 0)


def smooth_step(x, e0, e1):
    t = (x - e0) / (e1 - e0)
    return np.where(x < e0, 0.0, np.where(x > e1, 1.0, t * t * (3 - 2 * t)))


def gt7_curve(x):
    peak, alpha, mid, lin, toe = 2.5, 0.25, 0.538, 0.444, 1.280
    k = (lin - 1) / (alpha - 1)
    ka, kb, kc = peak * lin + peak * k, -peak * k * np.exp(lin / k), -1 / (k * peak)
    wl = smooth_step(x, 0, mid)
    xs = np.maximum(x, 0)
    toe_v = (1 - wl) * mid * np.power(xs / mid, toe) + wl * xs
    return np.where(x < 0, 0.0, np.where(x < lin * peak, toe_v, ka + kb * np.exp(xs * kc)))


def gt7(c):
    to_xyz = np.array([[0.4124564, 0.3575761, 0.1804375], [0.2126729, 0.7151522, 0.0721750], [0.0193339, 0.1191920, 0.9503041]])
    xyz_to_709 = np.array([[3.2404542, -1.5371385, -0.4985314], [-0.9692660, 1.8760108, 0.0415560], [0.0556434, -0.2040259, 1.0572252]])
    from_2020 = np.array([[0.636958, 0.1446169, 0.168881], [0.2627002, 0.6779981, 0.0593017], [0.0, 0.0280727, 1.0609851]])
    xyz_to_2020 = np.array([[1.7166512, -0.3556708, -0.2533663], [-0.6666844, 1.6164812, 0.0157685], [0.0176399, -0.0427706, 0.9421031]])
    rgb = mv(xyz_to_2020, mv(to_xyz, c))
    ucs = to_ictcp(rgb)
    skewed = gt7_curve(rgb)
    skewed_ucs = to_ictcp(skewed)
    target_ucs = to_ictcp(np.full(3, 2.5))[0]
    chroma = 1 - smooth_step(ucs[..., 0] / target_ucs, 0.98, 1.16)
    scaled = from_ictcp(np.stack([skewed_ucs[..., 0], ucs[..., 1] * chroma, ucs[..., 2] * chroma], -1))
    out = 0.4 * np.minimum(0.4 * skewed + 0.6 * scaled, 2.5)
    return mv(xyz_to_709, mv(from_2020, out))


CURVES = {abi.TONEMAP_NONE: lambda c: c, abi.TONEMAP_ACES: aces, abi.TONEMAP_AGX: agx, abi.TONEMAP_GT7: gt7}


def pcg3d16(v0, v1, v2):
    m = np.uint64(0xFFFFFFFF)
    v = [(np.asarray(x, np.uint64) * np.uint64(12829) + np.uint64(47989)) & m for x in (v0, v1, v2)]
    for _ in range(2):
        v[0] = (v[0] + v[1] * v[2]) & m
        v[1] = (v[1] + v[2] * v[0]) & m
        v[2] = (v[2] + v[0] * v[1]) & m
    return [x >> np.uint64(16) for x in v]


def restate(frame, s, record, bloom):
    """fs_main for every pixel of a float32 [H, W, 4] frame, in binary64"""
    H, W = frame.shape[:2]
    f64 = frame.astype(np.float64)
    y, x = np.mgrid[0:H, 0:W]
    u, v = (x.astype(F) + F(0.5)) / F(W), (y.astype(F) + F(0.5)) / F(H)
    src = tap(f64, u, v)
    flags = s.scene_flags
    c = src[..., :3] * (record.exposure if flags & EA else s.exposure)
    if flags & BL:
        c = c + tap(bloom.astype(np.float64), u, v)[..., :3] * s.bloom_intensity
    c = CURVES[s.tonemap_type](c)
    cx, cy = W // 2, H // 2
    if flags & CA:
        A, B = F(1.5220), F(0.00459) * F(s.chromatic_aberration_amount)  # FfxLensGetRGMag: the magnitudes place taps too
        n = lambda wl: A + B / (F(wl) * F(wl))
        rm, gm = (n(0.612) - F(1)) / (n(0.464) - F(1)), (n(0.549) - F(1)) / (n(0.464) - F(1))
        rx, ry = F(1) / F(2 * cx), F(1) / F(2 * cy)
        shift = lambda mag: (((x - cx).astype(F) * mag + F(cx) + F(0.5)) * rx, ((y - cy).astype(F) * mag + F(cy) + F(0.5)) * ry)
        c = np.stack([tap(f64, *shift(rm))[..., 0], tap(f64, *shift(gm))[..., 1], tap(f64, x.astype(F) * rx, y.astype(F) * ry)[..., 2]], -1)
    if flags & VG:
        m = np.cos(np.abs(x - cx) / cx * s.vignette_amount * np.pi / 4) ** 4 * np.cos(np.abs(y - cy) / cy * s.vignette_amount * np.pi / 4) ** 4
        c = c * np.clip(m, 0, 1)[..., None]
    if flags & FG:
        d = int(np.trunc(s.film_grain_scale / 8))
        q = (lambda a: np.full(a.shape, 0xFFFFFFFF, np.uint64)) if d == 0 else (lambda a: (np.trunc(a / d).astype(np.int64) & 0xFFFFFFFF).astype(np.uint64))
        h = pcg3d16(q(x), q(y), np.full(x.shape, s.film_grain_seed, np.uint64))
        # the simplex point in binary32, the shader's order
        sc = F(s.film_grain_scale)
        px, py = x.astype(F) / sc + (h[0].astype(F) * F(2 ** -16) - F(0.5)), y.astype(F) / sc + (h[1].astype(F) * F(2 ** -16) - F(0.5))
        f2, g2 = (np.sqrt(F(3)) - F(1)) / F(2), (F(3) - np.sqrt(F(3))) / F(6)
        uu = (px + py) * f2
        ix, iy = np.rint(px + uu), np.rint(py + uu)
        w = (ix + iy) * g2
        fx, fy = (px - (ix - w)).astype(np.float64), (py - (iy - w)).astype(np.float64)
        grain = (1 - 2 * 2 ** (-np.sqrt(fx * fx + fy * fy) * 3))[..., None]
        c = c + grain * np.minimum(c, 1 - c) * s.film_grain_amount
    alpha = src[..., 3:] if flags & TB else np.ones((H, W, 1))
    return np.concatenate([c, alpha], -1)


# ---------------------------------------------------------------- the comparison

def compare(so, frame, s, record, bloom, label):
    got = so.tonemap(frame, s, record, bloom).astype(np.float64)
    want = restate(frame, s, record, bloom)
    atol, rtol = TOLERANCE[s.tonemap_type]
    err = np.abs(got - want)
    # the taps blend neighbours in binary32 (off the texel centre at odd extents and under chromatic aberration): their rounding
    # scales with the largest texel of the 3 x 3 around, and the curves' slopes are at most about 1
    a = np.abs(frame.astype(np.float64))
    near = np.max([np.roll(np.roll(a, dy, 0), dx, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1)], axis=0)
    scale = np.maximum(np.abs(want), near)
    bound = atol + rtol * scale
    assert np.isfinite(want).all(), label
    assert (err <= bound).all(), f"{label}: worst {np.max(err / bound):.3g} of the tolerance"
    return float(np.max(err / bound))


@pytest.mark.parametrize("tonemap_type", [abi.TONEMAP_NONE, abi.TONEMAP_ACES, abi.TONEMAP_AGX, abi.TONEMAP_GT7],
                         ids=["none", "aces", "agx", "gt7"])
def test_restatement_equals_the_oracle(so, tonemap_type):
    rng = np.random.default_rng(100 + tonemap_type)
    worst = 0.0
    for w, h in ((48, 30), (37, 21)):
        frame = hdr_frame(rng, w, h)
        bloom = (hdr_frame(rng, w // 2, h // 2) * np.float32(0.25)).astype(np.float32)
        record = abi.Exposure(0.5, float(np.float32(rng.uniform(0.1, 3.0))))
        for flags in (0, EA | BL, EA | BL | VG | FG | TB, CA | VG | FG, EA | BL | CA | VG | FG):
            s = abi.tonemap_settings(flags, tonemap_type, exposure=float(np.float32(rng.uniform(0.2, 2.0))), film_grain_seed=int(rng.integers(16)))
            worst = max(worst, compare(so, frame, s, record, bloom, f"{w}x{h} flags {flags:#x}"))
        # the component defaults: AgX's reference curve aside, every default the pass reads
        s = abi.tonemap_settings(EA | BL | CA | VG | FG, tonemap_type)
        worst = max(worst, compare(so, frame, s, record, bloom, f"{w}x{h} defaults"))
    assert worst > 0.0  # the two do differ in the last bits
