"""An independent binary64 restatement of eye adaptation and bloom, written from the shader text (passes/histogram_generate.slang,
histogram_average.slang, bloom_prefilter.slang, bloom_downsample.slang, bloom_upsample.slang and the samplers of PostProcess.cpp), against
the binary32 oracle (oracle/oxc_oracle_post.c).  Frames: lit frames of the PBR oracle over the PBR tests' G-buffer planes, and synthetic
HDR frames.  Bins agree except for pixels whose binary64 mapped value lies within 1e-4 of an integer (the oracle's log2 and its
binary32 rounding may put them on the other side); those are counted and bounded.  The exposure and every bloom level agree within the
stated tolerances."""
import numpy as np
import pytest

from oxylus_b200 import abi

EDGE = 1e-4  # pixels whose binary64 mapped value lies this close to a bin edge may land in the neighbouring bin


@pytest.fixture(scope="module")
def so():
    import pyoracle_post

    pyoracle_post.build()
    return pyoracle_post


def lit_frame(w, h, seed):
    import pyoracle_pbr

    from tests.test_gpu_pbr import mixed_lights, random_planes, settings_for

    pyoracle_pbr.build()
    rng = np.random.default_rng(seed)
    pcam, planes = random_planes(rng, w, h)
    lights = mixed_lights(rng, 8)
    s = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT, len(lights))
    p = planes
    return pyoracle_pbr.apply_pbr(pcam, s, lights, p["depth"], p["albedo"], p["normal"], p["emissive"], p["metallic_roughness_occlusion"])


def hdr_frame(w, h, seed):
    rng = np.random.default_rng(seed)
    lum = np.exp2(rng.normal(0.0, 4.0, (h, w, 1)))
    return np.concatenate([rng.uniform(0, 1, (h, w, 3)) * lum, np.ones((h, w, 1))], axis=2).astype(np.float32)


FRAMES = [("lit-96x64", lambda: lit_frame(96, 64, 1)), ("lit-161x90", lambda: lit_frame(161, 90, 2)), ("hdr-128x72", lambda: hdr_frame(128, 72, 3)),
          ("hdr-67x33", lambda: hdr_frame(67, 33, 4))]


# ---------------------------------------------------------------- eye adaptation in binary64

def mapped64(frame, s):
    rgb = frame[..., :3].astype(np.float64)
    lum = rgb[..., 0] * 0.2127 + rgb[..., 1] * 0.7152 + rgb[..., 2] * 0.0722
    with np.errstate(divide="ignore", invalid="ignore"):
        m = (np.log2(lum) - s.min_exposure) / (s.max_exposure - s.min_exposure) * (255.0 - 1.0) + 1.0
    return lum, m


def bins64(frame, s):
    lum, m = mapped64(frame, s)
    b = np.clip(np.trunc(np.nan_to_num(m, nan=0.0, posinf=255, neginf=0)), 0, 255).astype(np.int64)
    b[lum < 0.001] = 0
    return b


def record64(hist, s, w, h, dt, last):
    weighted = int((np.arange(256, dtype=np.uint64) * hist.astype(np.uint64)).sum()) % 2 ** 32
    avg = weighted / max(w * h - int(hist[0]), 1.0) - 1.0
    desired = 2.0 ** (avg / 254.0 * (s.max_exposure - s.min_exposure) + s.min_exposure)
    adapted = last + (desired - last) * (1.0 - np.exp(-s.adaptation_speed * dt))
    ev100 = np.log2(adapted * 100.0 * s.ev100_bias / 12.5)
    return adapted, 1.0 / (2.0 ** ev100 * 1.2)


@pytest.mark.parametrize("name", [n for n, _ in FRAMES])
def test_bins_and_record(so, name):
    frame = dict(FRAMES)[name]()
    h, w = frame.shape[:2]
    s = abi.eye_adaptation_settings()
    rec, hist = so.eye_adaptation(frame, s, 0.1, abi.Exposure(1.0, 1.0))
    lum, m = mapped64(frame, s)
    b64 = bins64(frame, s)
    b32 = np.array([so.histogram_bin(s, *px[:3]) for px in frame.reshape(-1, 4)]).reshape(h, w)
    assert np.array_equal(np.bincount(b32.ravel(), minlength=256), hist)
    with np.errstate(invalid="ignore"):
        near = (np.abs(m - np.round(m)) < EDGE) | (np.abs(lum - 0.001) < 1e-9)
    differ = b32 != b64
    assert not (differ & ~near).any(), f"{int((differ & ~near).sum())} pixels differ away from a bin edge"
    assert int(near.sum()) <= max(3, w * h // 500), f"{int(near.sum())} pixels within {EDGE} of an edge"
    a64, e64 = record64(np.bincount(b64.ravel(), minlength=256), s, w, h, float(np.float32(0.1)), 1.0)
    assert abs(rec.adapted_luminance - a64) <= 1e-5 * abs(a64) + 1e-3 * abs(a64) * int(differ.sum())
    assert abs(rec.exposure - e64) <= 1e-5 * abs(e64) + 1e-3 * abs(e64) * int(differ.sum())


# ---------------------------------------------------------------- bloom in binary64

def tap64(src, u, v, border):
    """SampleLevel(linear, uv, 0).rgb of src [H, W, 3] at arrays u, v: ClampToBorder (transparent black) or ClampToEdge"""
    H, W = src.shape[:2]
    x, y = u * W - 0.5, v * H - 0.5
    x0, y0 = np.floor(x), np.floor(y)
    wx, wy = (x - x0)[..., None], (y - y0)[..., None]
    x0, y0 = x0.astype(np.int64), y0.astype(np.int64)

    def fetch(xi, yi):
        t = src[np.clip(yi, 0, H - 1), np.clip(xi, 0, W - 1)]
        if border:
            t = np.where(((xi < 0) | (xi >= W) | (yi < 0) | (yi >= H))[..., None], 0.0, t)
        return t

    top = fetch(x0, y0) * (1 - wx) + fetch(x0 + 1, y0) * wx
    bot = fetch(x0, y0 + 1) * (1 - wx) + fetch(x0 + 1, y0 + 1) * wx
    return top * (1 - wy) + bot * wy


def grid(w, h):
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    return (xs + 0.5) / w, (ys + 0.5) / h, 1.0 / w, 1.0 / h


OFF13 = [(-2, 2), (0, 2), (2, 2), (-2, 0), (0, 0), (2, 0), (-2, -2), (0, -2), (2, -2), (-1, 1), (1, 1), (-1, -1), (1, -1)]


def bloom64(frame, s, exposure):
    src = frame[..., :3].astype(np.float64)
    h, w = frame.shape[:2]
    lv = abi.bloom_levels(w, h)
    u, v, tu, tv = grid(lv[0][0], lv[0][1])
    t = [tap64(src, u + tu * dx, v + tv * dy, True) for dx, dy in OFF13]
    a, b, c, d, e, f, g, hh, i, j, k, l, m = t
    cs, ws = 0.0, 0.0
    for grp in ((a, b, d, e), (b, c, e, f), (d, e, g, hh), (e, f, hh, i), (j, k, l, m)):
        gv = np.minimum(sum(grp) * 0.25 * exposure, s.clamp_value)
        weight = 1.0 / (1.0 + gv @ np.array([0.299, 0.587, 0.114]))
        br = gv.max(axis=-1)
        knee = s.threshold * s.soft_threshold
        soft = np.clip(br - s.threshold + knee, 0.0, 2.0 * knee)
        soft = soft * soft * 0.25 / (knee + 1e-5)
        contrib = np.maximum(soft, br - s.threshold) / np.maximum(br, 1e-5)
        cs = cs + gv * contrib[..., None] * weight[..., None]
        ws = ws + weight
    down = [cs / (ws + 1e-5)[..., None]]
    for lw, lh, _ in lv[1:]:
        u, v, tu, tv = grid(lw, lh)
        t = [tap64(down[-1], u + tu * dx, v + tv * dy, True) for dx, dy in OFF13]
        a, b, c, d, e, f, g, hh, i, j, k, l, m = t
        down.append((a + c + g + i) * 0.03125 + (b + d + f + hh) * 0.0625 + (e + j + k + l + m) * 0.125)
    up = [None] * len(lv)
    for n in range(len(lv) - 1, 0, -1):
        srcl = down[n] if n == len(lv) - 1 else up[n]
        lw, lh, _ = lv[n - 1]
        u, v, tu, tv = grid(lw, lh)
        t = [tap64(srcl, u + tu * dx, v + tv * dy, False) for dx, dy in ((-1, 1), (0, 1), (1, 1), (-1, 0), (0, 0), (1, 0), (-1, -1), (0, -1), (1, -1))]
        a, b, c, d, e, f, g, hh, i = t
        tent = e * 0.25 + (b + d + f + hh) * 0.125 + (a + c + g + i) * 0.0625
        base = tap64(down[n - 1], u, v, False)
        up[n - 1] = base + (tent - base) * s.radius
    return down, up


@pytest.mark.parametrize("name", [n for n, _ in FRAMES])
@pytest.mark.parametrize("flags", [0, abi.SCENE_HAS_EYE_ADAPTATION])
def test_bloom_levels(so, name, flags):
    """every level of both chains within 2e-5 of the level's largest value plus 1e-4 relative; the knee's clamp and the
    max(brightness) choice are continuous, so no texel flips between branches by more than that"""
    frame = dict(FRAMES)[name]()
    h, w = frame.shape[:2]
    s = abi.bloom_settings(scene_flags=flags)
    record = abi.Exposure(0.3, 2.5)
    down32, up32 = so.bloom(frame, s, record)
    down64, up64 = bloom64(frame, s, float(np.float32(2.5)) if flags else 1.0)
    lv = abi.bloom_levels(w, h)
    for k, (lw, lh, off) in enumerate(lv):
        got = down32[off:off + lw * lh, :3].reshape(lh, lw, 3).astype(np.float64)
        scale = np.abs(down64[k]).max() + 1e-30
        assert np.all(np.abs(got - down64[k]) <= 2e-5 * scale + 1e-4 * np.abs(down64[k])), f"downsampled level {k}"
        if k < len(lv) - 1:
            got = up32[off:off + lw * lh, :3].reshape(lh, lw, 3).astype(np.float64)
            scale = np.abs(up64[k]).max() + 1e-30
            assert np.all(np.abs(got - up64[k]) <= 2e-5 * scale + 1e-4 * np.abs(up64[k])), f"upsampled level {k}"
    assert (down64[0] > 0).mean() > 0.01  # the threshold leaves something to bloom
