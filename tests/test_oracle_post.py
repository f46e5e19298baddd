"""The eye-adaptation and bloom oracle (oracle/oxc_oracle_post.c) against the specification in include/oxcull.h, pinned by hand: the
constants' bits, every bin boundary (min / max exposure, the 0.001 threshold, NaN, +-inf, negative and subnormal pixels), the mod-2^32
weighted sum, a ten-call adaptation sequence, the mip count, odd level extents, border and clamp taps at every edge, the single-level
chain and a constant frame's bloom."""
import math
import os
import re

import numpy as np
import pytest

from oxylus_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN, INF = float("nan"), float("inf")
f32 = np.float32


@pytest.fixture(scope="module")
def so():
    import pyoracle_post

    pyoracle_post.build()
    return pyoracle_post


def bits(x):
    return int(np.float32(x).view(np.uint32))


def test_constants_bits():
    """the literals' binary32 bits, as the header states them and the device header writes them"""
    src = open(f"{ROOT}/oxylus_b200/csrc/oxc_exposure.cuh").read() + open(f"{ROOT}/oxylus_b200/csrc/oxc_bloom.cuh").read()
    want = {"HISTOGRAM_LUM_R": (0.2127, 0x3E59CE07), "HISTOGRAM_LUM_G": (0.7152, 0x3F371759), "HISTOGRAM_LUM_B": (0.0722, 0x3D93DD98),
            "LUMINANCE_EPSILON": (0.001, 0x3A83126F), "EXPOSURE_K": (1.2, 0x3F99999A), "BLOOM_LUM_R": (0.299, 0x3E991687),
            "BLOOM_LUM_G": (0.587, 0x3F1645A2), "BLOOM_LUM_B": (0.114, 0x3DE978D5), "BLOOM_EPS": (1e-5, 0x3727C5AC)}
    for name, (decimal, b) in want.items():
        m = re.search(rf"{name} = (\S+)f;", src)
        assert m, name
        assert bits(float.fromhex(m.group(1))) == b == bits(decimal), name


def test_bin_boundaries(so):
    s = abi.eye_adaptation_settings()
    # NaN / inf / negative / subnormal / zero / below the threshold
    assert so.histogram_bin(s, NAN, 0, 0) == 0
    assert so.histogram_bin(s, 0, NAN, NAN) == 0
    assert so.histogram_bin(s, INF, 0, 0) == 255
    assert so.histogram_bin(s, INF, -INF, 0) == 0  # inf - inf = NaN luminance
    assert so.histogram_bin(s, -INF, 0, 0) == 0
    assert so.histogram_bin(s, -5.0, 0, 0) == 0
    assert so.histogram_bin(s, 1e-45, 1e-40, 0) == 0
    assert so.histogram_bin(s, 0, 0, 0) == 0
    # the 0.001 threshold on the blue channel alone: lum = b * 0.0722
    eps = f32(0.001)
    b_at = f32(eps / f32(0.0722))
    while f32(b_at * f32(0.0722)) < eps:
        b_at = np.nextafter(b_at, f32(1))
    below = np.nextafter(b_at, f32(0))
    assert f32(below * f32(0.0722)) < eps <= f32(b_at * f32(0.0722))
    assert so.histogram_bin(s, 0, 0, below) == 0
    assert so.histogram_bin(s, 0, 0, b_at) >= 1  # log2(0.001) = -9.97 > -11.5: mapped > 1
    # luminances 2^e through the green channel: the bin is the truncated remap of log2, within one bin of the exact value
    for e in range(-9, 18):
        g = f32(2.0 ** e) / f32(0.7152)
        lum = f32(f32(g) * f32(0.7152))
        got = so.histogram_bin(s, 0, g, 0)
        mapped = (math.log2(lum) + 11.5) / 29.5 * 254 + 1
        assert abs(got - min(max(math.trunc(mapped), 0), 255)) <= 1, (e, got, mapped)
    # around min and max: a settings window where the threshold does not interfere
    w = abi.eye_adaptation_settings(2.0, 6.0, 1.1, 1.0)
    assert so.histogram_bin(w, 0, 0, f32(3.99) / f32(0.0722)) == 0       # log2 < min: mapped < 1
    assert so.histogram_bin(w, 0, 0, f32(4.0) / f32(0.0722)) in (0, 1)   # at min: mapped = 1 up to log2's error
    assert so.histogram_bin(w, 0, 0, f32(4.2) / f32(0.0722)) >= 1
    assert so.histogram_bin(w, 0, 0, f32(63.0) / f32(0.0722)) in (253, 254)
    assert so.histogram_bin(w, 0, 0, f32(64.5) / f32(0.0722)) == 255     # above max
    assert so.histogram_bin(w, 0, 0, f32(1e30)) == 255
    # NaN settings: every pixel in bin 0; min == max: division by zero, +inf -> 255, below -> 0
    assert so.histogram_bin(abi.eye_adaptation_settings(NAN, 18.0), 1.0, 1.0, 1.0) == 0
    assert so.histogram_bin(abi.eye_adaptation_settings(3.0, 3.0), 0, 0, f32(100.0) / f32(0.0722)) == 255
    assert so.histogram_bin(abi.eye_adaptation_settings(3.0, 3.0), 0, 0, f32(1.0)) == 0
    # alpha is not read
    frame = np.float32([[[1.0, 2.0, 3.0, NAN], [1.0, 2.0, 3.0, -INF]]])
    _, hist = so.eye_adaptation(frame, s, 0.016, abi.Exposure(1.0, 1.0))
    assert hist.sum() == 2 and hist.max() == 2


def test_weighted_sum_wraps_mod_2_32(so):
    """bins with 16,843,010 pixels in bin 255: weighted = 255 * 16,843,010 = 2^32 + 254, so f32(weighted) = 254"""
    s = abi.eye_adaptation_settings()
    consts = so.constants(s, 4096, 4112, 0.5)
    bins = np.zeros(256, np.uint32)
    bins[255] = 16843010
    wrapped = so.histogram_average(bins, consts, s.min_exposure, abi.Exposure(1.0, 1.0))
    # the same record from a histogram whose weighted sum is 254 without wrapping: one pixel in bin 254, the rest in bin 0 would change
    # the dark count; use the formula directly
    pc = consts[0]
    avg = f32(f32(f32(254) / max(f32(pc - f32(0)), f32(1))) - f32(1))
    desired = 2.0 ** float(f32(f32(f32(avg / f32(254)) * consts[1]) + f32(s.min_exposure)))
    adapted = f32(f32(1) + f32(f32(f32(desired) - f32(1)) * consts[2]))
    assert abs(wrapped.adapted_luminance - adapted) <= abs(adapted) * 2 ** -22
    bins[255] = 16843009  # 255 * 16,843,009 = 2^32 - 1: no wrap
    no_wrap = so.histogram_average(bins, consts, s.min_exposure, abi.Exposure(1.0, 1.0))
    assert no_wrap.adapted_luminance > 1.0 > wrapped.adapted_luminance


def test_constants_item_1(so):
    s = abi.eye_adaptation_settings()
    c = so.constants(s, 3840, 2160, 0.016)
    assert c[0] == f32(3840 * 2160) and c[1] == f32(f32(18.0) - f32(-11.5))
    assert bits(c[3]) == bits(f32(f32(100.0) * f32(1.0)) / f32(12.5))
    assert abs(float(c[2]) - (1 - math.exp(-float(f32(1.1)) * float(f32(0.016))))) < 2e-7
    assert so.constants(s, 4, 4, 0.0)[2] == 0.0
    assert so.constants(s, 4, 4, INF)[2] == 1.0
    assert so.constants(s, 16777217, 1, 0.0)[0] == f32(16777216)  # f32(u32) rounds to nearest even
    assert math.isnan(so.constants(s, 4, 4, NAN)[2])


def test_adaptation_sequence(so):
    """ten calls with varying delta_time: dt = 0 keeps the record, dt = inf jumps to the desired luminance, the exposure follows
    1 / (2^log2(adapted * 8) * 1.2)"""
    s = abi.eye_adaptation_settings()
    rng = np.random.default_rng(2)
    frame = (np.exp2(rng.normal(0.0, 2.0, (40, 60, 1))) * np.ones((1, 1, 4))).astype(np.float32)
    rec = abi.Exposure(1.0, 1.0)
    dts = [0.016, 0.0, 0.033, 1.0, INF, 0.016, 1e-3, 0.25, 0.0, 0.1]
    seen = []
    for dt in dts:
        prev = abi.Exposure.from_buffer_copy(rec)
        rec, hist = so.eye_adaptation(frame, s, dt, rec)
        if dt == 0.0:
            assert rec.adapted_luminance == prev.adapted_luminance
        if dt == INF:
            infinite = rec.adapted_luminance
            again, _ = so.eye_adaptation(frame, s, INF, abi.Exposure(123.0, 1.0))
            # time_coeff = 1: the desired luminance whatever came before, up to the rounding of last + (desired - last)
            assert abs(again.adapted_luminance - infinite) <= infinite * 2 ** -22
        assert abs(rec.exposure - 1.0 / (rec.adapted_luminance * 8.0 * 1.2)) <= rec.exposure * 1e-5
        seen.append(rec.adapted_luminance)
    assert len(set(seen)) >= 4  # the frame does not change: after dt = inf the record stays at the desired luminance
    # with dt = inf the desired luminance is 2^((avg / 254) * range + min), avg the mean bin minus one over non-dark pixels
    _, hist = so.eye_adaptation(frame, s, INF, abi.Exposure(1.0, 1.0))
    avg = (np.arange(256) * hist).sum() / (hist.sum() - hist[0]) - 1
    assert abs(infinite - 2.0 ** (avg / 254 * 29.5 - 11.5)) <= infinite * 1e-5


def test_mip_count_against_log2f(so):
    """the bit length equals the reference's u32(log2f(f32(m))) + 1 for every m in 1..16384"""
    m = np.arange(1, 16385, dtype=np.uint32)
    ref = np.floor(np.log2(m.astype(np.float32))).astype(np.uint32) + 1
    for k in range(len(m)):
        assert so.level_count(2 * int(m[k]), 2) == ref[k] == abi.bloom_levels(2 * int(m[k]), 2).__len__()
    assert so.level_count(1920, 1080) == 10 and so.level_count(3840, 2160) == 11
    from oxylus_b200 import capi  # the library's size helpers (no device needed)

    lib = capi.load()
    for w, h in ((2, 2), (3, 3), (4, 2), (1921, 1079), (2, 1000), (1920, 1080), (3840, 2160), (32768, 7), (1, 1)):
        assert lib.oxc_bloom_level_count(w, h) == len(abi.bloom_levels(w, h)) == so.level_count(w, h)
        assert lib.oxc_bloom_chain_texels(w, h) == abi.bloom_chain_texels(w, h)
    assert so.level_count(3, 3) == 1 and so.level_count(2, 2) == 1 and so.level_count(4, 2) == 2


def test_level_extents_of_odd_sizes():
    assert [(w, h) for w, h, _ in abi.bloom_levels(1921, 1079)] == [(960, 539), (480, 269), (240, 134), (120, 67), (60, 33), (30, 16), (15, 8),
                                                                      (7, 4), (3, 2), (1, 1)]
    assert [(w, h) for w, h, _ in abi.bloom_levels(2, 1000)] == [(1, 500), (1, 250), (1, 125), (1, 62), (1, 31), (1, 15), (1, 7), (1, 3),
                                                                   (1, 1)]
    assert abi.bloom_chain_texels(3, 2) == 1
    lv = abi.bloom_levels(37, 29)
    assert lv[0] == (18, 14, 0) and lv[1] == (9, 7, 252) and abi.bloom_chain_texels(37, 29) == sum(w * h for w, h, _ in lv)


def test_border_and_clamp_taps(so):
    """a 3 x 2 plane: inside, taps are the bilinear blend; outside each edge, border reads 0 and clamp reads the edge texel"""
    p = np.zeros((2, 3, 4), np.float32)
    p[..., 0] = [[1, 2, 3], [4, 5, 6]]
    p[..., 1] = 10.0
    # texel centres: exact
    for y in range(2):
        for x in range(3):
            u, v = (x + 0.5) / 3, (y + 0.5) / 2
            for border in (0, 1):
                assert so.tap(p, u, v, border)[0] == p[y, x, 0]
    # half a texel past each edge: border blends with 0, clamp returns the edge
    edges = {"left": (0.0, 0.25, 1.0, 0.5), "right": (1.0, 0.25, 3.0, 1.5), "top": (0.5 / 3, 0.0, 1.0, 0.5),
             "bottom": (0.5 / 3, 1.0, 4.0, 2.0)}
    for name, (u, v, clamp_r, border_r) in edges.items():
        assert so.tap(p, u, v, False)[0] == pytest.approx(clamp_r, abs=1e-6), name
        assert so.tap(p, u, v, True)[0] == pytest.approx(border_r, abs=1e-6), name
        assert so.tap(p, u, v, True)[1] == pytest.approx(5.0, abs=1e-5), name
    # corners: border keeps a quarter of the corner texel
    assert so.tap(p, 0.0, 0.0, True)[0] == pytest.approx(0.25, abs=1e-6)
    assert so.tap(p, 1.0, 1.0, False)[0] == 6.0
    # far outside: border 0, clamp the nearest corner; NaN coordinates are NaN-safe
    assert (so.tap(p, -5.0, 7.0, True) == 0).all() and so.tap(p, -5.0, 7.0, False)[0] == 4.0
    assert np.isnan(so.tap(p, NAN, 0.5, False)[0])


def test_single_level_chain(so):
    for w, h in ((2, 2), (3, 3), (3, 2), (2, 3)):
        frame = np.random.default_rng(w * h).normal(size=(h, w, 4)).astype(np.float32) * 10
        down, up = so.bloom(frame, abi.bloom_settings(), None, np.full((1, 4), 7.0, np.float32))
        assert down.shape == (1, 4) and down[0, 3] == 1.0
        np.testing.assert_array_equal(up, np.float32([[0, 0, 0, 1]]))


def test_constant_frame(so):
    """a constant grey frame c: away from the border, the prefilter's five groups are c * exposure (clamped), the downsample's weights
    sum to 1 and the tent's too, so every interior texel of every large level is the prefiltered value"""
    c, clamp, thr, knee_f = 2.0, 4.0, 1.0, 0.125
    frame = np.broadcast_to(np.float32([c, c, c, 1.0]), (256, 512, 4)).copy()
    for exposure, flags in ((1.0, 0), (0.5, abi.SCENE_HAS_EYE_ADAPTATION)):
        s = abi.bloom_settings(thr, knee_f, clamp, 0.75, flags)
        down, up = so.bloom(frame, s, abi.Exposure(1.0, exposure))
        g = min(c * exposure, clamp)
        knee = thr * knee_f
        soft = min(max(g - thr + knee, 0.0), 2 * knee) ** 2 * 0.25 / (knee + 1e-5)
        contrib = max(soft, g - thr) / max(g, 1e-5)
        want = g * contrib * 5 * (1 / (1 + g)) / (5 * (1 / (1 + g)) + 1e-5)
        lv = abi.bloom_levels(512, 256)
        for k in range(3):
            w, h, off = lv[k]
            level = down[off:off + w * h].reshape(h, w, 4)
            np.testing.assert_allclose(level[8:-8, 8:-8, :3], want, rtol=1e-5)
            assert (level[..., 3] == 1).all()
            assert level[0, 0, 0] < want  # the border's transparent black darkens the edge
        # the upsampled image is lerp(want, tent of the smaller levels, 0.75); those levels are darkened by the border throughout
        w, h, off = lv[0]
        inner = up[:w * h].reshape(h, w, 4)[8:-8, 8:-8, :3]
        assert (inner <= want * (1 + 1e-5)).all() and (inner >= 0.25 * want * (1 - 1e-5)).all()
