"""Hand cases on the FXAA oracle (oracle/oxc_oracle_fxaa.c), the specification of include/oxcull.h oxc_fxaa: the constants' bits, frames
returned unchanged, step edges with the expected side and offset, the walk's reach and its break at every step, both outcomes of the variation test, the sub-pixel term, ClampToEdge
at the borders, degenerate extents, alpha, NaN and negative colours."""
import os
import re

import numpy as np
import pytest

from tests.test_gpu_fxaa import flat_frame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


@pytest.fixture(scope="module")
def so():
    import pyoracle_fxaa

    pyoracle_fxaa.build()
    return pyoracle_fxaa


def bits(x):
    return int(f32(x).view(np.uint32))


def test_constants_bits(so):
    """item 6: the oracle's binary32 literals and the device header's hex agree with the stated bits"""
    want = {"FXAA_EDGE_THRESHOLD_MIN": (0.0312, 0x3CFF9724), "FXAA_EDGE_THRESHOLD_MAX": (0.125, 0x3E000000),
            "FXAA_SUBPIXEL_QUALITY": (0.75, 0x3F400000), "FXAA_ONE_TWELFTH": (1.0 / 12.0, 0x3DAAAAAB)}
    src = open(f"{ROOT}/oxylus_b200/csrc/oxc_fxaa.cuh").read()
    table = so.constants()
    for k, (name, (decimal, b)) in enumerate(want.items()):
        m = re.search(rf"{name} = (\S+)f;", src)
        assert m, name
        assert bits(float.fromhex(m.group(1))) == b == bits(decimal) == bits(table[k]), name
    assert bits(f32(1.0) / f32(12.0)) == 0x3DAAAAAB  # the binary32 quotient equals the rounded binary64 one
    assert [so.quality(i) for i in range(12)] == [1, 1, 1, 1, 1, 1.5, 2, 2, 2, 2, 4, 8]


def test_constant_frame_unchanged(so):
    for value in ((0.8, 0.5, 0.3, 1.0), (100.0, 100.0, 100.0, 0.25), (0.0, 0.0, 0.0, 0.0)):
        f = flat_frame(13, 9, value)
        out, taps = so.fxaa(f, with_taps=True)
        np.testing.assert_array_equal(out, f)
        assert (taps == 5).all()


def test_below_threshold_unchanged(so):
    """a variation under max(0.0312, luma_max * 0.125) exits early: the output is the centre tap"""
    rng = np.random.default_rng(1)
    f = flat_frame(16, 12, (1.0, 1.0, 1.0, 1.0))
    f[..., :3] += rng.uniform(0, 0.2, (12, 16, 1)).astype(np.float32)  # luma range < 0.125 * luma_max ~ 0.13
    out, taps = so.fxaa(f, with_taps=True)
    assert (taps == 5).all()
    for y in range(12):
        for x in range(16):
            assert (out[y, x].view(np.uint32) == centre_tap(so, f, x, y).view(np.uint32)).all(), (x, y)


# the sub-pixel term of a pixel beside a straight edge: luma_average - center is a third of the range (the 3 x 3 weights 2, 2, 1, 1 on
# the far side), sub1 = 1 / 3, sub2 = (-2 / 3 + 3) / 9 = 7 / 27, sub_final = 0.75 * (7 / 27)^2
STRAIGHT_EDGE_SUB = 0.75 * (7.0 / 27.0) ** 2


def centre_tap(so, f, x, y):
    h, w = f.shape[:2]
    return so.tap(f, f32(f32(x + 0.5) / f32(w)), f32(f32(y + 0.5) / f32(h)))


@pytest.mark.parametrize("vertical", [True, False], ids=["vertical", "horizontal"])
def test_step_edge(so, vertical):
    """a long step edge between columns (rows) 15 and 16: only the two pixels beside it change, and none walks to an end (the edge is
    longer than the reach: 32 taps).  Both ends stay unreached, so distance1 = distance2 and pixel_offset = 0; the final offset is the
    sub-pixel term, toward the other side: the dark pixel moves STRAIGHT_EDGE_SUB of a texel toward the bright one and vice versa"""
    w, h = 32, 32
    f = flat_frame(w, h, (0.1, 0.1, 0.1, 1.0))
    if vertical:
        f[:, 16:, :3] = 2.0
    else:
        f[16:, :, :3] = 2.0
    out, taps = so.fxaa(f, with_taps=True)
    o = out if vertical else out.transpose(1, 0, 2)
    t = taps if vertical else taps.T
    changed = np.argwhere((o != (f if vertical else f.transpose(1, 0, 2))).any(axis=2))
    assert set(changed[:, 1].tolist()) <= {15, 16}
    dark, bright = o[:, 15, :3], o[:, 16, :3]
    np.testing.assert_allclose(dark, 0.1 + STRAIGHT_EDGE_SUB * 1.9, rtol=2e-5)
    np.testing.assert_allclose(bright, 2.0 - STRAIGHT_EDGE_SUB * 1.9, rtol=2e-5)
    assert (t[:, 15] == 32).all() and (t[:, 16] == 32).all()  # the walk never reaches an end of the edge: all 12 steps
    assert (t[:, :14] == 5).all() and (t[:, 18:] == 5).all()


def test_edge_ends_break_at_every_step(so):
    """a bright bar of length L on a dark row: the pixel below its left end reaches the left end at once and walks right until the
    bar ends; over L the walk's break lands after every step i = 2..11, which gives the one-sided tap counts 11 + i"""
    seen = set()
    for length in range(2, 40):
        f = flat_frame(64, 8, (0.02, 0.02, 0.02, 1.0))
        f[4:, 8:8 + length, :3] = 1.5
        _, taps = so.fxaa(f, with_taps=True)
        seen |= set(taps[3:5, 8:8 + length].ravel().tolist())
    assert set(range(13, 23)) <= seen


def test_correct_variation(so):
    """a horizontal edge, bright below (rows >= 16), seen from the dark pixel (17, 15).  The walk to the left runs out unreached; to the
    right it ends at column 20, the nearer end.  A: the bright side ends there, so the end reads dark like the centre: correct_variation
    is false, pixel_offset is dropped and the sub-pixel term alone moves the tap.  B: the dark side ends there, so the end reads the
    bright side: correct_variation is true and pixel_offset = 0.5 - distance2 / (distance1 + distance2) wins."""
    d, b = 0.1, 2.0
    a = flat_frame(40, 32, (d, d, d, 1.0))
    a[16:, :20, :3] = b
    out_a, taps_a = so.fxaa(a, with_taps=True)
    assert 13 < taps_a[15, 17] < 32  # the right end is reached within the walk
    np.testing.assert_allclose(out_a[15, 17, :3], d + STRAIGHT_EDGE_SUB * (b - d), rtol=2e-5)
    bb = flat_frame(40, 32, (b, b, b, 1.0))
    bb[:16, :20, :3] = d
    out_b = so.fxaa(bb)
    # in texels from the pixel centre 17.5: the right end is reached at step 3 on column 20, at 20.5 (distance2 = 3); the left walk runs
    # out unreached (the bright row continues, clamped at the border) at 17.5 - (1 + 1 + 1 + 1 + 1 + 1.5 + 2 * 4 + 4 + 8) = -9
    # (distance1 = 26.5); in A the same distances are formed and dropped
    offset = (out_b[15, 17, 0] - d) / (b - d)
    np.testing.assert_allclose(offset, 0.5 - 3.0 / (3.0 + 26.5), rtol=1e-4)


def test_isolated_bright_pixel(so):
    """one bright pixel on black: the sub-pixel term (luma_average far from the centre) wins and pulls the tap toward a neighbour"""
    f = flat_frame(9, 9, (0.0, 0.0, 0.0, 1.0))
    f[4, 4, :3] = 10.0
    out, taps = so.fxaa(f, with_taps=True)
    assert taps[4, 4] > 5
    assert 0.0 < out[4, 4, 0] < 10.0  # offset 0.75 * smoothstep(1)^2 = 0.75 of a texel toward a neighbour
    np.testing.assert_allclose(out[4, 4, 0], 2.5, rtol=1e-5)


def test_clamp_to_edge_at_the_borders(so):
    """taps beyond every border read the edge texel: a frame constant along each border's normal stays unchanged there, and the oracle
    tap at u < 0 or u > 1 equals the edge column"""
    rng = np.random.default_rng(3)
    f = rng.uniform(0, 2, (6, 5, 4)).astype(np.float32)
    for u, v, col, row in ((-0.5, 0.5 / 6, 0, 0), (1.5, 5.5 / 6, 4, 5), (0.5 / 5, -3.0, 0, 0), (4.5 / 5, 7.0, 4, 5)):
        np.testing.assert_allclose(so.tap(f, u, v), f[row, col], rtol=1e-6)
    np.testing.assert_allclose(so.tap(f, 0.5 / 5, 0.5 / 6, -1, -1), f[0, 0], rtol=1e-6)
    np.testing.assert_allclose(so.tap(f, 4.5 / 5, 5.5 / 6, 1, 1), f[5, 4], rtol=1e-6)
    stripes = np.repeat(rng.uniform(0, 4, (1, 12, 4)).astype(np.float32), 7, axis=0)  # vertical stripes, constant along y
    out = so.fxaa(stripes)
    assert np.isfinite(out).all()
    np.testing.assert_array_equal(out[0], out[3])
    np.testing.assert_array_equal(out[-1], out[3])


@pytest.mark.parametrize("w,h", [(1, 1), (1, 9), (9, 1)])
def test_degenerate_extents(so, w, h):
    rng = np.random.default_rng(w * 10 + h)
    f = rng.uniform(0, 4, (h, w, 4)).astype(np.float32)
    out, taps = so.fxaa(f, with_taps=True)
    assert np.isfinite(out).all() and ((taps == 5) | (taps >= 12)).all()
    if w == h == 1:
        np.testing.assert_array_equal(out, f)  # every tap reads the one texel


def test_alpha_follows_the_final_tap(so):
    """alpha is filtered like the colour: at an edge it blends with the neighbour's alpha"""
    f = flat_frame(16, 16, (0.0, 0.0, 0.0, 0.0))
    f[:, 8:] = (2.0, 2.0, 2.0, 1.0)
    out = so.fxaa(f)
    a = out[4:12, 7:9, 3]
    assert ((a > 0) & (a < 1)).all()
    np.testing.assert_array_equal(out[:, :6, 3], 0.0)


def test_nan_and_negative_colours(so):
    """a negative luma sum gives NaN (no error); a NaN pixel spreads only through the taps that read it; stored NaN is 0x7FFFFFFF"""
    assert np.isnan(so.luma(np.float32([-1.0, 0.0, 0.0])))
    assert so.luma(np.float32([1.0, 1.0, 1.0])) == f32(np.sqrt(f32(f32(f32(0.299) + f32(0.587)) + f32(0.114))))
    f = flat_frame(12, 12, (0.5, 0.5, 0.5, 1.0))
    f[6, 6, 0] = np.nan
    f[2, 2, :3] = -3.0
    out = so.fxaa(f)
    nan = np.isnan(out)
    assert nan.any() and (out.view(np.uint32)[nan] == 0x7FFFFFFF).all()
    assert not nan[:, 10:].any() and not nan[10:, :].any()
