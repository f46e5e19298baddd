"""The GTAO oracle (oracle/oxc_oracle_gtao.c) pinned by hand: the Hilbert table, the R2 noise, fast_acos, the sector bitmask, the
linearization, the pyramid's weighted average and its virtual-pyramid rule at small sizes, the edges, the denoise's weights at the
borders, canonical_pow against binary64 and the trilinear weights."""
import os
import sys

import numpy as np
import pytest

from oxylus_b200 import abi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

f32 = np.float32


@pytest.fixture(scope="module")
def go():
    import pyoracle_gtao

    pyoracle_gtao.build()
    return pyoracle_gtao


def test_hilbert_table(go):
    """a bijection onto 0..4095 whose consecutive indices are grid neighbours, starting as the reference's curve does"""
    idx = np.array([[go.hilbert_index(x, y) for x in range(64)] for y in range(64)])
    assert sorted(idx.reshape(-1).tolist()) == list(range(4096))
    pos = np.zeros((4096, 2), int)
    for y in range(64):
        for x in range(64):
            pos[idx[y, x]] = (x, y)
    assert (np.abs(np.diff(pos, axis=0)).sum(1) == 1).all()
    assert [go.hilbert_index(x, y) for x, y in ((0, 0), (1, 0), (1, 1), (0, 1), (0, 2), (0, 3), (1, 3), (1, 2))] == [0, 1, 2, 3, 4, 5, 6, 7]
    assert go.hilbert_index(63, 0) == 4095


def test_r2_noise(go):
    for x, y, ni in ((0, 0, 0), (5, 9, 0), (70, 3, 0), (5, 9, 3), (5, 9, 67)):
        index = go.hilbert_index(x % 64, y % 64) + 288 * (ni % 64)
        fi = f32(index)
        want = [f32(f32(0.5) + fi * f32(0.75487766624669276005)), f32(f32(0.5) + fi * f32(0.5698402909980532659114))]
        want = [f32(v - np.floor(v)) for v in want]
        np.testing.assert_array_equal(go.noise(x, y, ni), np.float32(want))
    np.testing.assert_array_equal(go.noise(0, 0), [0.5, 0.5])
    np.testing.assert_array_equal(go.noise(70, 3, 64), go.noise(6, 3, 0))


def test_fast_acos(go):
    assert go.fast_acos(1.0) == 0.0
    assert go.fast_acos(-1.0) == f32(3.1415926535897932384626433832795)
    assert go.fast_acos(0.0) == f32(1.57079632679)
    res = f32(f32(f32(-0.156583) * f32(0.5)) + f32(1.57079632679)) * f32(np.sqrt(f32(0.5)))
    assert go.fast_acos(0.5) == res and go.fast_acos(-0.5) == f32(f32(3.1415926535897932384626433832795) - res)
    xs = np.linspace(-1.0, 1.0, 401)
    assert max(abs(go.fast_acos(x) - np.arccos(x)) for x in xs) < 1.1e-2  # the first-order approximation's own error


def test_update_sectors(go):
    assert go.update_sectors(0.3, 0.3, 0x1234) == 0x1234  # zero width: unchanged
    assert go.update_sectors(0.5, 0.2, 7) == 7            # negative width saturates to zero
    assert go.update_sectors(0.0, 1.0) == 0xFFFFFFFF       # the full arc
    assert go.update_sectors(1.0, 1.0) == 0                # start 32 clamps to 31 but the width is zero
    assert go.update_sectors(0.99, 1.0) == 0x80000000      # start 31, one sector
    assert go.update_sectors(0.0, 1.0 / 32) == 1
    assert go.update_sectors(0.25, 0.5) == 0x0000FF00      # sectors 8..15
    assert go.update_sectors(0.26, 0.5) == 0x0000FF00      # start truncates, the width 7.68 rounds up
    assert go.update_sectors(0.26, 0.52) == 0x0001FF00     # ceil: touching a sector activates it


def test_calc_sector_mask_both_directions(go):
    """a sample on the view ray whose back face stays on that ray spans no angle; a sample off to one side covers the sectors between
    its front and back horizons, in the lower half of the slice for sampling direction +1 and mirrored into the upper half for -1"""
    v = np.float32([0.0, 0.0, 1.0])
    assert go.calc_sector_mask(0.5, [0.0, 0.0, 1.0], v, 1.0, 0.0) == 0
    side = np.float32([0.2, 0.0, 1.0])  # front horizon acos(1 / sqrt(1.04)) = 0.197, back face (0.2, 0, 0.5): 0.381
    pos = go.calc_sector_mask(0.5, side, v, 1.0, 0.0)
    neg = go.calc_sector_mask(0.5, side, v, -1.0, 0.0)
    assert pos == 0x00003000 and neg == 0x000C0000  # [0.379, 0.437] * 32 and [0.563, 0.621] * 32
    assert go.calc_sector_mask(0.5, side, v, 1.0, 0.3) == 0x00018000  # the normal's angle n shifts the arc by n / pi


def test_linearize_near_and_far(go):
    proj = synth.perspective_reverse_z(60.0, 16 / 9, 0.1, 1000.0)
    assert abs(go.linearize(proj, 1.0) - 0.1) < 1e-6
    assert abs(go.linearize(proj, 0.0) - 1000.0) < 1e-2
    assert go.linearize(proj, 0.0) >= f32(1000.0) * f32(0.999)  # sky


def test_weighted_average(go):
    assert go.weighted_average(2.0, 2.0, 2.0, 2.0) == 2.0
    assert go.weighted_average(2.0, 2.0, 2.0, 50.0) == 2.0  # an outlier beyond the falloff has weight 0
    assert 2.0 < go.weighted_average(2.0, 2.0, 2.0, 2.2) < 2.2
    assert go.weighted_average(np.nan, 3.0, 3.0, 3.0) != go.weighted_average(np.nan, 3.0, 3.0, 3.0)  # NaN min skipped, NaN term stays


def _frame(go, depth, normals=None, preset=0):
    h, w = depth.shape
    proj, view = synth.camera_matrices(w, h)
    n = np.zeros((h, w, 4), np.float32) if normals is None else normals
    return go.generate_ambient_occlusion(abi.gtao_camera(proj, view, 1000.0), abi.gtao_settings(preset), depth, n), proj


def test_constant_image_gives_constant_mips(go):
    r, proj = _frame(go, np.full((40, 72), 0.01, np.float32))
    assert (r["mips"] == go.linearize(proj, 0.01)).all()


@pytest.mark.parametrize("w,h", [(1, 1), (3, 2), (17, 9)])
def test_virtual_pyramid_rule(go, w, h):
    """level k at t averages level k-1 at 2t .. 2t + (1, 1) of the pyramid continued past the extent by clamping level 0"""
    rng = np.random.default_rng(w * h)
    depth = rng.uniform(0.001, 0.05, (h, w)).astype(np.float32)
    r, proj = _frame(go, depth)
    lin = np.vectorize(lambda d: go.linearize(proj, d))(depth).astype(np.float32)

    def level(k, x, y):
        if k == 0:
            return lin[min(y, h - 1), min(x, w - 1)]
        return go.weighted_average(level(k - 1, 2 * x, 2 * y), level(k - 1, 2 * x + 1, 2 * y), level(k - 1, 2 * x, 2 * y + 1),
                                   level(k - 1, 2 * x + 1, 2 * y + 1))

    layout, total = abi.gtao_mip_layout(w, h)
    assert total == go.mip_offset(w, h, 5) and [o for o, _, _ in layout] == [go.mip_offset(w, h, k) for k in range(5)]
    for k, (off, lw, lh) in enumerate(layout):
        want = np.float32([[level(k, x, y) for x in range(lw)] for y in range(lh)])
        np.testing.assert_array_equal(r["mips"][off:off + lw * lh].reshape(lh, lw), want, err_msg=f"level {k}")


def test_edges(go):
    """a flat plane (constant linear depth) packs to 0xFFFFFFFF; a depth step zeroes the edge across it and keeps the others"""
    proj, _ = synth.camera_matrices(32, 16)
    d_near, d_far = proj[14] / f32(5.0) - proj[10], proj[14] / f32(9.0) - proj[10]
    r, _ = _frame(go, np.full((16, 32), d_near, np.float32))
    assert (r["edges"] == 0xFFFFFFFF).all()
    depth = np.full((16, 32), d_near, np.float32)
    depth[:, 16:] = d_far
    e = _frame(go, depth)[0]["edges"]
    left_of_step, right_of_step = e[8, 15], e[8, 16]
    assert (right_of_step >> 8) & 0xFF == 0 or (left_of_step >> 8) & 0xFF == 0  # right edge of the near side / left of the far
    assert left_of_step & 0xFF == 0xFF and (left_of_step >> 16) == 0xFFFF    # left, top, bottom stay connected
    assert e[8, 4] == 0xFFFFFFFF and e[8, 28] == 0xFFFFFFFF


def _unorm(p, i):
    return f32(f32((int(p) >> (8 * i)) & 0xFF) / f32(255.0))


def test_denoise_weights_and_borders(go):
    """the 3 x 3 weights from the edges, by hand, at an interior pixel and at all four borders and corners (clamp to edge)"""
    rng = np.random.default_rng(3)
    h, w = 5, 6
    noisy = rng.random((h, w)).astype(np.float16).view(np.uint16)
    edges = rng.integers(0, 2**32, (h, w), dtype=np.uint64).astype(np.uint32)

    def at(a, x, y):
        return a[min(max(y, 0), h - 1), min(max(x, 0), w - 1)]

    for x, y in ((2, 2), (0, 2), (w - 1, 2), (3, 0), (3, h - 1), (0, 0), (w - 1, h - 1)):
        ec, el, er, et, eb = at(edges, x, y), at(edges, x - 1, y), at(edges, x + 1, y), at(edges, x, y - 1), at(edges, x, y + 1)
        lw, rw = f32(_unorm(ec, 0) * _unorm(el, 1)), f32(_unorm(ec, 1) * _unorm(er, 0))
        tw, bw = f32(_unorm(ec, 2) * _unorm(et, 3)), f32(_unorm(ec, 3) * _unorm(eb, 2))
        k = f32(0.425)
        tl = f32(k * f32(f32(tw * _unorm(et, 0)) + f32(lw * _unorm(el, 2))))
        tr = f32(k * f32(f32(tw * _unorm(et, 1)) + f32(rw * _unorm(er, 2))))
        bl = f32(k * f32(f32(bw * _unorm(eb, 0)) + f32(lw * _unorm(el, 3))))
        br = f32(k * f32(f32(bw * _unorm(eb, 1)) + f32(rw * _unorm(er, 3))))
        taps = [((0, 0), f32(1.2)), ((-1, 0), lw), ((1, 0), rw), ((0, -1), tw), ((0, 1), bw), ((-1, -1), tl), ((1, -1), tr), ((-1, 1), bl),
                ((1, 1), br)]
        s, sw = f32(0.0), f32(0.0)
        for i, ((dx, dy), wt) in enumerate(taps):
            v = f32(np.uint16(at(noisy, x + dx, y + dy)).view(np.float16))
            s = f32(v * wt) if i == 0 else f32(s + f32(v * wt))
            sw = wt if i == 0 else f32(sw + wt)
        assert go.denoise_pixel(noisy, edges, x, y, 1.0) == f32(s / sw), (x, y)
        assert go.denoise_pixel(noisy, edges, x, y, 1.2) == go.pow_canonical(f32(s / sw), 1.2)


def test_canonical_pow(go):
    """within 1 ulp of the correctly rounded binary32 power (binary64 numpy.power, rounded) over 10^6 inputs, and its exact cases"""
    import ctypes as C

    lib = go.lib()
    rng = np.random.default_rng(9)
    x = np.exp2(rng.uniform(-24.0, 0.0, 1_000_000)).astype(np.float32)
    y = rng.uniform(0.25, 8.0, 1_000_000).astype(np.float32)
    fn = lib.orc_pow_canonical
    got = np.fromiter((fn(C.c_float(a), C.c_float(b)) for a, b in zip(x.tolist(), y.tolist())), np.float32, len(x))
    want = np.power(x.astype(np.float64), y.astype(np.float64)).astype(np.float32)
    ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    assert ulps.max() <= 1 and (ulps == 0).mean() > 0.999
    for yy in (0.25, 1.2, 8.0, -3.0, np.inf, np.nan):
        assert go.pow_canonical(1.0, yy) == 1.0
    for yy in (0.25, 1.2, 8.0, np.inf):
        assert go.pow_canonical(0.0, yy) == 0.0
    assert go.pow_canonical(0.37, 0.0) == 1.0 and go.pow_canonical(np.nan, 0.0) == 1.0
    assert go.pow_canonical(0.5, 2.0) == 0.25 and go.pow_canonical(0.25, 0.5) == 0.5
    assert np.isnan(go.pow_canonical(np.nan, 1.2)) and np.isnan(go.pow_canonical(0.5, np.nan)) and np.isnan(go.pow_canonical(-0.5, 2.0))
    assert go.pow_canonical(0.0, -1.0) == np.inf and go.pow_canonical(np.inf, 2.0) == np.inf and go.pow_canonical(np.inf, -2.0) == 0.0
    assert go.pow_canonical(0.5, np.inf) == 0.0 and go.pow_canonical(2.0, np.inf) == np.inf and go.pow_canonical(0.5, -np.inf) == np.inf
    assert go.pow_canonical(1e-30, 8.0) == 0.0 and go.pow_canonical(3e38, 8.0) == np.inf


def test_trilinear_weights_from_constant_levels(go):
    """a pyramid whose level k holds the constant c_k: SampleLevel reads (1 - f) * c_lo + f * c_hi anywhere, clamp included"""
    w, h = 37, 21
    layout, total = abi.gtao_mip_layout(w, h)
    c = np.float32([1.0, 3.0, 7.0, 20.0, 50.0])
    mips = np.zeros(total, np.float32)
    for k, (off, lw, lh) in enumerate(layout):
        mips[off:off + lw * lh] = c[k]
    for u, v, lam in ((0.5, 0.5, 0.0), (0.1, 0.9, 0.25), (-3.0, 2.0, 1.5), (0.99, 0.01, 2.75), (0.3, 0.3, 3.5), (0.3, 0.3, 4.0)):
        lo = int(np.floor(lam))
        hi = min(lo + 1, 4)
        f = f32(f32(lam) - f32(lo))
        want = f32(f32(f32(1.0) - f) * c[lo]) + f32(f * c[hi])
        assert go.sample_level(mips, w, h, u, v, lam) == f32(want), (u, v, lam)
    # a linear ramp in x at level 0 is reproduced at texel centres and clamped outside
    off, lw, lh = layout[0]
    ramp = np.tile(np.arange(lw, dtype=np.float32), (lh, 1))
    mips[off:off + lw * lh] = ramp.reshape(-1)
    assert go.sample_level(mips, w, h, (10 + 0.5) / w, 0.5, 0.0) == 10.0
    assert go.sample_level(mips, w, h, (10.5 + 0.5) / w, 0.5, 0.0) == 10.5
    assert go.sample_level(mips, w, h, -5.0, 0.5, 0.0) == 0.0 and go.sample_level(mips, w, h, 7.0, 0.5, 0.0) == lw - 1
