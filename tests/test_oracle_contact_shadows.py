"""The contact-shadow oracle (oracle/oxc_oracle_contact_shadows.c) pinned by hand: the step-count rule, the frustum clips of the ray,
the nearest and bilinear taps, smoothstep(1, 0.3, .), the bias constant, the output range on hostile frames, and analytic scenes (a box
on a plane, a lone plane)."""
import os
import sys

import numpy as np
import pytest

from oxylus_b200 import abi
from tests.test_gpu_contact_shadows import box_on_plane, contact_camera_for, random_depth, random_settings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

f32 = np.float32


@pytest.fixture(scope="module")
def co():
    import pyoracle_contact_shadows

    pyoracle_contact_shadows.build()
    return pyoracle_contact_shadows


def test_bias_constant(co):
    """(1.0 + bias) is fl(1 + fl(2e-6)) = 1 + 17 ulps; rounding 1.000002 once from binary64 gives the same bits"""
    b = co.bias_factor()
    assert b.view(np.uint32) == 0x3F800011
    assert b == f32(1.0) + f32(2e-6) == f32(1.000002)


@pytest.mark.parametrize("steps,end_x,want", [(1, 0.5, 2), (2, 0.5, 2), (8, 0.5, 8), (64, 0.5, 25), (64, 0.9, 45), (8, 0.01, 2), (64, 0.03, 2)])
def test_step_count(co, steps, end_x, want):
    """max(2, min(steps, floor(length of the ray in pixels))) on a 100 x 100 frame: a clip-space x of 0.5 is 25 px; rays shorter
    than 2 px take 2 steps whatever the setting"""
    assert co.step_count((0.0, 0.0, 0.5), (end_x, 0.0, 0.5), 100, 100, steps) == want


def test_step_count_of_a_pixel(co):
    """orc_cs_pixel reports the step count it marched: the default 8 on a long ray, 64 on a long ray with 64 steps"""
    ccam, proj = contact_camera_for(160, 90)
    depth = random_depth(np.random.default_rng(1), 160, 90, proj, hostile=False)
    for steps in (1, 2, 8, 64):
        _, n, _, _ = co.pixel(ccam, abi.contact_shadow_settings((1.0, 0.1, 0.0), steps, 0.1, 50.0), depth, 80, 80)
        assert n == max(2, steps)


def test_clip_keeps_a_ray_inside_the_frustum(co):
    s, e = co.clip_ray((0.1, -0.2, 0.5), (0.4, 0.3, 0.6))
    np.testing.assert_allclose(s, (0.1, -0.2, 0.5), atol=1e-7)
    np.testing.assert_allclose(e, (0.4, 0.3, 0.6), atol=1e-7)


def test_clip_end_at_the_far_edges(co):
    """the end is pulled back to the first far edge it crosses: x = 1 here, then z = 1 (reversed Z: depth 1 is the near plane)"""
    s, e = co.clip_ray((0.0, 0.0, 0.5), (3.0, 0.0, 0.5))
    np.testing.assert_allclose(s, (0.0, 0.0, 0.5), atol=1e-7)
    np.testing.assert_allclose(e, (1.0, 0.0, 0.5), atol=1e-6)
    s, e = co.clip_ray((0.0, 0.0, 0.5), (0.2, 0.0, 1.5))
    np.testing.assert_allclose(e, (0.1, 0.0, 1.0), atol=1e-6)
    s, e = co.clip_ray((0.0, 0.5, 0.5), (0.0, -3.0, 0.5))  # toward the far edge y = -1
    np.testing.assert_allclose(e, (0.0, -1.0, 0.5), atol=1e-6)


def test_clip_start_at_the_near_edges(co):
    """a start outside x / y is moved along the ray to the edge it enters through; z is not clipped at the start"""
    s, e = co.clip_ray((-2.0, 0.0, 0.5), (0.5, 0.0, 0.5))
    np.testing.assert_allclose(s, (-1.0, 0.0, 0.5), atol=1e-6)
    np.testing.assert_allclose(e, (0.5, 0.0, 0.5), atol=1e-6)
    s, e = co.clip_ray((0.0, 1.5, 0.5), (0.0, 0.0, 0.5))
    np.testing.assert_allclose(s, (0.0, 1.0, 0.5), atol=1e-6)
    s, e = co.clip_ray((0.0, 0.0, 1.5), (0.0, 0.0, 0.5))
    assert s[2] == f32(1.5)


def test_clip_with_the_end_behind_the_eye(co):
    """to_cs multiplies the direction by sign(end_cs.z): an end with negative z flips the ray"""
    s, e = co.clip_ray((0.0, 0.0, 0.5), (0.5, 0.0, -0.5))
    np.testing.assert_allclose(s, (0.0, 0.0, 0.5), atol=1e-7)
    np.testing.assert_allclose(e, (-0.25, 0.0, 1.0), atol=1e-6)


def test_clip_with_sign_zero(co):
    """sign(end_cs.z) = 0 zeroes the direction: the ray keeps its start and has length 0 (the divisions by a zero delta give infinities
    that max(0, .) and min(1, .) absorb)"""
    s, e = co.clip_ray((0.2, 0.3, 0.5), (0.7, -0.4, 0.0))
    np.testing.assert_array_equal(s, f32([0.2, 0.3, 0.5]))
    np.testing.assert_array_equal(e, s)
    assert co.step_count(s, e, 100, 100, 8) == 2


def test_nearest_tap():
    """floor(u * W), clamped to the edge, NaN to texel 0"""
    import pyoracle_contact_shadows as co

    d = np.arange(12, dtype=np.float32).reshape(3, 4) + 1
    for x in range(4):
        for y in range(3):
            assert co.nearest(d, (x + 0.5) / 4, (y + 0.5) / 3) == d[y, x]
    assert co.nearest(d, 0.0, 0.0) == d[0, 0]
    assert co.nearest(d, 0.2499, 0.0) == d[0, 0] and co.nearest(d, 0.25, 0.0) == d[0, 1]
    assert co.nearest(d, 1.0, 1.0) == d[2, 3]
    assert co.nearest(d, 7.0, -3.0) == d[0, 3]
    assert co.nearest(d, float("nan"), float("inf")) == d[2, 0]
    assert co.nearest(d, float("-inf"), float("nan")) == d[0, 0]


def test_bilinear_tap():
    """texel centres give the texel, midpoints the mean, the borders clamp to the edge texels"""
    import pyoracle_contact_shadows as co

    d = (np.arange(12, dtype=np.float32).reshape(3, 4) * 2 + 1) ** 2
    for x in range(4):
        for y in range(3):
            assert co.bilinear(d, (x + 0.5) / 4, (y + 0.5) / 3) == d[y, x]
    assert co.bilinear(d, 0.25, 0.5 / 3) == f32(d[0, 0] + f32(0.5) * (d[0, 1] - d[0, 0]))
    mid = co.bilinear(d, 0.5, 1.0 / 3)
    top, bot = d[0, 1] + f32(0.5) * (d[0, 2] - d[0, 1]), d[1, 1] + f32(0.5) * (d[1, 2] - d[1, 1])
    assert mid == f32(top + f32(0.5) * (bot - top))
    assert co.bilinear(d, 0.0, 0.0) == d[0, 0] and co.bilinear(d, 1.0, 1.0) == d[2, 3]
    assert co.bilinear(d, -5.0, 0.5 / 3) == d[0, 0] and co.bilinear(d, 5.0, 2.5 / 3) == d[2, 3]
    assert np.isnan(co.bilinear(d, float("nan"), 0.5))


def test_smoothstep_reversed_edges(co):
    assert co.smoothstep(1.0, 0.3, 0.0) == 1.0
    assert co.smoothstep(1.0, 0.3, 1.0) == 0.0
    t = np.clip((f32(0.5) - f32(1.0)) / (f32(0.3) - f32(1.0)), 0, 1).astype(np.float32)
    assert co.smoothstep(1.0, 0.3, 0.5) == f32(f32(t * t) * f32(f32(3.0) - f32(2.0) * t))
    assert co.smoothstep(1.0, 0.3, 0.2) == 1.0 and co.smoothstep(1.0, 0.3, 2.0) == 0.0
    assert co.smoothstep(1.0, 0.3, float("nan")) == 0.0


@pytest.mark.parametrize("seed", range(6))
def test_output_range_on_hostile_frames(co, seed):
    """every output is in [0, 1] and none is NaN, for NaN / Inf / denormal / negative depth and hostile settings"""
    rng = np.random.default_rng(seed)
    ccam, proj = contact_camera_for(97, 61, yaw=31.0 * seed)
    depth = random_depth(rng, 97, 61, proj, hostile=True)
    for hostile in (False, True):
        out = co.contact_shadows(ccam, random_settings(rng, hostile=hostile), depth)
        assert not np.isnan(out).any() and ((out >= 0) & (out <= 1)).all()


def test_nan_thickness_is_never_in_contact(co):
    ccam, proj = contact_camera_for(97, 61)
    depth = random_depth(np.random.default_rng(3), 97, 61, proj, hostile=True)
    s = abi.contact_shadow_settings((0.3, 0.8, 0.2), 16, float("nan"), 2.0)
    assert (co.contact_shadows(ccam, s, depth) == 1.0).all()


def test_box_on_plane(co):
    """a grazing sun behind the box: the ground along the box's front base is in contact (< 1), open ground is exactly 1; with the sun
    beside it (+x) the side face the camera does not see casts nothing (the rays pass behind the front face, deeper than the 0.1 m
    thickness)"""
    w, h = 640, 360
    ccam, _ = contact_camera_for(w, h)
    depth, ground, x, z = box_on_plane(w, h)
    base = ground & (np.abs(x) < 0.9) & (z > -7.0) & (z < -6.8)
    open_ground = ground & ((np.abs(x) > 4.0) | (z > -5.0))
    assert base.sum() > 50 and open_ground.sum() > 10000
    for sun in ((0.0, 0.25, -1.0), (0.3, 0.2, -1.0)):
        for length, steps in ((1.0, 16), (0.3, 8)):
            out = co.contact_shadows(ccam, abi.contact_shadow_settings(sun, steps, 0.1, length), depth)
            assert (out[base] < 1).all() and (out[open_ground] == 1).all()
    side = ground & (x > -1.6) & (x < -1.05) & (z < -7.2) & (z > -8.8)
    out = co.contact_shadows(ccam, abi.contact_shadow_settings((1.0, 0.25, 0.0), 16, 0.1, 1.0), depth)
    assert side.sum() > 50 and (out[side] == 1).all()


def test_lone_plane_does_not_self_shadow(co):
    """measured: a lone ground plane seen from 1 m above is exactly 1 on every pixel, with the reference's defaults, a grazing sun and
    a long 64-step ray (reversed-Z depth is affine in screen space on a plane, so the bilinear tap reconstructs it and the ray stays
    above it)"""
    w, h = 640, 360
    ccam, _ = contact_camera_for(w, h)
    depth, ground, _, _ = box_on_plane(w, h, box=False)
    for s in (abi.contact_shadow_settings(), abi.contact_shadow_settings((1.0, 0.25, 0.0), 16, 0.1, 1.0),
              abi.contact_shadow_settings((0.2, 0.05, -1.0), 64, 0.1, 3.0)):
        out = co.contact_shadows(ccam, s, depth)
        assert ground.sum() > 100000 and (out == 1).all()
