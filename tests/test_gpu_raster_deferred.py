"""The deferred queue of the vis-buffer raster against the CPU oracle, bit for bit, with the queues too small for the frame.

k_raster_visbuffer draws a triangle in its own lane only when its edge functions fit 32 bits and its box holds at most 128
pixels; it queues the data word of every other triangle (invalid vertex, not narrow, large box) for k_raster_deferred, which
clips them or sends them to the chunk queue of k_raster_big.  A deferred queue that overflows makes k_raster_deferred walk the
pass again for the triangles it could not hold, clipped ones included; a chunk queue that overflows makes it draw in 8x4-pixel
tiles.  A clipped triangle past the deferred queue's capacity also raises OXC_STATUS_CLIP_OVERFLOW.
OXC_CLIP_CAPACITY and OXC_BIG_CAPACITY set the two capacities."""
import numpy as np
import pytest

from oxylus_b200 import abi
from tests.test_gpu_parity import _alpha_tables
from tests.test_gpu_raster import FRAMES, H, W, camera, capi, make_ctx, reference, reference_frames, stress, threshold  # noqa: F401

pytestmark = pytest.mark.gpu


def make_ctx_with(capi, sc, deferred_capacity, big_capacity):  # noqa: F811 (capi: the fixture's value)
    import os

    env = {"OXC_CLIP_CAPACITY": deferred_capacity, "OXC_BIG_CAPACITY": big_capacity}
    for k, v in env.items():
        if v is not None:
            os.environ[k] = str(v)
    try:
        return make_ctx(capi, sc)
    finally:
        for k in env:
            os.environ.pop(k, None)


@pytest.mark.parametrize("deferred_capacity,big_capacity", [(None, 1), (1, None), (1, 1), (1, 5), (2, 3)])
def test_deferred_overflow_draws_every_triangle(capi, orc, deferred_capacity, big_capacity):  # noqa: F811
    """a quad of two triangles over the middle 128 x 128 pixels of a 256 x 256 image (not narrow, boxes far over 128 pixels) and
    no clipped one: whatever overflows, the image is the oracle's, the count is 2 and the status word stays clear"""
    from tests.helpers_scene import quad_scene

    w = h = 256
    sc, cam = quad_scene(w, h, depth_a=0.3, depth_b=0.7)
    hs = orc.HostScene(sc)
    mi, _, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    ref = orc.clear_visbuffer(w, h)
    ntri, _ = orc.raster_clip(hs, mi, np.zeros(1, dtype=np.uint32), 0, 1, cam, ref)
    assert ntri == 2
    ctx = make_ctx_with(capi, sc, deferred_capacity, big_capacity)
    vis_dev = ctx.alloc(w * h * 8)
    for _ in range(2):  # twice: the counters are reset per launch
        ctx.clear_visbuffer(vis_dev, w, h)
        ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
        ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, False)
        ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis_dev)
        np.testing.assert_array_equal(ctx.download(vis_dev, np.uint64, w * h).reshape(h, w), ref)
        assert ctx.raster_triangle_count() == 2
        assert ctx.check_status() == 0
    ctx.free(vis_dev)
    ctx.close()


def two_frames(capi, ctx, sc, refs):
    """frames 0 and 1 of the stress scene's reference (same camera, no occluder), with no clip pass: frame 0's late pass and
    frame 1's early pass hold the survivors.  Each frame's image and triangle count are the oracle's; a clipped triangle past
    the deferred queue's capacity raises OXC_STATUS_CLIP_OVERFLOW and nothing else is flagged.  Returns the survivors per pass."""
    vis_dev = ctx.alloc(W * H * 8)
    passes = []
    for f, ref in enumerate(refs):
        cam = camera(sc, False)
        ctx.clear_visbuffer(vis_dev, W, H)
        ctx.clear_hiz()
        ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
        ctx.cull_meshlets(cam, abi.CULL_TEST_ALL, True)
        e = int(ctx.visibility()["early"][0])
        ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, W, H, vis_dev)
        ctx.build_hiz_packed(vis_dev, W, H)
        ctx.cull_meshlets(cam, abi.CULL_TEST_ALL | abi.CULL_LATE_PASS, True)
        l = int(ctx.visibility()["late"][0])
        ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL | abi.CULL_LATE_PASS, W, H, vis_dev)
        assert (e, l) == (ref["early"], ref["late"]), f
        np.testing.assert_array_equal(ctx.download(vis_dev, np.uint64, W * H).reshape(H, W), ref["vis64"], err_msg=f"frame {f}")
        assert ctx.raster_triangle_count() == ref["ntri_early"] + ref["ntri_late"], f
        flags = ctx.status_flags()
        assert flags & ~abi.STATUS_CLIP_OVERFLOW == 0, (f, flags)
        if flags:
            with pytest.raises(capi.OxcError):
                ctx.check_status()
        passes.append((e, l))
    ctx.free(vis_dev)
    assert passes[0][1] > 0 and passes[1][0] > 0, passes
    return passes


QUEUES = [(None, 2), (3, None), (3, 2), (64, 7)]


@pytest.mark.parametrize("deferred_capacity,big_capacity", QUEUES)
def test_deferred_overflow_at_full_grabs(capi, orc, stress, reference, deferred_capacity, big_capacity):  # noqa: F811
    """the stress scene (strips of 1 x 65 to 1 x 129 pixels, boxes of 129 pixels to the whole screen, triangles across the
    near and guard-band planes) with small queues, in both passes: the raster alone draws the oracle's image"""
    refs, _ = reference
    ctx = make_ctx_with(capi, stress, deferred_capacity, big_capacity)
    two_frames(capi, ctx, stress, refs[:2])
    ctx.close()


def test_deferred_overflow_with_alpha_split(capi, orc, stress):  # noqa: F811
    """every other instance alpha-tested: the overflow walk covers the opaque half of the split list only (the alpha raster
    draws the other half), and the raster draws the oracle's image"""
    sc = stress
    keep = sc.mesh_instances["material_index"].copy()
    sc.mesh_instances["material_index"] = np.arange(sc.mesh_instance_count) % 2
    try:
        ctx = make_ctx_with(capi, sc, 3, 2)
        tab, texels = _alpha_tables(capi, orc, ctx)
        refs, _ = reference_frames(orc, sc, materials=tab, frames=FRAMES[:2])
        two_frames(capi, ctx, sc, refs)
        for d in texels:
            ctx.free(d)
        ctx.close()
    finally:
        sc.mesh_instances["material_index"] = keep
