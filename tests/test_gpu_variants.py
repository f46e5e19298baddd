"""The cull passes off the reference frame's call pattern, against the CPU oracle through the C ABI (include/oxcull.h).

tests/test_gpu_parity.py runs every pass with CULL_TEST_ALL and one camera, and clears the Hi-Z pyramid before every early pass.
This module covers what else the ABI accepts: every <HIZ, OCC, LATE, ZERO> instantiation of k_cull_meshlets (pyramid cleared,
built, or written from outside; every subset of the four cull flags; the mesh pass's camera or another one), an occlusion toggle
across frames, the mesh-level flags with their LOD write-back and the automatic shard id base, the raster and triangle cull on a
camera other than the mesh pass's, and the hostile-input frames of tests/emulated_torture_check.py.  Same bar as the parity
suite: bit-exact; survivor and index order is atomics-ordered, so those are compared as sorted sets."""
import os
import re

import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests import emulated_torture_check as torture
from tests.test_gpu_parity import SCENES, make_ctx

pytestmark = pytest.mark.gpu

FRUSTUM, LOD, OCC, LATE = abi.CULL_TEST_FRUSTUM, abi.CULL_SELECT_LOD, abi.CULL_TEST_OCCLUSION, abi.CULL_LATE_PASS
FLAG_SETS = [f | s | o | l for f in (0, FRUSTUM) for s in (0, LOD) for o in (0, OCC) for l in (0, LATE)]
PYRAMIDS = ("cleared", "built", "external")

VARIANT_SCENES = {
    "small": SCENES["small"],
    "ragged_lods": SCENES["ragged_lods"],
    # 1-3 meshlets per mesh instance: one 32-entry slab of the meshlet cull spans many instances
    "fragmented": dict(n_meshlets=4000, width=640, height=360, n_unique_meshes=48, meshlets_per_mesh=(1, 3), max_lods=3, ragged=True),
}


def make_scene(name):
    if name == "hostile":  # NaN / Inf / negative / denormal bounds, garbage cones, degenerate transforms
        return torture.mutate(synth.make_scene(config_index=2, **SCENES["small"]), np.random.default_rng(1), "all")
    return synth.make_scene(config_index=2, **VARIANT_SCENES[name])


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module", params=list(VARIANT_SCENES) + ["hostile"])
def scene(request):
    return make_scene(request.param)


@pytest.fixture(scope="module", params=["ragged_lods", "fragmented"])
def lod_scene(request):
    return make_scene(request.param)


def instantiation(use_hiz, flags, cleared):
    """The k_cull_meshlets<HIZ, OCC, LATE, ZERO> oxc_cull_meshlets launches: OCC and LATE are the flags' bits, ZERO says the
    pyramid still holds what oxc_clear_hiz wrote (no oxc_build_hiz* or oxc_mark_hiz_dirty since); all three need use_hiz."""
    h = bool(use_hiz)
    return (h, h and bool(flags & OCC), h and bool(flags & LATE), h and bool(cleared))


def dispatched_instantiations():
    """every k_cull_meshlets instantiation oxc_cull_meshlets can launch, read from its dispatch in oxcull.cu"""
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oxylus_b200", "csrc", "oxcull.cu")).read()
    body = src[src.index("int oxc_cull_meshlets("):]
    body = body[: body.index("\n}\n")]
    found = {tuple(a == "true" for a in m) for m in re.findall(r"GO\((true|false), (true|false), (true|false), (true|false)\)", body)}
    assert len(found) == 9, found
    return found


def random_mask(ctx, seed):
    return np.random.default_rng(seed).integers(0, 2**32, size=ctx.out.visibility_mask_words, dtype=np.uint64).astype(np.uint32)


def assert_segments(ctx, visible, e, l, tag):
    got = ctx.visible_indices(e + l)
    np.testing.assert_array_equal(np.sort(got[:e]), np.sort(visible[:e]), err_msg=f"{tag}: early survivors")
    np.testing.assert_array_equal(np.sort(got[e:]), np.sort(visible[e:e + l]), err_msg=f"{tag}: late survivors")


def test_cull_meshlets_variant_matrix(capi, orc, scene):
    """every pyramid state x every subset of the four flags x two cameras (the mesh pass's, and one that makes the meshlet pass
    rebuild InstCull), from a random persistent mask, plus the plain variant: counters, early and late survivors, whole mask"""
    hs = orc.HostScene(scene)
    ctx = make_ctx(capi, scene)
    w, h = scene.width, scene.height
    hw, hh = scene.hiz_extent()
    occ_dev = ctx.alloc(w * h * 4)
    ctx.upload(occ_dev, scene.occluder_depth)
    pyramid = {"cleared": orc.Hiz(hw, hh), "built": orc.build_hiz(scene.occluder_depth, orc.Hiz(hw, hh)),
               "external": orc.build_hiz(np.ascontiguousarray(scene.occluder_depth[::-1, ::-1]), orc.Hiz(hw, hh))}
    cam_a, cam_b = scene.camera(0.0), scene.camera(7.0)
    mi, vis0, _ = orc.cull_meshes(hs, cam_a, abi.CULL_TEST_ALL)
    mask0 = random_mask(ctx, 5)
    reached, early_all = set(), {}
    for state in PYRAMIDS:
        for flags in FLAG_SETS:
            for cam_name, cam in (("a", cam_a), ("b", cam_b)):
                tag = f"pyramid {state}, flags {flags:#x}, camera {cam_name}"
                ctx.cull_meshes(cam_a, abi.CULL_TEST_ALL)
                if state == "built":
                    ctx.build_hiz(occ_dev, w, h)
                else:
                    ctx.clear_hiz()
                    if state == "external":  # written behind the library's back, then declared
                        ctx.upload_hiz(pyramid["external"].data)
                        ctx.mark_hiz_dirty()
                ctx.set_mask(mask0)
                ctx.cull_meshlets(cam, flags, True)
                reached.add(instantiation(True, flags, state == "cleared"))
                vis, mask = vis0.copy(), mask0.copy()
                visible, cmd = orc.cull_meshlets_hiz(hs, mi, vis, cam, flags, pyramid[state], mask)
                e, l = int(vis["early"][0]), int(vis["late"][0])
                v = ctx.visibility()
                assert (int(v["early"][0]), int(v["late"][0]), int(ctx.cull_triangles_cmd()["x"][0])) == (e, l, int(cmd["x"][0])), tag
                assert_segments(ctx, visible, e, l, tag)
                np.testing.assert_array_equal(ctx.mask(), mask, err_msg=f"{tag}: mask")
                if flags == abi.CULL_TEST_ALL and cam_name == "a":
                    early_all[state] = e
    for cam_name, cam in (("a", cam_a), ("b", cam_b)):
        ctx.cull_meshes(cam_a, abi.CULL_TEST_ALL)
        ctx.set_mask(mask0)
        ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, use_hiz=False)
        reached.add(instantiation(False, abi.CULL_TEST_FRUSTUM, False))
        visible, cmd = orc.cull_meshlets(hs, mi, vis0.copy(), cam)
        n = int(cmd["x"][0])
        assert int(ctx.cull_triangles_cmd()["x"][0]) == n and int(ctx.visibility()["early"][0]) == 0, f"plain, camera {cam_name}"
        np.testing.assert_array_equal(np.sort(ctx.visible_indices(n)), np.sort(visible[:n]), err_msg=f"plain, camera {cam_name}")
        np.testing.assert_array_equal(ctx.mask(), mask0, err_msg=f"plain, camera {cam_name}: the plain variant keeps the mask")
    assert reached == dispatched_instantiations()
    # the pyramids occlude something, so the early pass's Hi-Z stages decided the non-cleared cases
    assert early_all["built"] < early_all["cleared"] and early_all["external"] < early_all["cleared"], early_all
    ctx.free(occ_dev)
    ctx.close()


def test_occlusion_toggle_frames(capi, orc, scene):
    """three two-pass frames on one context with occlusion off in the middle one, as an engine's occlusion toggle runs them; frames 1
    and 2 start from the pyramid the frame before built.  After every pass: counters, survivors, mask, packed image, triangle count,
    every Hi-Z level."""
    hs = orc.HostScene(scene)
    ctx = make_ctx(capi, scene)
    w, h = scene.width, scene.height
    vis_dev, occ_dev = ctx.alloc(w * h * 8), ctx.alloc(w * h * 4)
    ctx.upload(occ_dev, scene.occluder_depth)
    hiz = orc.Hiz(*scene.hiz_extent())
    mask = np.zeros(ctx.out.visibility_mask_words, dtype=np.uint32)
    ctx.clear_hiz()
    for f, flags in enumerate((abi.CULL_TEST_ALL, FRUSTUM | LOD, abi.CULL_TEST_ALL)):
        cam = scene.camera(2.0 * f)
        img = orc.merge_occluder_depth(orc.clear_visbuffer(w, h), scene.occluder_depth)
        ctx.clear_visbuffer_with_depth(vis_dev, occ_dev, w, h)
        mi, vis, _ = orc.cull_meshes(hs, cam, flags)
        ctx.cull_meshes(cam, flags)
        visible, ntri = None, 0
        for late in (0, LATE):
            tag = f"frame {f} {'late' if late else 'early'}"
            visible, _ = orc.cull_meshlets_hiz(hs, mi, vis, cam, flags | late, hiz, mask, visible)
            ctx.cull_meshlets(cam, flags | late, True)
            e, l = int(vis["early"][0]), int(vis["late"][0])
            ntri += orc.raster_clip(hs, mi, visible, e if late else 0, l if late else e, cam, img)[0]
            ctx.raster_visbuffer(cam, flags | late, w, h, vis_dev)
            v = ctx.visibility()
            assert (int(v["total"][0]), int(v["early"][0]), int(v["late"][0])) == (int(vis["total"][0]), e, l), tag
            assert_segments(ctx, visible, e, l if late else 0, tag)
            np.testing.assert_array_equal(ctx.mask(), mask, err_msg=f"{tag}: mask")
            np.testing.assert_array_equal(ctx.download(vis_dev, np.uint64, w * h).reshape(h, w), img, err_msg=f"{tag}: image")
            assert ctx.raster_triangle_count() == ntri, tag
            if not late:
                ctx.build_hiz_packed(vis_dev, w, h)
                orc.build_hiz(orc.resolve(img)[1], hiz)
            levels = ctx.hiz_levels()
            assert len(levels) == hiz.levels
            for lvl, got in enumerate(levels):
                np.testing.assert_array_equal(got.view(np.uint32), hiz.level(lvl).view(np.uint32), err_msg=f"{tag}: Hi-Z mip {lvl}")
    ctx.free(vis_dev)
    ctx.free(occ_dev)
    ctx.close()


# SELECT_LOD alternates on / off, so every frame starts from the LODs the previous one wrote back
MESH_FLAG_SEQUENCE = (FRUSTUM | LOD, FRUSTUM, abi.CULL_TEST_ALL | LATE, 0, LOD, FRUSTUM, FRUSTUM | LOD)


def test_cull_meshes_flag_sequence(capi, orc, lod_scene):
    """oxc_cull_meshes under each mesh-level flag set, one after the other on one context: meshlet-instance list, total, dispatch
    size and every mesh instance's written-back lod_index"""
    sc = lod_scene
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc)
    n = sc.mesh_instance_count
    reset = 0
    for k, flags in enumerate(MESH_FLAG_SEQUENCE):
        cam = sc.camera(3.0 * k)
        held = hs.mesh_instances["lod_index"].copy()
        mi, vis, cmd = orc.cull_meshes(hs, cam, flags)
        ctx.cull_meshes(cam, flags)
        total = int(vis["total"][0])
        assert int(ctx.visibility()["total"][0]) == total, flags
        assert int(ctx.cull_meshlets_cmd()["x"][0]) == int(cmd["x"][0]), flags
        np.testing.assert_array_equal(ctx.meshlet_instances(total), mi[:total], err_msg=f"flags {flags:#x}")
        np.testing.assert_array_equal(ctx.mesh_instances(n)["lod_index"], hs.mesh_instances["lod_index"], err_msg=f"flags {flags:#x}")
        if flags & FRUSTUM and not flags & LOD:
            reset += int(np.count_nonzero((held > 0) & (hs.mesh_instances["lod_index"] == 0)))
    assert reset > 0  # some instance entered a frame without SELECT_LOD holding a LOD above 0
    ctx.close()


@pytest.mark.parametrize("flags", [FRUSTUM, abi.CULL_TEST_ALL], ids=["frustum", "test_all"])
def test_shard_auto_id_base(capi, orc, lod_scene, flags):
    """oxc_set_shard_auto at two split points: the shard's survivor ids, automatic id base included, are the whole scene's ids
    of that range, so k_count_prefix_meshlets counts what k_cull_meshes emits under these flags"""
    sc = lod_scene
    n = sc.mesh_instance_count
    cam = sc.camera(4.0)
    hs = orc.HostScene(sc)
    mi, vis, _ = orc.cull_meshes(hs, cam, flags)
    ref, cmd = orc.cull_meshlets(hs, mi, vis, cam)
    ref = ref[: int(cmd["x"][0])]
    owner = mi["mesh_instance_index"][ref]
    for first, count in ((n // 3, n // 3), (n // 2, n - n // 2)):
        want = np.sort(ref[(owner >= first) & (owner < first + count)])
        ctx = make_ctx(capi, sc)
        ctx.set_shard_auto(first, count)
        ctx.cull_meshes(cam, flags)
        ctx.cull_meshlets(cam, FRUSTUM, use_hiz=False)
        got = int(ctx.cull_triangles_cmd()["x"][0])
        assert got == len(want) > 0, (first, count)
        np.testing.assert_array_equal(np.sort(ctx.visible_indices(got)), want, err_msg=f"shard [{first}, +{count})")
        ctx.close()
    # under TEST_FRUSTUM alone the prefix must not select LODs: with selection the instances below the split would emit fewer
    below = [int(orc.cull_meshes(orc.HostScene(sc), cam, f, 0, n // 3)[1]["total"][0]) for f in (FRUSTUM, FRUSTUM | LOD)]
    assert below[0] != below[1], below


def test_mixed_cameras_through_triangle_passes(capi, orc, scene):
    """mesh pass on camera a, meshlet pass on camera b (against a built pyramid and a random mask), then the raster and the
    triangle cull on camera b and once more on camera a: InstCull is rebuilt twice within one frame"""
    hs = orc.HostScene(scene)
    ctx = make_ctx(capi, scene, reordered=True)
    w, h = scene.width, scene.height
    vis_dev, occ_dev = ctx.alloc(w * h * 8), ctx.alloc(w * h * 4)
    ctx.upload(occ_dev, scene.occluder_depth)
    cam_a, cam_b = scene.camera(0.0), scene.camera(6.0)
    mask0 = random_mask(ctx, 9)
    hiz = orc.build_hiz(scene.occluder_depth, orc.Hiz(*scene.hiz_extent()))
    mi, vis, _ = orc.cull_meshes(hs, cam_a, abi.CULL_TEST_ALL)
    visible, _ = orc.cull_meshlets_hiz(hs, mi, vis, cam_b, abi.CULL_TEST_ALL, hiz, mask0.copy())
    e = int(vis["early"][0])
    ctx.cull_meshes(cam_a, abi.CULL_TEST_ALL)
    ctx.build_hiz(occ_dev, w, h)
    ctx.set_mask(mask0)
    ctx.cull_meshlets(cam_b, abi.CULL_TEST_ALL, True)
    assert int(ctx.visibility()["early"][0]) == e > 0
    assert_segments(ctx, visible, e, 0, "meshlet pass on camera b")
    for name, cam in (("b", cam_b), ("a", cam_a)):
        img = orc.clear_visbuffer(w, h)
        ntri = orc.raster_clip(hs, mi, visible, 0, e, cam, img)[0]
        ctx.clear_visbuffer(vis_dev, w, h)
        ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis_dev)
        np.testing.assert_array_equal(ctx.download(vis_dev, np.uint64, w * h).reshape(h, w), img, err_msg=f"raster on camera {name}")
        assert ctx.raster_triangle_count() == ntri, name
        ref_idx, ref_draw = orc.cull_triangles(hs, mi, visible, 0, e, cam)
        ctx.cull_triangles(cam, abi.CULL_TEST_ALL)
        dc = ctx.draw_cmd()
        assert int(dc["index_count"][0]) == int(ref_draw["index_count"][0]), name
        got = ctx.reordered_indices(int(dc["index_count"][0])).reshape(-1, 3)
        ref_idx = ref_idx.reshape(-1, 3)
        np.testing.assert_array_equal(got[np.argsort(got[:, 0], kind="stable")], ref_idx[np.argsort(ref_idx[:, 0], kind="stable")],
                                      err_msg=f"triangle cull on camera {name}")
    ctx.free(vis_dev)
    ctx.free(occ_dev)
    ctx.close()


@pytest.fixture(scope="module")
def torture_base():
    return torture.base_scene()


@pytest.mark.parametrize("case", torture.cases(), ids=lambda c: c[0])
def test_hostile_frames(capi, orc, torture_base, case):
    """the hostile-input frames of tests/emulated_torture_check.py on the device: NaN / Inf / denormal / negative bounds, garbage
    cones, extreme transforms, hostile cameras, the alpha material table and a hostile external depth.  The hardware's
    rcp.approx.ftz / rsqrt.approx.ftz return what the emulated library's IEEE stand-ins do not (-Inf for a negative denormal):
    only here do the filtered predicates' preconditions meet them."""
    assert torture.run_case(torture_base, case), case[0]
