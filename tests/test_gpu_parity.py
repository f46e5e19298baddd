"""CUDA path vs CPU oracle on the same seeded inputs, through the C ABI (include/oxcull.h).

Bar (BASELINE.json north_star): bit-exact for integer outputs (meshlet_instances, survivor ID sets, visibility
bitmask, triangle index sets, packed vis buffer) and for Hi-Z depths (min-only pyramid => exact, tolerance 0 ULP).
Survivor / index ORDER is atomics-ordered in the reference (SURVEY §8a quirk 8) => compared as sorted sets.
"""
import numpy as np
import pytest

from oxylus_b200 import abi, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


def make_ctx(capi, sc, reordered=False, views=0):
    hw, hh = sc.hiz_extent()
    ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh, alloc_reordered_indices=reordered,
                       max_views=views)
    ctx.set_scene(sc)
    return ctx


SCENES = {
    "small": dict(n_meshlets=6000, width=640, height=360, n_unique_meshes=16),
    "ragged_lods": dict(n_meshlets=9000, width=800, height=450, n_unique_meshes=24, max_lods=3, ragged=True),
    "box": dict(n_meshlets=20000, width=1280, height=720, n_unique_meshes=32, placement="box"),
    "medium": dict(n_meshlets=150000, width=1920, height=1080, n_unique_meshes=64),
}


@pytest.fixture(scope="module", params=list(SCENES))
def scene(request):
    return synth.make_scene(config_index=2, **SCENES[request.param])


def test_cull_meshes_parity(capi, orc, scene):
    hs = orc.HostScene(scene)
    ctx = make_ctx(capi, scene)
    for yaw in (0.0, 25.0):
        cam = scene.camera(yaw)
        mi_ref, vis_ref, cmd_ref = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
        ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
        vis = ctx.visibility()
        total = int(vis_ref["total"][0])
        assert int(vis["total"][0]) == total
        assert int(ctx.cull_meshlets_cmd()["x"][0]) == int(cmd_ref["x"][0])
        # deterministic expansion order == oracle's serial order: compare the arrays themselves
        np.testing.assert_array_equal(ctx.meshlet_instances(total), mi_ref[:total])
        np.testing.assert_array_equal(ctx.mesh_instances(scene.mesh_instance_count)["lod_index"], hs.mesh_instances["lod_index"])
    ctx.close()


def test_cull_meshes_flag_quirk(capi, orc, scene):
    """without TestFrustum nothing is emitted (cull_meshes.slang:34 `HAS_FLAG(TestFrustum) && test_frustum`)"""
    ctx = make_ctx(capi, scene)
    ctx.cull_meshes(scene.camera(), abi.CULL_SELECT_LOD)
    assert int(ctx.visibility()["total"][0]) == 0
    ctx.close()


def _frame_gpu(capi, ctx, sc, cam, occluder_dev, vis_dev, hiz_from_packed=True):
    """early -> raster -> hiz -> late -> raster, low-level ABI calls.  Returns intermediates."""
    w, h = sc.width, sc.height
    ctx.clear_visbuffer(vis_dev, w, h)
    ctx.clear_hiz()
    if occluder_dev is not None:
        ctx.merge_depth(vis_dev, occluder_dev, w, h)
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    ctx.cull_meshlets(cam, abi.CULL_TEST_ALL, True)
    vis_e = ctx.visibility()
    e = int(vis_e["early"][0])
    mask_e = ctx.mask()
    tcmd_e = int(ctx.cull_triangles_cmd()["x"][0])
    ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis_dev)
    if hiz_from_packed:
        ctx.build_hiz_packed(vis_dev, w, h)
    else:
        depth_dev = ctx.alloc(w * h * 4)
        ctx.resolve_visbuffer(vis_dev, w, h, None, depth_dev)
        ctx.build_hiz(depth_dev, w, h)
        ctx.sync()
        ctx.free(depth_dev)
    hiz = ctx.hiz_levels()
    ctx.cull_meshlets(cam, abi.CULL_TEST_ALL | abi.CULL_LATE_PASS, True)
    vis_l = ctx.visibility()
    l = int(vis_l["late"][0])
    tcmd_l = int(ctx.cull_triangles_cmd()["x"][0])
    ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL | abi.CULL_LATE_PASS, w, h, vis_dev)
    img = ctx.download(vis_dev, np.uint64, w * h).reshape(h, w)
    return dict(early=e, late=l, mask_after_early=mask_e, mask=ctx.mask(), visible=ctx.visible_indices(e + l), hiz=hiz,
                vis64=img, tcmd_early=tcmd_e, tcmd_late=tcmd_l, total=int(vis_l["total"][0]), ntri=ctx.raster_triangle_count())


def test_two_pass_frames_parity(capi, orc, scene):
    """three consecutive frames (camera yawing 2 deg / frame) — every intermediate of the two-pass pipeline."""
    hs = orc.HostScene(scene)
    ctx = make_ctx(capi, scene)
    w, h = scene.width, scene.height
    vis_dev = ctx.alloc(w * h * 8)
    occ_dev = ctx.alloc(w * h * 4)
    ctx.upload(occ_dev, scene.occluder_depth)
    mask_ref = np.zeros(ctx.out.visibility_mask_words, dtype=np.uint32)
    for f in range(3):
        cam = scene.camera(2.0 * f)
        ref = orc.frame(hs, cam, w, h, mask_ref, scene.occluder_depth)
        got = _frame_gpu(capi, ctx, scene, cam, occ_dev, vis_dev, hiz_from_packed=(f != 1))
        assert got["total"] == int(ref["visibility"]["total"][0])
        assert got["early"] == ref["early"], f"frame {f}"
        assert got["late"] == ref["late"], f"frame {f}"
        assert got["tcmd_early"] == ref["early"] and got["tcmd_late"] == ref["late"]
        np.testing.assert_array_equal(got["mask_after_early"], ref["mask_after_early"])
        np.testing.assert_array_equal(got["mask"], mask_ref)
        e, l = ref["early"], ref["late"]
        np.testing.assert_array_equal(np.sort(got["visible"][:e]), np.sort(ref["visible"][:e]))
        np.testing.assert_array_equal(np.sort(got["visible"][e:e + l]), np.sort(ref["visible"][e:e + l]))
        for lvl in range(ref["hiz"].levels):  # Hi-Z depths: bit-exact (0 ULP)
            np.testing.assert_array_equal(got["hiz"][lvl].view(np.uint32), ref["hiz"].level(lvl).view(np.uint32))
        np.testing.assert_array_equal(got["vis64"], ref["vis64"])
        assert got["ntri"] == ref["ntri_early"] + ref["ntri_late"]
    ctx.free(vis_dev)
    ctx.free(occ_dev)
    ctx.close()


def test_cull_meshlets_plain_parity(capi, orc, scene):
    hs = orc.HostScene(scene)
    ctx = make_ctx(capi, scene)
    cam = scene.camera(10.0)
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    ref, cmd = orc.cull_meshlets(hs, mi, vis, cam)
    n = int(cmd["x"][0])
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, use_hiz=False)
    assert int(ctx.cull_triangles_cmd()["x"][0]) == n
    assert int(ctx.visibility()["early"][0]) == 0  # the plain variant never touches visibility (cull_meshlets.slang:55-70)
    np.testing.assert_array_equal(np.sort(ctx.visible_indices(n)), np.sort(ref[:n]))
    ctx.close()


def test_cull_triangles_parity(capi, orc):
    sc = synth.make_scene(config_index=3, **SCENES["ragged_lods"])
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc, reordered=True)
    cam = sc.camera(5.0)
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    ref_vis, cmd = orc.cull_meshlets(hs, mi, vis, cam)
    n = int(cmd["x"][0])
    ref_idx, ref_draw = orc.cull_triangles(hs, mi, ref_vis, 0, n, cam)
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, use_hiz=False)
    ctx.cull_triangles(cam, abi.CULL_TEST_FRUSTUM)
    dc = ctx.draw_cmd()
    assert int(dc["index_count"][0]) == int(ref_draw["index_count"][0])
    assert int(dc["instance_count"][0]) == 1
    got = ctx.reordered_indices(int(dc["index_count"][0])).reshape(-1, 3)
    # each triangle is three consecutive indices (instance<<8 | corner); order of triangles is atomics-ordered
    order_g = np.argsort(got[:, 0], kind="stable")
    order_r = np.argsort(ref_idx.reshape(-1, 3)[:, 0], kind="stable")
    np.testing.assert_array_equal(got[order_g], ref_idx.reshape(-1, 3)[order_r])
    ctx.close()


def test_small_primitive_cull_parity(capi, orc):
    """north_star's small-primitive cull, opt-in on both triangle paths: (a) oxc_raster_visbuffer(small_primitive_cull=1)
    draws the identical image and counts exactly the oracle's number of culled triangles fewer; (b)
    oxc_cull_triangles_small_primitive emits the oracle's shorter index buffer."""
    sc = synth.make_scene(config_index=3, **SCENES["medium"])
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc, reordered=True)
    cam = sc.camera(1.0)
    w, h = sc.width, sc.height
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    ref_vis, cmd = orc.cull_meshlets(hs, mi, vis, cam)
    n = int(cmd["x"][0])
    ref_idx, ref_draw, culled = orc.cull_triangles_small_primitive(hs, mi, ref_vis, 0, n, cam, w, h)
    full_idx, _ = orc.cull_triangles(hs, mi, ref_vis, 0, n, cam)
    assert culled > 0 and len(full_idx) - len(ref_idx) == 3 * culled
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, use_hiz=False)
    # (b) index buffer
    ctx.cull_triangles_small_primitive(cam, abi.CULL_TEST_FRUSTUM, w, h)
    dc = ctx.draw_cmd()
    assert int(dc["index_count"][0]) == int(ref_draw["index_count"][0])
    got = ctx.reordered_indices(int(dc["index_count"][0])).reshape(-1, 3)
    np.testing.assert_array_equal(got[np.argsort(got[:, 0], kind="stable")],
                                  ref_idx.reshape(-1, 3)[np.argsort(ref_idx.reshape(-1, 3)[:, 0], kind="stable")])
    # (a) raster: same image, fewer counted triangles
    vis_dev = ctx.alloc(w * h * 8)
    images, counts = [], []
    for spc in (False, True):
        ctx.clear_visbuffer(vis_dev, w, h)
        ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis_dev, small_primitive_cull=spc)
        images.append(ctx.download(vis_dev, np.uint64, w * h))
        counts.append(ctx.raster_triangle_count())
    np.testing.assert_array_equal(images[0], images[1])
    assert counts[0] == len(full_idx) // 3 and counts[1] == counts[0] - culled
    ref_img = orc.clear_visbuffer(w, h)
    orc.raster_clip(hs, mi, ref_vis, 0, n, cam, ref_img)  # the product's raster clips what the plain spec drops
    np.testing.assert_array_equal(images[1].reshape(h, w), ref_img)
    ctx.free(vis_dev)
    ctx.close()


def test_wide_id_packing_and_24_bit_refusal(capi, orc):
    """Scenes that can emit more than 2^24 meshlet instances overflow the reference's 24 + 8 bit vis-buffer word: the raster
    refuses them (OXC_E_CAPACITY) unless the context was created with wide_ids (26 + 6 bits).  The wide packing is the
    oracle's image with every id word repacked — same winners (the tie-break order (id, triangle) is preserved)."""
    # (a) wide packing on a small scene with a large id base: ids beyond 2^24
    sc = synth.make_scene(config_index=2, **SCENES["small"])
    hs = orc.HostScene(sc)
    w, h = sc.width, sc.height
    hw, hh = sc.hiz_extent()
    ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh, wide_ids=True)
    ctx.set_scene(sc)
    base = (1 << 25) + 12345
    base_dev = ctx.alloc(4)
    ctx.upload(base_dev, np.array([base], dtype=np.uint32))
    ctx.set_shard(0, sc.mesh_instance_count, base_dev)
    cam = sc.camera(0.0)
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    ref_vis, cmd = orc.cull_meshlets(hs, mi, vis, cam)
    n = int(cmd["x"][0])
    ref_img = orc.clear_visbuffer(w, h)
    orc.raster_clip(hs, mi, ref_vis, 0, n, cam, ref_img)  # the product's raster clips what the plain spec drops
    data = (ref_img & 0xFFFFFFFF).astype(np.uint64)
    drawn = data != 0xFFFFFFFF
    repacked = np.where(drawn, (((data >> 8) + base) << 6) | (data & 0xFF), data)
    want = (ref_img & np.uint64(0xFFFFFFFF00000000)) | repacked
    vis_dev = ctx.alloc(w * h * 8)
    ctx.clear_visbuffer(vis_dev, w, h)
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, use_hiz=False)
    np.testing.assert_array_equal(np.sort(ctx.visible_indices(n)), np.sort(ref_vis[:n]) + base)
    ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis_dev)
    got = ctx.download(vis_dev, np.uint64, w * h).reshape(h, w)
    np.testing.assert_array_equal(got, want)
    assert ctx.out.vis_primitive_bits == 6
    ctx.free(vis_dev); ctx.free(base_dev)
    ctx.close()
    # (b) a 17 M scene: refused with the reference packing, accepted with the wide one
    big = synth.make_scene(17_000_000, config_index=2, width=640, height=360)
    bhw, bhh = big.hiz_extent()
    for wide in (False, True):
        ctx = capi.Context(0, big.mesh_instance_count, big.max_meshlet_instance_count, bhw, bhh, wide_ids=wide)
        ctx.set_scene(big)
        cam = big.camera(0.0)
        vis_dev = ctx.alloc(640 * 360 * 8)
        ctx.clear_visbuffer(vis_dev, 640, 360)
        ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
        ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, use_hiz=False)
        if wide:
            ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, 640, 360, vis_dev)
            ctx.sync()
            assert ctx.check_status() == 0 and ctx.raster_triangle_count() > 0
        else:
            with pytest.raises(capi.OxcError, match="wide_ids"):
                ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, 640, 360, vis_dev)
        ctx.free(vis_dev)
        ctx.close()


def test_scene_validation_and_capacity_errors(capi):
    """ADVICE r1: a scene larger than the create-time capacities, or with an index out of range, is an error from oxc_set_scene
    (OXC_E_CAPACITY / OXC_E_INVALID), not silent device-memory corruption."""
    sc = synth.make_scene(config_index=2, **SCENES["small"])
    hw, hh = sc.hiz_extent()
    ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count - 1, hw, hh)
    with pytest.raises(capi.OxcError, match="max_meshlet_instances"):
        ctx.set_scene(sc)
    ctx.close()
    for field, bad in (("mesh_index", len(sc.meshes)), ("transform_index", len(sc.transforms)), ("lod_index", 9)):
        ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
        keep = sc.mesh_instances[field][3]
        sc.mesh_instances[field][3] = bad
        try:
            with pytest.raises(capi.OxcError, match=field):
                ctx.set_scene(sc)
        finally:
            sc.mesh_instances[field][3] = keep
        ctx.close()
    # a shard context sized for its own share accepts the scene once the shard is set, and refuses a range that does not fit
    from oxylus_b200 import dist as oxdist

    half = sc.mesh_instance_count // 2
    need = int(oxdist.lod0_counts_of(sc)[:half].sum())
    ctx = capi.Context(0, sc.mesh_instance_count, need, hw, hh, max_mask_bits=sc.max_meshlet_instance_count)
    ctx.set_shard_auto(0, half)
    ctx.set_scene(sc)
    with pytest.raises(capi.OxcError, match="max_meshlet_instances"):
        ctx.set_shard_auto(0, sc.mesh_instance_count)
    ctx.close()


def test_hiz_build_shapes(capi, orc):
    """depth sizes whose Hi-Z extent differs from size/2 (point-sample mapping), incl. a sub-tile pyramid."""
    rng = np.random.default_rng(7)
    for (w, h) in [(1920, 1080), (3840, 2160), (640, 360), (100, 60), (64, 64), (1000, 520)]:
        hw, hh = abi.hiz_extent(w, h)
        depth = rng.random((h, w), dtype=np.float32)
        ref = orc.build_hiz(depth, orc.Hiz(hw, hh))
        ctx = capi.Context(0, 1, 1, hw, hh)
        d_dev = ctx.alloc(w * h * 4)
        ctx.upload(d_dev, depth)
        ctx.build_hiz(d_dev, w, h)
        got = ctx.hiz_levels()
        assert len(got) == ref.levels
        for lvl in range(ref.levels):
            np.testing.assert_array_equal(got[lvl].view(np.uint32), ref.level(lvl).view(np.uint32), err_msg=f"{w}x{h} mip {lvl}")
        ctx.free(d_dev)
        ctx.close()


def test_multiview_parity(capi, orc):
    sc = synth.make_scene(40000, config_index=4, width=1280, height=720, n_unique_meshes=32, placement="box")
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc, views=16)
    cam = sc.camera()
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    total = int(vis["total"][0])
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    dirs = synth.uniform(sc.seed, 90, 48, -1.0, 1.0).reshape(16, 3)
    dirs[:, 1] = -np.abs(dirs[:, 1]) - 0.2
    views = np.concatenate([synth.make_ortho_view(dirs[v], (0.0, 0.0, -200.0), 60.0 * (1 + v % 4), 800.0, sc.mesh_instance_count)
                            for v in range(16)])
    for directional in (1, 0):
        ref_bits, ref_counts = orc.cull_meshlets_multiview(hs, mi, total, views, directional)
        ctx.cull_meshlets_multiview(views, directional)
        np.testing.assert_array_equal(ctx.view_bits(total), ref_bits)
        np.testing.assert_array_equal(ctx.view_counts(), ref_counts)
    # perspective cameras as views, positional cone: view 0 must equal the plain single-view cull
    pviews = np.concatenate([sc.camera(3.0 * v) for v in range(8)])
    ref_bits, ref_counts = orc.cull_meshlets_multiview(hs, mi, total, pviews, 0)
    ctx.cull_meshlets_multiview(pviews, 0)
    np.testing.assert_array_equal(ctx.view_bits(total), ref_bits)
    ref_plain, cmd = orc.cull_meshlets(hs, mi, vis, sc.camera(0.0))
    np.testing.assert_array_equal(np.nonzero(ref_bits & 1)[0], np.sort(ref_plain[: int(cmd["x"][0])]))
    ctx.close()


def test_renderer_host_mirror(capi, orc):
    """oxr_render (C++ RendererInstance mirror, HOST in / HOST out) vs the oracle frame sequence."""
    sc = synth.make_scene(config_index=2, **SCENES["small"])
    hs = orc.HostScene(sc)
    r = capi.Renderer(0, sc, alloc_reordered_indices=True)
    mask_ref = np.zeros((sc.max_meshlet_instance_count + 31) // 32, dtype=np.uint32)
    for f in range(3):
        cam = sc.camera(-3.0 * f)
        ref = orc.frame(hs, cam, sc.width, sc.height, mask_ref, sc.occluder_depth)
        got = r.render(cam, sc.occluder_depth)
        assert (got["total"], got["early"], got["late"]) == (int(ref["visibility"]["total"][0]), ref["early"], ref["late"])
        v32, d = orc.resolve(ref["vis64"])
        np.testing.assert_array_equal(got["vis32"], v32)
        np.testing.assert_array_equal(got["depth"].view(np.uint32), d.view(np.uint32))
        np.testing.assert_array_equal(np.sort(got["visible"]), np.sort(ref["visible"][: ref["early"] + ref["late"]]))
        assert got["raster_triangles"] == ref["ntri_early"] + ref["ntri_late"]
        assert got["draw_index_count_early"] == 3 * ref["ntri_early"] and got["draw_index_count_late"] == 3 * ref["ntri_late"]
        np.testing.assert_array_equal(r.ctx.mask(), mask_ref)
    r.close()


def test_empty_and_edge_inputs(capi, orc):
    """no survivors / camera looking away / single meshlet / zero mesh instances in the camera."""
    sc = synth.make_scene(1, config_index=2, width=128, height=64, n_unique_meshes=1, meshlets_per_mesh=(1, 1))
    ctx = make_ctx(capi, sc, reordered=True)
    w, h = sc.width, sc.height
    vis_dev = ctx.alloc(w * h * 8)
    for yaw in (0.0, 180.0):
        hs = orc.HostScene(sc)
        cam = sc.camera(yaw)
        mask_ref = np.zeros(ctx.out.visibility_mask_words, dtype=np.uint32)
        ctx.reset_visibility_mask()
        ref = orc.frame(hs, cam, w, h, mask_ref, None)
        got = _frame_gpu(capi, ctx, sc, cam, None, vis_dev)
        assert (got["total"], got["early"], got["late"]) == (int(ref["visibility"]["total"][0]), ref["early"], ref["late"])
        np.testing.assert_array_equal(got["vis64"], ref["vis64"])
        np.testing.assert_array_equal(got["mask"], mask_ref)
    cam = sc.camera()
    cam["mesh_instance_count"] = 0  # cull_meshes.slang:28
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    ctx.cull_meshlets(cam, abi.CULL_TEST_ALL, True)
    ctx.cull_triangles(cam, abi.CULL_TEST_ALL)
    assert int(ctx.visibility()["total"][0]) == 0 and int(ctx.draw_cmd()["index_count"][0]) == 0
    ctx.free(vis_dev)
    ctx.close()


def test_call_sequence_errors(capi):
    ctx = capi.Context(0, 4, 64, 64, 64)
    cam = np.zeros(1, dtype=abi.CULL_CAMERA_DT)
    with pytest.raises(capi.OxcError):
        ctx.cull_meshes(cam)  # no scene
    with pytest.raises(capi.OxcError):
        capi.Context(0, 4, 64, 48, 64)  # non power-of-two hiz
    ctx.close()


def test_dequantize_half_all_inputs(capi, orc):
    """both device decoders vs the oracle for all 65536 half patterns (NaN payloads may differ: hardware quiets sNaNs)."""
    ctx = capi.Context(0, 1, 1, 64, 64)
    a, b = ctx.alloc(65536 * 4), ctx.alloc(65536 * 4)
    rc = ctx.lib.oxc_debug_dequantize_half(ctx.h, a, b, ctx.stream)
    assert rc == 0
    canon = ctx.download(a, np.float32, 65536)
    hw = ctx.download(b, np.float32, 65536)
    want = np.array([orc.dequantize_half(h) for h in range(65536)], dtype=np.float32)
    nan = np.isnan(want)
    # (signalling-NaN payloads are quietened when the oracle's float crosses ctypes: compare NaN-ness there)
    np.testing.assert_array_equal(canon[~nan].view(np.uint32), want[~nan].view(np.uint32))
    assert np.all(np.isnan(canon[nan]))
    np.testing.assert_array_equal(hw[~nan].view(np.uint32), want[~nan].view(np.uint32))
    assert np.all(np.isnan(hw[nan]))
    ctx.free(a)
    ctx.free(b)
    ctx.close()


def test_hiz_split_build_equals_single_pass(capi, orc):
    """multi-GPU split (mip 0 only -> [all_reduce] -> mips 1..) == the one-shot pyramid, packed source."""
    rng = np.random.default_rng(11)
    for (w, h) in [(1920, 1080), (100, 60)]:
        hw, hh = abi.hiz_extent(w, h)
        depth = rng.random((h, w), dtype=np.float32)
        packed = (depth.view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(0xFFFFFFFF)
        ref = orc.build_hiz(depth, orc.Hiz(hw, hh))
        ctx = capi.Context(0, 1, 1, hw, hh)
        v_dev = ctx.alloc(w * h * 8)
        ctx.upload(v_dev, packed)
        ctx.build_hiz_mip0_packed(v_dev, w, h)
        ctx.build_hiz_from_mip0()
        got = ctx.hiz_levels()
        for lvl in range(ref.levels):
            np.testing.assert_array_equal(got[lvl].view(np.uint32), ref.level(lvl).view(np.uint32), err_msg=f"{w}x{h} mip {lvl}")
        ctx.free(v_dev)
        ctx.close()


def test_renderer_persistent_depth_and_transform_updates(capi, orc):
    """oxr_set_external_depth + oxr_update_transforms (per-frame HOST inputs of the e2e bench) vs the oracle."""
    sc = synth.make_scene(config_index=2, **SCENES["small"])
    r = capi.Renderer(0, sc)
    r.set_external_depth(sc.occluder_depth)
    mask_ref = np.zeros((sc.max_meshlet_instance_count + 31) // 32, dtype=np.uint32)
    rng = np.random.default_rng(5)
    xf = sc.transforms.copy()
    for f in range(3):
        # move a third of the instances a little every frame
        sel = rng.random(len(xf)) < 0.33
        xf["world"][sel, 12:15] += rng.normal(0, 0.5, size=(int(sel.sum()), 3)).astype(np.float32)
        sc_f = synth.Scene(sc.meshes, sc.mesh_instances, xf.copy(), sc.blob, sc.max_meshlet_instance_count, sc.width, sc.height, sc.seed)
        hs = orc.HostScene(sc_f)
        cam = sc.camera(1.5 * f)
        ref = orc.frame(hs, cam, sc.width, sc.height, mask_ref, sc.occluder_depth)
        r.update_transforms(xf)
        got = r.render(cam, None)
        v32, d = orc.resolve(ref["vis64"])
        assert (got["total"], got["early"], got["late"]) == (int(ref["visibility"]["total"][0]), ref["early"], ref["late"])
        np.testing.assert_array_equal(got["vis32"], v32)
        np.testing.assert_array_equal(np.sort(got["visible"]), np.sort(ref["visible"][: ref["early"] + ref["late"]]))
        np.testing.assert_array_equal(r.ctx.mask(), mask_ref)
    r.close()


def test_renderer_pipelined_submit_wait(capi, orc):
    """oxr_submit / oxr_wait (two frames in flight, copy stream) deliver the same results as the oracle, frame by frame."""
    sc = synth.make_scene(config_index=2, **SCENES["small"])
    hs = orc.HostScene(sc)
    r = capi.Renderer(0, sc)
    r.set_external_depth(sc.occluder_depth)
    mask_ref = np.zeros((sc.max_meshlet_instance_count + 31) // 32, dtype=np.uint32)
    bufs = [dict(vis32=np.zeros((sc.height, sc.width), np.uint32), depth=np.zeros((sc.height, sc.width), np.float32),
                 idx=np.zeros(sc.max_meshlet_instance_count, np.uint32)) for _ in range(2)]
    refs, prev = [], None

    def check(frame_index, res):
        ref = refs[frame_index]
        b = bufs[frame_index % 2]
        assert (res["total"], res["early"], res["late"]) == ref[0]
        np.testing.assert_array_equal(b["vis32"], ref[1])
        np.testing.assert_array_equal(b["depth"].view(np.uint32), ref[2].view(np.uint32))
        np.testing.assert_array_equal(np.sort(b["idx"][: res["early"] + res["late"]]), ref[3])

    for f in range(5):
        cam = sc.camera(2.0 * f)
        ref = orc.frame(hs, cam, sc.width, sc.height, mask_ref, sc.occluder_depth)
        v32, d = orc.resolve(ref["vis64"])
        n = ref["early"] + ref["late"]
        refs.append(((int(ref["visibility"]["total"][0]), ref["early"], ref["late"]), v32, d, np.sort(ref["visible"][:n])))
        t = r.submit(cam, bufs[f % 2])
        if prev is not None:
            check(f - 1, r.wait(prev))
        prev = t
    check(4, r.wait(prev))
    np.testing.assert_array_equal(r.ctx.mask(), mask_ref)
    with pytest.raises(capi.OxcError):
        r.wait(0)  # nothing in flight
    r.close()


def test_terrain_cull_parity(capi, orc):
    """terrain_cull.slang equivalent (SURVEY §8f.3): early / late passes against a real Hi-Z, own mask, bit-exact."""
    rng = np.random.default_rng(21)
    w, h = 1280, 720
    hw, hh = abi.hiz_extent(w, h)
    terrain = np.zeros(1, dtype=abi.TERRAIN_DT)
    terrain["world_min"][0] = (-300.0, -500.0)
    terrain["world_size"][0] = (600.0, 600.0)
    terrain["patch_count"][0] = (96, 80)
    terrain["base_height"] = -30.0
    terrain["height_scale"] = 40.0
    n = 96 * 80
    lo = rng.random(n, dtype=np.float32) * 0.6
    minmax = np.stack([lo, lo + rng.random(n, dtype=np.float32) * 0.4], axis=1).astype(np.float32)
    minmax[::97, 1] = minmax[::97, 0]  # flat patches -> the 1e-3 floor of the extent
    depth = (rng.random((h, w), dtype=np.float32) * 0.02).astype(np.float32)
    depth[200:500, 300:900] = 0.01  # a large near occluder region
    ref_hiz = orc.build_hiz(depth, orc.Hiz(hw, hh))
    ctx = capi.Context(0, 1, 1, hw, hh)
    d_dev = ctx.alloc(w * h * 4); ctx.upload(d_dev, depth); ctx.build_hiz(d_dev, w, h)
    mm_dev = ctx.alloc(minmax.nbytes); ctx.upload(mm_dev, minmax)
    vis_dev, mask_dev, cmd_dev = ctx.alloc(n * 4), ctx.alloc(((n + 31) // 32) * 4), ctx.alloc(16)
    mask_ref = rng.integers(0, 2**32, size=(n + 31) // 32, dtype=np.uint64).astype(np.uint32)
    ctx.upload(mask_dev, mask_ref)
    cam = synth.make_camera(w, h, 0, yaw_deg=8.0, eye=(0.0, 5.0, 60.0))
    for flags in (abi.CULL_TEST_FRUSTUM | abi.CULL_TEST_OCCLUSION, abi.CULL_TEST_FRUSTUM | abi.CULL_TEST_OCCLUSION | abi.CULL_LATE_PASS,
                  abi.CULL_TEST_FRUSTUM):
        ref_vis, ref_cmd = orc.cull_terrain(terrain, minmax, cam, flags, ref_hiz, mask_ref)
        ctx.cull_terrain(terrain, mm_dev, cam, flags, vis_dev, mask_dev, cmd_dev)
        cmd = ctx.download(cmd_dev, abi.DRAW_INDIRECT_DT, 1)
        assert (int(cmd["vertex_count"][0]), int(cmd["instance_count"][0])) == (4, int(ref_cmd["instance_count"][0]))
        np.testing.assert_array_equal(np.sort(ctx.download(vis_dev, np.uint32, len(ref_vis))), np.sort(ref_vis))
        np.testing.assert_array_equal(ctx.download(mask_dev, np.uint32, len(mask_ref)), mask_ref)
        assert 0 < len(ref_vis) < n
    for p in (d_dev, mm_dev, vis_dev, mask_dev, cmd_dev):
        ctx.free(p)
    ctx.close()


def test_filtered_predicates_adversarial_boundaries(capi, orc):
    """Boxes steered (bisection on the f32 instance translation, evaluated with the oracle's own mvp + projection) so
    that a projected texel coordinate lands within ~1e-5 of an INTEGER Hi-Z texel boundary, and Hi-Z depths set within
    an ulp of the box's max.z: the filtered fast path must classify these as ambiguous and fall back to the canonical
    path -> decisions identical to the oracle."""
    import ctypes as C

    from tests.helpers_scene import boxes_scene

    w, h = 1920, 1080
    hw, hh = abi.hiz_extent(w, h)
    cam0 = synth.make_camera(w, h, 0)
    pv = np.ascontiguousarray(cam0["projection_view"][0], dtype=np.float32)
    rng = np.random.default_rng(99)
    n = 4000
    half = lambda a: np.asarray(a, np.float32).astype(np.float16).astype(np.float32)  # noqa: E731
    centers = half(np.stack([rng.uniform(-2, 2, n), rng.uniform(-2, 2, n), rng.uniform(-2, 2, n)], axis=1))
    extents = half(rng.uniform(0.2, 3.0, size=(n, 3)))
    trans = np.stack([rng.uniform(-40, 40, n), rng.uniform(-20, 20, n), -rng.uniform(20, 200, n)], axis=1).astype(np.float32)
    lib = orc.lib()

    def proj(i, t):
        wm = np.eye(4, dtype=np.float32)
        wm[3, :3] = t
        wflat = np.ascontiguousarray(wm.reshape(16))
        mvp = np.zeros(16, dtype=np.float32)
        lib.orc_mat4_mul(C.c_void_p(pv.ctypes.data), C.c_void_p(wflat.ctypes.data), C.c_void_p(mvp.ctypes.data))
        out = np.zeros(6, dtype=np.float32)
        cc, ee = np.ascontiguousarray(centers[i]), np.ascontiguousarray(extents[i])
        ok = lib.orc_project_aabb(C.c_void_p(mvp.ctypes.data), C.c_float(0.1), C.c_void_p(cc.ctypes.data),
                                  C.c_void_p(ee.ctypes.data), C.c_void_p(out.ctypes.data))
        return ok, out

    steered = 0
    for i in range(n):
        which = i % 4  # 0: min x, 1: max x, 2: min y, 3: max y
        col, size, axis = ((0, hw, 0), (3, hw, 0), (1, hh, 1), (4, hh, 1))[which]
        ok, o = proj(i, trans[i])
        if not ok:
            continue
        target = float(np.round(o[col] * size))
        if target < 2 or target > size - 3:
            continue
        t = trans[i].copy()
        lo, hi = np.float32(t[axis] - 1.0), np.float32(t[axis] + 1.0)
        t[axis] = lo; okl, ol = proj(i, t)
        t[axis] = hi; okh, oh = proj(i, t)
        if not (okl and okh):
            continue
        inc = oh[col] > ol[col]
        if not (min(ol[col], oh[col]) * size < target < max(ol[col], oh[col]) * size):
            continue
        for _ in range(60):
            mid = np.float32((np.float64(lo) + np.float64(hi)) / 2)
            if mid == lo or mid == hi:
                break
            t[axis] = mid
            _, om = proj(i, t)
            if (om[col] * size < target) == inc:
                lo = mid
            else:
                hi = mid
        trans[i, axis] = lo if i % 8 < 4 else hi
        steered += 1
    assert steered > n // 2
    sc, cdec, edec = boxes_scene(centers, extents, w, h, translations=trans)
    cam = synth.make_camera(w, h, sc.mesh_instance_count)
    hs = orc.HostScene(sc)
    # how close did we get?  (diagnostic: most steered coordinates are within 1e-4 texel of an integer)
    close = 0
    for i in range(0, n, 7):
        ok, o = proj(i, trans[i])
        col, size, _ = ((0, hw, 0), (3, hw, 0), (1, hh, 1), (4, hh, 1))[i % 4]
        if ok and abs(o[col] * size - np.round(o[col] * size)) < 1e-3:
            close += 1
    assert close > 50
    # Hi-Z: depth around every third box set within an ulp of (its max.z + 1e-7) so the final compare is tight too
    depth = np.zeros((h, w), dtype=np.float32)
    for i in range(0, n, 3):
        ok, o = proj(i, trans[i])
        if ok:
            x0, x1 = int(max(0, o[0] * w - 8)), int(min(w, o[3] * w + 8))
            y0, y1 = int(max(0, o[1] * h - 8)), int(min(h, o[4] * h + 8))
            z = np.float32(o[5]) + np.float32(1e-7)
            z = np.nextafter(z, np.float32(2.0 if i % 2 else -1.0))
            depth[y0:y1, x0:x1] = np.maximum(depth[y0:y1, x0:x1], z)
    ref_hiz = orc.build_hiz(depth, orc.Hiz(hw, hh))
    ctx = make_ctx(capi, sc)
    d_dev = ctx.alloc(w * h * 4)
    ctx.upload(d_dev, depth)
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    mask_ref = np.zeros(ctx.out.visibility_mask_words, dtype=np.uint32)
    flags = abi.CULL_TEST_ALL | abi.CULL_LATE_PASS
    ref_vis, _ = orc.cull_meshlets_hiz(hs, mi, vis, cam, flags, ref_hiz, mask_ref)
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    ctx.build_hiz(d_dev, w, h)
    ctx.cull_meshlets(cam, flags, True)
    nl = int(vis["late"][0])
    assert int(ctx.visibility()["late"][0]) == nl and 0 < nl < int(vis["total"][0])
    np.testing.assert_array_equal(np.sort(ctx.visible_indices(nl)), np.sort(ref_vis[:nl]))
    np.testing.assert_array_equal(ctx.mask(), mask_ref)
    ctx.free(d_dev)
    ctx.close()


def test_full_size_config1_parity(capi, orc):
    """BASELINE.json configs[1] at FULL size (1 M meshlet instances, 1920x1080): three two-pass frames through the C++
    host mirror, bit-exact against the (threaded) oracle frame: survivors, mask, vis buffer, depth, triangle counts."""
    import os

    sc = synth.make_scene(1_000_000, config_index=2, width=1920, height=1080)
    hs = orc.HostScene(sc)
    r = capi.Renderer(0, sc)
    r.set_external_depth(sc.occluder_depth)
    mask_ref = np.zeros((sc.max_meshlet_instance_count + 31) // 32, dtype=np.uint32)
    threads = min(64, os.cpu_count() or 1)
    for f in range(3):
        cam = sc.camera(2.0 * (f % 2))
        ref = orc.cpu_frame(hs, cam, sc.width, sc.height, mask_ref, sc.occluder_depth, threads)
        got = r.render(cam, None)
        e, l = int(ref["visibility"]["early"][0]), int(ref["visibility"]["late"][0])
        assert (got["total"], got["early"], got["late"]) == (int(ref["visibility"]["total"][0]), e, l)
        v32, d = orc.resolve(ref["vis64"])
        np.testing.assert_array_equal(got["vis32"], v32)
        np.testing.assert_array_equal(got["depth"].view(np.uint32), d.view(np.uint32))
        np.testing.assert_array_equal(np.sort(got["visible"]), np.sort(ref["visible"][: e + l]))
        np.testing.assert_array_equal(r.ctx.mask(), mask_ref)
        assert got["raster_triangles"] == ref["triangles"]
    r.close()


def test_full_size_config2_properties(capi):
    """BASELINE.json configs[2] at FULL size (10 M meshlet instances, 3840x2160): size-independent properties (the oracle
    would take minutes): survivor ids unique and in range; early and late sets disjoint; mask popcount == number of
    visible decisions; every vis-buffer id is a survivor of this frame; idempotence (same camera again -> same image,
    no new late survivors beyond the steady state); deterministic replay."""
    sc = synth.make_scene(10_000_000, config_index=3, width=3840, height=2160)
    r = capi.Renderer(0, sc)
    r.set_external_depth(sc.occluder_depth)
    cam = sc.camera(0.0)
    prev = None
    for f in range(4):  # 4 frames: the steady state (frames 2 -> 3) is part of what is checked
        got = r.render(cam, None)
        n = got["early"] + got["late"]
        ids = got["visible"]
        assert got["total"] == 10_000_000 and len(ids) == n
        assert ids.max() < got["total"] and len(np.unique(ids)) == n          # unique, in range
        mask = r.ctx.mask()
        pop = int(np.unpackbits(mask.view(np.uint8)).sum())
        assert pop <= n or f > 0                                               # frame 0: every set bit was emitted late
        if f == 0:
            assert got["early"] == 0 and pop == got["late"]                    # SURVEY quirk 2
        inst = got["vis32"][got["vis32"] != 0xFFFFFFFF] >> 8
        assert np.isin(np.unique(inst), ids).all()                             # drawn ids are survivors of this frame
        assert got["raster_triangles"] <= 64 * n
        if prev is not None and f >= 3:                                        # steady state: identical frames
            np.testing.assert_array_equal(got["vis32"], prev["vis32"])
            np.testing.assert_array_equal(np.sort(ids), np.sort(prev["visible"]))
            assert got["late"] == prev["late"]
        prev = got
    r.close()


def test_full_size_config2_parity(capi, orc):
    """BASELINE.json configs[2] at FULL size (10 M meshlet instances, 3840x2160 vis buffer, per-triangle cull + SW raster):
    two two-pass frames through the C++ host mirror, bit-exact against the threaded oracle frame — survivor set, visibility
    mask, packed image (ids + depth), triangle count."""
    import os

    sc = synth.make_scene(10_000_000, config_index=3, width=3840, height=2160)
    hs = orc.HostScene(sc)
    r = capi.Renderer(0, sc)
    r.set_external_depth(sc.occluder_depth)
    mask_ref = np.zeros((sc.max_meshlet_instance_count + 31) // 32, dtype=np.uint32)
    threads = min(64, os.cpu_count() or 1)
    for f in range(2):
        cam = sc.camera(2.0 * (f % 2))
        ref = orc.cpu_frame(hs, cam, sc.width, sc.height, mask_ref, sc.occluder_depth, threads)
        got = r.render(cam, None)
        e, l = int(ref["visibility"]["early"][0]), int(ref["visibility"]["late"][0])
        assert (got["total"], got["early"], got["late"]) == (int(ref["visibility"]["total"][0]), e, l)
        v32, d = orc.resolve(ref["vis64"])
        np.testing.assert_array_equal(got["vis32"], v32)
        np.testing.assert_array_equal(got["depth"].view(np.uint32), d.view(np.uint32))
        np.testing.assert_array_equal(np.sort(got["visible"]), np.sort(ref["visible"][: e + l]))
        np.testing.assert_array_equal(r.ctx.mask(), mask_ref)
        assert got["raster_triangles"] == ref["triangles"]
    # the pyramid the late pass used was built from the early image; its 2048^2 build is covered bit for bit by
    # test_hiz_build_shapes (3840x2160 included) and, here, by the late survivor set being identical
    assert r.ctx.check_status() == 0
    r.close()


def test_full_size_config3_multiview_parity(capi, orc):
    """BASELINE.json configs[3] at FULL size: 16 shadow-cascade views x 5 M meshlet instances in ONE batched launch; view
    bits and per-view counts bit-exact against the oracle (evaluated in parallel chunks: the C oracle releases the GIL)."""
    import os
    from concurrent.futures import ThreadPoolExecutor

    n_views = 16
    sc = synth.make_scene(5_000_000, config_index=4, width=1920, height=1080, placement="box")
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc, views=n_views)
    cam = sc.camera()
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    total = int(vis["total"][0])
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    assert int(ctx.visibility()["total"][0]) == total and total > 2_000_000
    dirs = synth.uniform(sc.seed, 90, 3 * n_views, -1.0, 1.0).reshape(n_views, 3)
    dirs[:, 1] = -np.abs(dirs[:, 1]) - 0.2
    views = np.concatenate([synth.make_ortho_view(dirs[v], (0.0, 0.0, -200.0), 60.0 * (1 + v % 4), 800.0, sc.mesh_instance_count)
                            for v in range(n_views)])
    workers = min(32, os.cpu_count() or 1)
    edges = np.linspace(0, total, workers * 4 + 1).astype(np.int64)

    def chunk(k):
        a, b = int(edges[k]), int(edges[k + 1])
        return orc.cull_meshlets_multiview(hs, np.ascontiguousarray(mi[a:b]), b - a, views, 1)

    with ThreadPoolExecutor(workers) as ex:
        parts = list(ex.map(chunk, range(len(edges) - 1)))
    ref_bits = np.concatenate([p[0] for p in parts])
    ref_counts = np.sum([p[1] for p in parts], axis=0).astype(np.uint32)
    ctx.cull_meshlets_multiview(views, 1)
    np.testing.assert_array_equal(ctx.view_bits(total), ref_bits)
    np.testing.assert_array_equal(ctx.view_counts(), ref_counts)
    ctx.close()


def test_cull_meshlets_hpb_parity(capi, orc):
    """cull_meshlets_hpb.slang equivalent: coarse view + 10 ortho clipmaps with page offsets, dirty flags, random R8UI page
    pyramid (64x64 pages, 7 mips); survivor set bit-exact."""
    sc = synth.make_scene(60000, config_index=4, width=1280, height=720, n_unique_meshes=32, placement="box")
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc, views=10)
    cam0 = sc.camera()
    mi, vis, _ = orc.cull_meshes(hs, cam0, abi.CULL_TEST_ALL)
    ctx.cull_meshes(cam0, abi.CULL_TEST_ALL)
    rng = np.random.default_rng(17)
    light = np.float64([0.3, -0.8, -0.5])
    n_clip = 10
    clip = np.zeros(n_clip, dtype=abi.CLIPMAP_DT)
    for c in range(n_clip):
        v = synth.make_ortho_view(light, (0.0, 0.0, -200.0), 12.0 * (1.6 ** c), 1200.0, sc.mesh_instance_count)
        clip["projection_view_mat"][c] = v["projection_view"][0]
        clip["page_offset"][c] = rng.integers(-40, 40, size=2)
        clip["z_near"][c] = 0.0
    coarse = synth.make_ortho_view(light, (0.0, 0.0, -200.0), 12.0 * (1.6 ** (n_clip - 1)), 1200.0, sc.mesh_instance_count)
    coarse["position"][0] = -light / np.linalg.norm(light)
    size, levels = 64, 7
    lv = [(rng.random((n_clip, size, size)) < 0.12).astype(np.uint8)]
    for l in range(1, levels):
        p = lv[l - 1]
        lv.append(np.maximum(np.maximum(p[:, 0::2, 0::2], p[:, 0::2, 1::2]), np.maximum(p[:, 1::2, 0::2], p[:, 1::2, 1::2])))
    hpb = np.concatenate([a.reshape(-1) for a in lv])
    hpb_dev = ctx.alloc(hpb.nbytes)
    ctx.upload(hpb_dev, hpb)
    for dirty in ([1] * n_clip, [1, 0, 1, 0, 0, 1, 0, 0, 0, 1], [0] * n_clip):
        ref, cmd = orc.cull_meshlets_hpb(hs, mi, vis, coarse, clip, dirty, hpb, size, levels)
        ctx.cull_meshlets_hpb(coarse, clip, dirty, hpb_dev, size, levels)
        n = int(cmd["x"][0])
        assert int(ctx.cull_triangles_cmd()["x"][0]) == n
        np.testing.assert_array_equal(np.sort(ctx.visible_indices(n)), np.sort(ref))
        assert (n == 0) == (sum(dirty) == 0)
    assert 0 < n_clip
    ctx.free(hpb_dev)
    ctx.close()


def _assert_planes_equal(got, ref, name):
    """bit-exact, except that NaNs only have to be NaNs (x86 and PTX disagree on the default NaN's sign / payload)"""
    g, r = got.view(np.uint32), ref.view(np.uint32)
    nan_g, nan_r = np.isnan(got), np.isnan(ref)
    np.testing.assert_array_equal(nan_g, nan_r, err_msg=name)
    np.testing.assert_array_equal(np.where(nan_g, 0, g), np.where(nan_r, 0, r), err_msg=name)


def _decode_gpu(ctx, cam, w, h, vis64_dev=None, vis32_dev=None, planes=("lambda_", "ddx", "ddy", "uv_normal", "uv_grad")):
    dev = {k: ctx.alloc(w * h * 16) for k in planes}
    ctx.decode_visbuffer(cam, w, h, dev, vis64_dev=vis64_dev, vis32_dev=vis32_dev)
    out = {k: ctx.download(p, np.float32, w * h * 4).reshape(h, w, 4) for k, p in dev.items()}
    for p in dev.values():
        ctx.free(p)
    return out


def test_decode_visbuffer_parity(capi, orc, scene):
    """visbuffer_decode.slang (geometry part): barycentrics, derivatives, uv (+ gradients), oct normal — every float
    bit-exact against the oracle, from the packed 64-bit image and from the resolved R32UI attachment; discarded
    texels (clear, terrain sentinel, out-of-range instance) produce zeros."""
    hs = orc.HostScene(scene)
    ctx = make_ctx(capi, scene)
    w, h = scene.width, scene.height
    vis_dev = ctx.alloc(w * h * 8)
    occ_dev = ctx.alloc(w * h * 4)
    ctx.upload(occ_dev, scene.occluder_depth)
    mask_ref = np.zeros(ctx.out.visibility_mask_words, dtype=np.uint32)
    for f in range(2):
        cam = scene.camera(2.0 * f)
        ref = orc.frame(hs, cam, w, h, mask_ref, scene.occluder_depth)
        got = _frame_gpu(capi, ctx, scene, cam, occ_dev, vis_dev)
        np.testing.assert_array_equal(got["vis64"], ref["vis64"])
    total = int(ref["visibility"]["total"][0])
    v32, _ = orc.resolve(ref["vis64"])
    want = orc.decode_visbuffer(hs, ref["meshlet_instances"], total, cam, v32)
    assert (want["lambda_"][:, :, 3] == 1.0).sum() > 100
    dec = _decode_gpu(ctx, cam, w, h, vis64_dev=vis_dev)
    for k in want:
        _assert_planes_equal(dec[k], want[k], k)
    # R32UI input + hostile texels + a subset of planes
    v32b = v32.copy()
    v32b[0, :7] = [(0xFFFFFE << 8) | 5, ((total + 3) << 8) | 1, (total << 8), 0xFFFFFF00, ((total - 1) << 8), 0, 0xFFFFFFFF]
    want = orc.decode_visbuffer(hs, ref["meshlet_instances"], total, cam, v32b)
    v32_dev = ctx.alloc(w * h * 4)
    ctx.upload(v32_dev, v32b)
    dec = _decode_gpu(ctx, cam, w, h, vis32_dev=v32_dev, planes=("lambda_", "uv_normal"))
    for k in dec:
        _assert_planes_equal(dec[k], want[k], k)
    with pytest.raises(capi.OxcError):
        ctx.decode_visbuffer(cam, w, h, {}, vis64_dev=vis_dev, vis32_dev=v32_dev)
    for p in (vis_dev, occ_dev, v32_dev):
        ctx.free(p)
    ctx.close()


def test_decode_visbuffer_full_size(capi, orc):
    """configs[1] at full size: decode of the steady-state 1920x1080 frame, bit-exact; also meshes without vertex
    attributes (null pointers) and the vertex-index range check."""
    import os

    sc = synth.make_scene(1_000_000, config_index=2, width=1920, height=1080)
    hs = orc.HostScene(sc)
    r = capi.Renderer(0, sc)
    r.set_external_depth(sc.occluder_depth)
    mask_ref = np.zeros((sc.max_meshlet_instance_count + 31) // 32, dtype=np.uint32)
    threads = min(64, os.cpu_count() or 1)
    cam = sc.camera(0.0)
    for f in range(2):
        ref = orc.cpu_frame(hs, cam, sc.width, sc.height, mask_ref, sc.occluder_depth, threads)
        got = r.render(cam, None)
    v32, _ = orc.resolve(ref["vis64"])
    np.testing.assert_array_equal(got["vis32"], v32)
    total = int(ref["visibility"]["total"][0])
    want = orc.decode_visbuffer(hs, ref["meshlet_instances"], total, cam, v32)
    ctx = r.ctx
    v32_dev = ctx.alloc(v32.nbytes)
    ctx.upload(v32_dev, v32)
    dec = _decode_gpu(ctx, cam, sc.width, sc.height, vis32_dev=v32_dev)
    assert (dec["lambda_"][:, :, 3] == 1.0).sum() > 200_000
    for k in want:
        _assert_planes_equal(dec[k], want[k], k)
    ctx.free(v32_dev)
    r.close()


def test_decode_null_attributes_and_index_guard(capi, orc):
    from tests.helpers_scene import quad_scene

    W = H = 16
    for attributes, vertex_count in ((False, 4), (True, 4), (True, 2)):
        sc, cam = quad_scene(W, H, attributes=attributes)
        sc.meshes["vertex_count"] = vertex_count
        hs = orc.HostScene(sc)
        ctx = make_ctx(capi, sc)
        mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
        ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
        v32 = np.full((H, W), 0xFFFFFFFF, dtype=np.uint32)
        v32[4:12, 4:12] = np.arange(64).reshape(8, 8) % 2
        want = orc.decode_visbuffer(hs, mi, 1, cam, v32)
        v32_dev = ctx.alloc(v32.nbytes)
        ctx.upload(v32_dev, v32)
        dec = _decode_gpu(ctx, cam, W, H, vis32_dev=v32_dev)
        for k in want:
            _assert_planes_equal(dec[k], want[k], f"{k} attributes={attributes} vertex_count={vertex_count}")
        assert (dec["lambda_"][4:12, 4:12, 3] == (1.0 if vertex_count == 4 else 2.0)).all()
        ctx.free(v32_dev)
        ctx.close()


def test_build_hpb_parity(capi, orc):
    """rmvsm_downsample_hpb.slang: page table -> hierarchical page bitmap, fused single-launch path (size <= 256) and
    the per-level path, exact; the result drives oxc_cull_meshlets_hpb identically to the oracle's pyramid."""
    sc = synth.make_scene(2000, config_index=2, width=640, height=360, n_unique_meshes=8)
    ctx = make_ctx(capi, sc)
    rng = np.random.default_rng(23)
    for size, layers, levels in ((128, 10, 8), (64, 3, 7), (256, 2, 9), (512, 2, 10), (1, 1, 1), (4, 2, 5), (96, 1, 4)):
        pt = (rng.integers(0, 32, size=(layers, size, size)).astype(np.uint32)
              | (rng.integers(0, 65536, size=(layers, size, size)).astype(np.uint32) << 16))
        pt[rng.random(pt.shape) < 0.7] &= ~np.uint32(1)  # most pages invisible: sparse pyramid like a real frame
        want = orc.build_hpb(pt, levels)
        pt_dev, hpb_dev = ctx.alloc(pt.nbytes), ctx.alloc(want.nbytes)
        ctx.upload(pt_dev, pt)
        ctx.upload(hpb_dev, np.full(want.nbytes, 0xAB, dtype=np.uint8))
        ctx.build_hpb(pt_dev, size, layers, hpb_dev, levels)
        got = ctx.download(hpb_dev, np.uint8, want.nbytes)
        np.testing.assert_array_equal(got, want, err_msg=f"size {size} layers {layers} levels {levels}")
        ctx.free(pt_dev)
        ctx.free(hpb_dev)
    ctx.close()


def test_mgpu_api_single_rank(capi, orc):
    """oxc_mgpu_* with a communicator of ONE rank (what a 1-GPU box can run; 2 and 8 ranks are checked against one GPU by
    tools/check_multi_gpu.py and inside bench.py): exchange_hiz == generate_hiz, exchange_frame gathers this rank's
    counters and survivors, an undersized gather segment raises the overflow status."""
    import torch

    from oxylus_b200 import pipeline

    sc = synth.make_scene(config_index=2, **SCENES["box"])
    hs = orc.HostScene(sc)
    uid = capi.Context.mgpu_unique_id()
    assert len(uid) == abi.MGPU_ID_BYTES
    pipe = pipeline.VisibilityPipeline(sc, device=0, shard=(0, sc.mesh_instance_count), auto_id_base=True,
                                       mgpu=dict(rank=0, world=1, unique_id=uid, survivor_capacity=sc.max_meshlet_instance_count))
    info = pipe.ctx.mgpu_info()
    assert (info.active, info.rank, info.world) == (1, 0, 1)
    mask_ref = np.zeros((sc.max_meshlet_instance_count + 31) // 32, dtype=np.uint32)
    for f in range(3):
        cam = sc.camera(2.0 * f)
        ref = orc.frame(hs, cam, sc.width, sc.height, mask_ref, sc.occluder_depth)
        pipe.frame(cam)
        pipe.exchange_frame(slot=f & 1)
        torch.cuda.synchronize()
        assert pipe.ctx.check_status() == 0
        cnt, ids = pipe.ctx.mgpu_gathered(f & 1)
        e, l = ref["early"], ref["late"]
        assert cnt.tolist() == [[int(ref["visibility"]["total"][0]), e, l, e + l]]
        np.testing.assert_array_equal(np.sort(ids[0]), np.sort(ref["visible"][: e + l]))
        np.testing.assert_array_equal(pipe.vis64.cpu().numpy().view(np.uint64), ref["vis64"])
        for a, b in zip(pipe.ctx.hiz_levels(), [ref["hiz"].level(k) for k in range(len(pipe.ctx.hiz_levels()))]):
            np.testing.assert_array_equal(a.view(np.uint32), np.asarray(b).view(np.uint32))
    pipe.close()
    # a gather segment smaller than the survivor list is a hard error, not a truncation
    pipe = pipeline.VisibilityPipeline(sc, device=0, shard=(0, sc.mesh_instance_count), auto_id_base=True,
                                       mgpu=dict(rank=0, world=1, unique_id=capi.Context.mgpu_unique_id(), survivor_capacity=16))
    pipe.frame(sc.camera(0.0))
    pipe.exchange_frame(slot=0)
    torch.cuda.synchronize()
    assert pipe.ctx.status_flags() & abi.STATUS_SURVIVOR_OVERFLOW
    with pytest.raises(capi.OxcError, match="gather capacity"):
        pipe.ctx.check_status()
    pipe.close()


def test_mark_visible_pages_parity(capi, orc):
    """rmvsm_mark_visible_pages.slang equivalent vs the oracle on a 1920x1080 depth image of a ground plane: page tables and
    occupancy bit for bit, allocation requests as a set (push order is atomics order in the reference too)."""
    from tests.test_oracle_units import make_vsm_case

    sc = synth.make_scene(config_index=2, **SCENES["small"])
    ctx = make_ctx(capi, sc)
    for (w, h, size) in ((1920, 1080, 64), (333, 177, 48)):
        inv_pv, res, cm, vsm, depth, pt0 = make_vsm_case(w, h, size=size)
        pt_ref = pt0.copy()
        occ_ref = np.zeros(32 * 32, dtype=np.uint32)
        cap = 1 << 16
        req_ref, n_ref = orc.mark_visible_pages(inv_pv, res, cm, vsm, depth, pt_ref, occ_ref, cap)
        assert n_ref > 100
        d_depth, d_pt, d_occ = ctx.alloc(depth.nbytes), ctx.alloc(pt0.nbytes), ctx.alloc(occ_ref.nbytes)
        d_cnt, d_req = ctx.alloc(4), ctx.alloc(cap * 12)
        ctx.upload(d_depth, depth); ctx.upload(d_pt, pt0); ctx.upload(d_occ, np.zeros_like(occ_ref)); ctx.upload(d_cnt, np.zeros(1, np.uint32))
        ctx.mark_visible_pages(inv_pv, res, cm, vsm, d_depth, d_pt, d_occ, d_cnt, d_req, cap)
        np.testing.assert_array_equal(ctx.download(d_pt, np.uint32, pt0.size).reshape(pt0.shape), pt_ref)
        np.testing.assert_array_equal(ctx.download(d_occ, np.uint32, occ_ref.size), occ_ref)
        n = int(ctx.download(d_cnt, np.uint32, 1)[0])
        assert n == n_ref
        got = ctx.download(d_req, np.int32, n * 3).reshape(-1, 3)
        assert sorted(map(tuple, got.tolist())) == sorted(map(tuple, req_ref.tolist()))
        # second call on the updated tables: everything is visible already -> no new request
        ctx.upload(d_cnt, np.zeros(1, np.uint32))
        ctx.mark_visible_pages(inv_pv, res, cm, vsm, d_depth, d_pt, d_occ, d_cnt, d_req, cap)
        assert int(ctx.download(d_cnt, np.uint32, 1)[0]) == 0
        for d in (d_depth, d_pt, d_occ, d_cnt, d_req):
            ctx.free(d)
    ctx.close()


def test_builder_scene_parity(capi, orc):
    """content produced by the mesh builder (oxb_build_mesh: scan meshlets, meshopt-style bounds / cones, 2 LODs) through
    the whole GPU path: cull_meshes (LOD selection), two-pass frames, raster, decode — bit-exact against the oracle; and
    oxc_set_scene rejects a blob whose meshlet table is not 16-byte aligned instead of faulting later."""
    from tests.test_builder_cpu import torus

    pos, nrm, uv, i0, i1 = torus(128, 64)
    pos2, nrm2, uv2, j0, j1 = torus(40, 20, R=1.0, r=0.45, seed=9)
    built = [capi.BuiltMesh(pos, [(i0, 0.0), (i1, 0.03)], normals=nrm, texcoords=uv),
             capi.BuiltMesh(pos2, [(j0, 0.0), (j1, 0.08)], normals=nrm2)]
    rng = np.random.default_rng(11)
    n = 160
    xf = np.zeros((n, 4, 4), dtype=np.float32)  # [col][row]
    for i in range(n):
        q = rng.standard_normal(4)
        q /= np.linalg.norm(q)
        w, x, y, z = q
        rot = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                        [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                        [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        s = rng.uniform(0.4, 2.5, size=3)  # non-uniform scale
        m = np.eye(4)
        m[:3, :3] = rot * s[None, :]
        m[:3, 3] = (rng.uniform(-60, 60), rng.uniform(-25, 25), -rng.uniform(6, 220))
        xf[i] = m.T
    sc = capi.assemble_scene(built, rng.integers(0, 2, size=n), xf.reshape(n, 16), 1280, 720)
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc, reordered=True)
    w, h = sc.width, sc.height
    vis_dev = ctx.alloc(w * h * 8)
    mask_ref = np.zeros(ctx.out.visibility_mask_words, dtype=np.uint32)
    for f in range(3):
        cam = sc.camera(3.0 * f)
        ref = orc.frame(hs, cam, w, h, mask_ref, None)
        got = _frame_gpu(capi, ctx, sc, cam, None, vis_dev)
        total = int(ref["visibility"]["total"][0])
        assert (got["total"], got["early"], got["late"]) == (total, ref["early"], ref["late"])
        np.testing.assert_array_equal(ctx.meshlet_instances(total), ref["meshlet_instances"][:total])
        np.testing.assert_array_equal(ctx.mesh_instances(n)["lod_index"], hs.mesh_instances["lod_index"])
        np.testing.assert_array_equal(np.sort(got["visible"]), np.sort(ref["visible"][: ref["early"] + ref["late"]]))
        np.testing.assert_array_equal(got["mask"], mask_ref)
        np.testing.assert_array_equal(got["vis64"], ref["vis64"])
        for a, b in zip(got["hiz"], [ref["hiz"].level(l) for l in range(ref["hiz"].levels)]):
            np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))
    assert len(set(hs.mesh_instances["lod_index"])) == 2 and ref["early"] > 100
    v32, _ = orc.resolve(ref["vis64"])
    want = orc.decode_visbuffer(hs, ref["meshlet_instances"], total, cam, v32)
    dec = _decode_gpu(ctx, cam, w, h, vis64_dev=vis_dev)
    assert (dec["lambda_"][:, :, 3] == 1.0).sum() > 20000
    for k in want:
        _assert_planes_equal(dec[k], want[k], k)
    # meshlet table at a 4-byte offset -> OXC_E_INVALID from oxc_set_scene (8-byte alignment is the reference's layout
    # and is accepted: test_reference_blob_alignment_is_accepted)
    bad = capi.assemble_scene(built, [0], xf.reshape(n, 16)[:1], 64, 64)
    lods = np.frombuffer(bad.blob, dtype=abi.MESH_LOD_DT, count=1, offset=int(bad.meshes["lods"][0]))
    lods = lods.copy()
    lods["meshlets"] += 4
    bad.blob[int(bad.meshes["lods"][0]): int(bad.meshes["lods"][0]) + 64] = lods.view(np.uint8)
    with pytest.raises(capi.OxcError):
        ctx.set_scene(bad)
    ctx.free(vis_dev)
    ctx.close()


def test_reference_blob_alignment_is_accepted(capi, orc):
    """The reference's builder aligns the Meshlet / MeshletBounds tables to 8 bytes (blob_append(..., 8),
    AssetManager_GLTF.cpp:749-750) while the kernels load those records as 128-bit words: oxc_set_scene relocates such
    tables inside its device copy.  The same scene with every blob offset shifted by 8 bytes gives identical frames."""
    sc = synth.make_scene(20000, config_index=2, width=960, height=540, n_unique_meshes=24, max_lods=3, ragged=True)
    shifted = synth.Scene(sc.meshes.copy(), sc.mesh_instances.copy(), sc.transforms.copy(),
                          np.concatenate([np.zeros(8, dtype=np.uint8), sc.blob, np.zeros(8, dtype=np.uint8)]),
                          sc.max_meshlet_instance_count, sc.width, sc.height, sc.seed, occluder_depth=sc.occluder_depth)
    for f in ("vertex_positions", "vertex_normals", "texture_coords", "lods"):
        shifted.meshes[f] = np.where(sc.meshes[f] != 0, sc.meshes[f] + 8, 0) if f in ("vertex_normals", "texture_coords") else sc.meshes[f] + 8
    for m in shifted.meshes:
        lods = np.frombuffer(shifted.blob, dtype=abi.MESH_LOD_DT, count=int(m["lod_count"]), offset=int(m["lods"])).copy()
        for f in ("indices", "meshlets", "meshlet_bounds", "local_triangle_indices", "indirect_vertex_indices"):
            lods[f] += 8
        shifted.blob[int(m["lods"]): int(m["lods"]) + lods.nbytes] = lods.view(np.uint8)
    lod0 = np.frombuffer(shifted.blob, dtype=abi.MESH_LOD_DT, count=1, offset=int(shifted.meshes["lods"][0]))[0]
    assert lod0["meshlets"] % 16 == 8 and lod0["meshlet_bounds"] % 16 == 8
    w, h = sc.width, sc.height
    results = []
    for scene_ in (sc, shifted):
        ctx = make_ctx(capi, scene_)
        vis_dev = ctx.alloc(w * h * 8)
        occ_dev = ctx.alloc(w * h * 4)
        ctx.upload(occ_dev, sc.occluder_depth)
        frames = [_frame_gpu(capi, ctx, scene_, sc.camera(2.0 * f), occ_dev, vis_dev) for f in range(2)]
        results.append(frames)
        ctx.free(vis_dev)
        ctx.free(occ_dev)
        ctx.close()
    hs = orc.HostScene(shifted)   # the oracle reads the shifted blob directly (no alignment requirement)
    mask_ref = np.zeros((sc.max_meshlet_instance_count + 31) // 32, dtype=np.uint32)
    for f in range(2):
        a, b = results[0][f], results[1][f]
        ref = orc.frame(hs, sc.camera(2.0 * f), w, h, mask_ref, sc.occluder_depth)
        assert (a["total"], a["early"], a["late"], a["ntri"]) == (b["total"], b["early"], b["late"], b["ntri"])
        assert (b["early"], b["late"]) == (ref["early"], ref["late"])
        np.testing.assert_array_equal(a["vis64"], b["vis64"])
        np.testing.assert_array_equal(b["vis64"], ref["vis64"])
        np.testing.assert_array_equal(a["mask"], b["mask"])
        np.testing.assert_array_equal(np.sort(a["visible"]), np.sort(b["visible"]))


def test_clear_with_depth_equals_clear_then_merge(capi):
    """oxc_clear_visbuffer_with_depth == oxc_clear_visbuffer + oxc_merge_depth for every depth bit pattern class
    (zeros, ones, denormals, negative, inf, NaN payloads)"""
    sc = synth.make_scene(2000, config_index=2, width=256, height=128, n_unique_meshes=4)
    ctx = make_ctx(capi, sc)
    w, h = 256, 128
    rng = np.random.default_rng(5)
    bits = rng.integers(0, 2**32, size=w * h, dtype=np.uint64).astype(np.uint32)
    bits[:8] = [0, 0x80000000, 0x3F800000, 0x7F800000, 0xFF800000, 0x7FC00001, 0x00000001, 0xFFFFFFFF]
    depth = bits.view(np.float32)
    d_dev, a_dev, b_dev = ctx.alloc(w * h * 4), ctx.alloc(w * h * 8), ctx.alloc(w * h * 8)
    ctx.upload(d_dev, depth)
    ctx.clear_visbuffer(a_dev, w, h)
    ctx.merge_depth(a_dev, d_dev, w, h)
    ctx.upload(b_dev, np.full(w * h, 0x1234567812345678, dtype=np.uint64))
    ctx.clear_visbuffer_with_depth(b_dev, d_dev, w, h)
    a, b = ctx.download(a_dev, np.uint64, w * h), ctx.download(b_dev, np.uint64, w * h)
    np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(b >> np.uint64(32), bits.astype(np.uint64))
    assert ctx.raster_triangle_count() == 0
    for p in (d_dev, a_dev, b_dev):
        ctx.free(p)
    ctx.close()


def test_raster_big_triangle_queue_and_overflow(capi, orc):
    """large triangles are deferred to k_raster_big in <= 64x32-pixel chunks; when the queue is full (or a reservation
    straddles its end) they are rasterised inline — the image is the oracle's either way"""
    import os

    from tests.helpers_scene import quad_scene

    W = H = 256
    sc, cam = quad_scene(W, H, depth_a=0.3, depth_b=0.7)
    hs = orc.HostScene(sc)
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    visible = np.zeros(1, dtype=np.uint32)
    ref = orc.clear_visbuffer(W, H)
    ntri, _ = orc.raster_clip(hs, mi, visible, 0, 1, cam, ref)
    assert ntri == 2 and (ref != 0xFFFFFFFF).sum() > 10000
    for cap in (None, 5, 12, 1):
        if cap is None:
            os.environ.pop("OXC_BIG_CAPACITY", None)
        else:
            os.environ["OXC_BIG_CAPACITY"] = str(cap)
        try:
            ctx = make_ctx(capi, sc)
        finally:
            os.environ.pop("OXC_BIG_CAPACITY", None)
        vis_dev = ctx.alloc(W * H * 8)
        for _ in range(2):  # twice: the counters are reset per launch
            ctx.clear_visbuffer(vis_dev, W, H)
            ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
            ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, False)
            ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, W, H, vis_dev)
            got = ctx.download(vis_dev, np.uint64, W * H).reshape(H, W)
            np.testing.assert_array_equal(got, ref, err_msg=f"capacity {cap}")
            assert ctx.raster_triangle_count() == 2
        ctx.free(vis_dev)
        ctx.close()


def test_clip_pass_parity(capi, orc):
    """Near / side-plane clipping vs the oracle's clipped raster: a ground plane through the camera (coarse: 2 huge triangles;
    medium: 24x24 quads, some of them crossing the near / side planes).  oxc_raster_visbuffer queues the triangles the plain
    rules drop and clips them itself; the stand-alone oxc_raster_visbuffer_clip_pass on top changes nothing; with the queue
    exhausted (1 entry) the status word says so and the stand-alone pass completes the image."""
    import os
    from tests.test_oracle_clip import ground_scene

    for cells in (1, 24):
        sc = ground_scene(cells, width=640, height=360)
        hs = orc.HostScene(sc)
        cam = sc.camera()
        w, h = sc.width, sc.height
        mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
        visible, cmd = orc.cull_meshlets(hs, mi, vis, cam)
        visible = visible[: int(cmd["x"][0])]
        ref = orc.clear_visbuffer(w, h)
        ntri, nclip = orc.raster_clip(hs, mi, visible, 0, len(visible), cam, ref)
        assert nclip > 0
        ref_plain = orc.clear_visbuffer(w, h)
        orc.raster(hs, mi, visible, 0, len(visible), cam, ref_plain)
        assert not np.array_equal(ref, ref_plain)  # the clipped triangles do cover pixels
        for capacity in (None, "1"):
            if capacity:
                os.environ["OXC_CLIP_CAPACITY"] = capacity
            try:
                ctx = make_ctx(capi, sc)
            finally:
                os.environ.pop("OXC_CLIP_CAPACITY", None)
            vis_dev = ctx.alloc(w * h * 8)
            ctx.clear_visbuffer(vis_dev, w, h)
            ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
            ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, False)
            ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis_dev)
            got = ctx.download(vis_dev, np.uint64, w * h).reshape(h, w)
            if capacity is None:
                np.testing.assert_array_equal(got, ref)
                assert ctx.check_status() == 0
            elif nclip > 1:
                assert ctx.status_flags() & abi.STATUS_CLIP_OVERFLOW
                with pytest.raises(capi.OxcError):
                    ctx.check_status()
            ctx.raster_visbuffer_clip_pass(cam, abi.CULL_TEST_ALL, w, h, vis_dev)
            got = ctx.download(vis_dev, np.uint64, w * h).reshape(h, w)
            np.testing.assert_array_equal(got, ref)
            assert ctx.raster_triangle_count() == ntri
            ctx.free(vis_dev)
            ctx.close()


def _alpha_tables(capi, orc, ctx):
    """four materials (opaque; RGBA8 checker, linear + repeat; R8 noise, nearest + clamp, albedo alpha 0.8; R8 gradient, linear +
    mirrored / repeat) as an oracle table (host texels) and set on the context (device texels)"""
    from tests.test_oracle_alpha import checker, material

    rng = np.random.default_rng(5)
    images = [(checker(16, 2), abi.IMAGE_RGBA8_UNORM), (rng.integers(0, 256, (8, 8), dtype=np.uint8), abi.IMAGE_R8_UNORM),
              (np.ascontiguousarray(np.tile(np.linspace(0, 255, 16).astype(np.uint8), (16, 1))), abi.IMAGE_R8_UNORM)]
    mats = np.array([material(), material(image=0, cutoff=0.5), material(image=1, cutoff=0.3, albedo_a=0.8, sampler=1),
                     material(image=2, cutoff=0.5, sampler=2)], dtype=abi.MATERIAL_DT)
    smp = np.array([abi.sampler(), abi.sampler(abi.FILTER_NEAREST, abi.FILTER_NEAREST, u=abi.ADDRESS_CLAMP_TO_EDGE, v=abi.ADDRESS_CLAMP_TO_EDGE),
                    abi.sampler(u=abi.ADDRESS_MIRRORED_REPEAT)], dtype=abi.SAMPLER_DT)
    tab = orc.MaterialTable(mats, images, smp)
    dev, ptrs = tab.device_images(ctx)
    ctx.set_materials(mats, dev, smp)
    return tab, ptrs


def test_alpha_discard_parity(capi, orc):
    """visbuffer_encode.slang:54-66: with a material table set, the raster discards fragments whose albedo alpha is below the
    cutoff.  Two-pass frames (so the holes reach the Hi-Z and the late cull) on a scene whose mesh instances cycle through four
    materials: survivors, mask, packed image and triangle count equal the oracle's frame bit for bit; switching the table off
    again gives the plain frame; a material index outside the table raises OXC_STATUS_BAD_MATERIAL."""
    sc = synth.make_scene(config_index=2, **SCENES["small"])
    sc.mesh_instances["material_index"] = np.arange(sc.mesh_instance_count) % 4
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc)
    tab, texels = _alpha_tables(capi, orc, ctx)
    w, h = sc.width, sc.height
    vis_dev = ctx.alloc(w * h * 8)
    occ_dev = ctx.alloc(w * h * 4)
    ctx.upload(occ_dev, sc.occluder_depth)
    mask_ref = np.zeros(ctx.out.visibility_mask_words, dtype=np.uint32)
    mask_plain = np.zeros_like(mask_ref)
    differs = False
    for f in range(3):
        cam = sc.camera(2.0 * f)
        ref = orc.frame(hs, cam, w, h, mask_ref, sc.occluder_depth, materials=tab)
        plain = orc.frame(orc.HostScene(sc), cam, w, h, mask_plain, sc.occluder_depth)
        differs = differs or not np.array_equal(ref["vis64"], plain["vis64"])
        got = _frame_gpu(capi, ctx, sc, cam, occ_dev, vis_dev)
        assert (got["early"], got["late"]) == (ref["early"], ref["late"]), f"frame {f}"
        np.testing.assert_array_equal(got["mask"], mask_ref)
        e, l = ref["early"], ref["late"]
        np.testing.assert_array_equal(np.sort(got["visible"][:e]), np.sort(ref["visible"][:e]))
        np.testing.assert_array_equal(np.sort(got["visible"][e : e + l]), np.sort(ref["visible"][e : e + l]))
        np.testing.assert_array_equal(got["vis64"], ref["vis64"])
        assert got["ntri"] == ref["ntri_early"] + ref["ntri_late"]
        assert ctx.check_status() == 0
    assert differs  # the table does discard fragments in this scene
    # table off: the plain encode again (mask continues from the alpha frames on both sides)
    ctx.set_materials(None)
    cam = sc.camera(6.0)
    ref = orc.frame(hs, cam, w, h, mask_ref, sc.occluder_depth)
    got = _frame_gpu(capi, ctx, sc, cam, occ_dev, vis_dev)
    np.testing.assert_array_equal(got["vis64"], ref["vis64"])
    np.testing.assert_array_equal(got["mask"], mask_ref)
    # a material index outside the table: rasterised as opaque, flagged
    from tests.test_oracle_alpha import material

    ctx.set_materials(np.array([material()], dtype=abi.MATERIAL_DT))  # 1 material, no image: the test stays off, nothing to flag
    _frame_gpu(capi, ctx, sc, cam, occ_dev, vis_dev)
    assert ctx.check_status() == 0
    tab1, tex1 = _alpha_tables(capi, orc, ctx)
    sc2 = synth.make_scene(config_index=2, **SCENES["small"])
    sc2.mesh_instances["material_index"] = np.where(np.arange(sc2.mesh_instance_count) % 5 == 0, 9, 1)
    ctx.set_scene(sc2)
    ctx.reset_visibility_mask()
    got = _frame_gpu(capi, ctx, sc2, cam, occ_dev, vis_dev)
    assert ctx.status_flags() & abi.STATUS_BAD_MATERIAL
    with pytest.raises(capi.OxcError):
        ctx.check_status()
    # ... and the image is the oracle's, which treats such instances as opaque too
    ref = orc.frame(orc.HostScene(sc2), cam, w, h, np.zeros_like(mask_ref), sc2.occluder_depth, materials=tab1)
    np.testing.assert_array_equal(got["vis64"], ref["vis64"])
    for d in texels + tex1 + [vis_dev, occ_dev]:
        ctx.free(d)
    ctx.close()


def test_renderer_alpha_discard_pipelined(capi, orc):
    """oxr_set_materials on the host mirror: the pipelined frames (oxr_submit / oxr_wait replay the frame from CUDA graphs) are
    re-captured with the alpha kernels in them when the table is set and again when it is removed — every frame equals the
    oracle's frame with / without the table"""
    sc = synth.make_scene(config_index=2, **SCENES["small"])
    sc.mesh_instances["material_index"] = np.arange(sc.mesh_instance_count) % 4
    hs = orc.HostScene(sc)
    r = capi.Renderer(0, sc)
    r.set_external_depth(sc.occluder_depth)
    tab, texels = _alpha_tables(capi, orc, r.ctx)  # sets the table on the context; the renderer call below is what drops the graphs
    r.set_materials(None)
    mask_ref = np.zeros((sc.max_meshlet_instance_count + 31) // 32, dtype=np.uint32)
    bufs = [dict(vis32=np.zeros((sc.height, sc.width), np.uint32), depth=np.zeros((sc.height, sc.width), np.float32),
                 idx=np.zeros(sc.max_meshlet_instance_count, np.uint32)) for _ in range(2)]
    images = [(d, int(im["width"]), int(im["height"]), int(im["format"]), int(im["level_count"])) for d, im in zip(texels, tab.images)]
    with_table = [False, False, True, True, True, False, False]
    refs, prev = [], None

    def check(frame_index, res):
        ref = refs[frame_index]
        b = bufs[frame_index % 2]
        assert (res["total"], res["early"], res["late"]) == ref[0], frame_index
        np.testing.assert_array_equal(b["vis32"], ref[1])
        np.testing.assert_array_equal(b["depth"].view(np.uint32), ref[2].view(np.uint32))
        np.testing.assert_array_equal(np.sort(b["idx"][: res["early"] + res["late"]]), ref[3])

    for f, on in enumerate(with_table):
        cam = sc.camera(2.0 * f)
        if f and on != with_table[f - 1]:
            if prev is not None:  # the table belongs to the frames in flight: drain before changing it
                check(f - 1, r.wait(prev))
                prev = None
            r.set_materials(tab.materials if on else None, images, tab.samplers)
        ref = orc.frame(hs, cam, sc.width, sc.height, mask_ref, sc.occluder_depth, materials=tab if on else None)
        v32, d = orc.resolve(ref["vis64"])
        n = ref["early"] + ref["late"]
        refs.append(((int(ref["visibility"]["total"][0]), ref["early"], ref["late"]), v32, d, np.sort(ref["visible"][:n])))
        t = r.submit(cam, bufs[f % 2])
        if prev is not None:
            check(f - 1, r.wait(prev))
        prev = t
    check(len(with_table) - 1, r.wait(prev))
    np.testing.assert_array_equal(r.ctx.mask(), mask_ref)
    assert not np.array_equal(refs[1][1], refs[2][1])
    for d in texels:
        r.ctx.free(d)
    r.close()


def test_alpha_discard_clip_path_parity(capi, orc):
    """a textured ground plane through the camera, alpha tested: every triangle on screen takes the clip path (uv carried
    through the cuts) and the coarse version's two triangles are far above the whole-warp threshold"""
    from tests.test_oracle_alpha import checker, material, textured_ground

    for cells in (1, 24):
        sc = textured_ground(cells, width=640, height=360)
        sc.mesh_instances["material_index"] = 0
        hs = orc.HostScene(sc)
        cam = sc.camera()
        w, h = sc.width, sc.height
        tex = checker(4, 1, rgba=False)
        mats = np.array([material(image=0, cutoff=0.5)], dtype=abi.MATERIAL_DT)
        tab = orc.MaterialTable(mats, [(tex, abi.IMAGE_R8_UNORM)])
        mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
        visible, cmd = orc.cull_meshlets(hs, mi, vis, cam)
        visible = visible[: int(cmd["x"][0])]
        ref = orc.clear_visbuffer(w, h)
        ntri, nalpha = orc.raster_alpha(hs, mi, visible, 0, len(visible), cam, ref, tab)
        assert nalpha == ntri > 0
        plain = orc.clear_visbuffer(w, h)
        orc.raster_clip(hs, mi, visible, 0, len(visible), cam, plain)
        assert 0 < ((ref & 0xFFFFFFFF) != 0xFFFFFFFF).sum() < ((plain & 0xFFFFFFFF) != 0xFFFFFFFF).sum()
        ctx = make_ctx(capi, sc)
        tex_dev = ctx.alloc(tex.size)
        ctx.upload(tex_dev, tex)
        ctx.set_materials(mats, [(tex_dev, 4, 4, abi.IMAGE_R8_UNORM)])
        vis_dev = ctx.alloc(w * h * 8)
        ctx.clear_visbuffer(vis_dev, w, h)
        ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
        ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, False)
        ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis_dev)
        got = ctx.download(vis_dev, np.uint64, w * h).reshape(h, w)
        np.testing.assert_array_equal(got, ref)
        assert ctx.raster_triangle_count() == ntri
        assert ctx.check_status() == 0
        with pytest.raises(capi.OxcError):  # a material that names an image outside the table is refused
            ctx.set_materials(np.array([material(image=3)], dtype=abi.MATERIAL_DT), [(tex_dev, 4, 4, abi.IMAGE_R8_UNORM)])
        ctx.free(vis_dev)
        ctx.free(tex_dev)
        ctx.close()


def test_plain_c_host_runs(capi, tmp_path):
    """examples/host_min.c on the GPU: the quad covers exactly a quarter of the 64x48 image"""
    from tests.test_abi_cpu import _build_host_min
    import subprocess

    res = subprocess.run([_build_host_min(tmp_path)], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "768 of 3072 pixels" in res.stdout


# ---- alpha-tested discard: mip chains, golden fixture, random triangles, overdraw counter, clip-pass interaction, plain-C host
#      (DESIGN.md §4.3); also run on the SIMT-emulated library (plain, ASan, UBSan builds) ----


def test_alpha_discard_mipmapped_parity(capi, orc):
    """images with mip chains: the level comes from the quad differences of the interpolated uv (SampleGrad, visbuffer_encode.slang:
    57-60).  (1) two-pass frames on the synthetic scene — RGBA8 checker with a box-filtered chain (trilinear), R8 noise chain with
    nearest mipmap mode, a single-level gradient with mag = nearest / min = linear; (2) the textured ground plane through the
    camera with a chain of constant levels: the level bands towards the horizon, across clipped screen-filling triangles.  All
    bit-identical to the oracle."""
    from tests.test_oracle_alpha import checker, material, textured_ground

    rng = np.random.default_rng(9)
    images = [(orc.mip_chain(checker(32, 4)), abi.IMAGE_RGBA8_UNORM), (orc.mip_chain(rng.integers(0, 256, (16, 16), dtype=np.uint8)), abi.IMAGE_R8_UNORM),
              (np.ascontiguousarray(np.tile(np.linspace(0, 255, 16).astype(np.uint8), (16, 1))), abi.IMAGE_R8_UNORM)]
    mats = np.array([material(), material(image=0, cutoff=0.5), material(image=1, cutoff=0.45, sampler=1), material(image=2, cutoff=0.5, sampler=2)],
                    dtype=abi.MATERIAL_DT)
    smp = np.array([abi.sampler(), abi.sampler(mip=abi.MIPMAP_NEAREST, u=abi.ADDRESS_MIRRORED_REPEAT, v=abi.ADDRESS_CLAMP_TO_EDGE),
                    abi.sampler(mag=abi.FILTER_NEAREST, min=abi.FILTER_LINEAR)], dtype=abi.SAMPLER_DT)
    tab = orc.MaterialTable(mats, images, smp)
    flat = orc.MaterialTable(mats, [(images[0][0][0], images[0][1]), (images[1][0][0], images[1][1]), images[2]], smp)  # level 0 only
    sc = synth.make_scene(config_index=2, **SCENES["small"])
    sc.mesh_instances["material_index"] = np.arange(sc.mesh_instance_count) % 4
    # spread the texture coordinates so that minification occurs: scale every instance's uv range by drawing closer / farther is
    # the scene's business; here the chain is simply short enough (32 / 16 texels) for the small on-screen meshlets to minify
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc)
    dev, ptrs = tab.device_images(ctx)
    ctx.set_materials(mats, dev, smp)
    w, h = sc.width, sc.height
    vis_dev = ctx.alloc(w * h * 8)
    occ_dev = ctx.alloc(w * h * 4)
    ctx.upload(occ_dev, sc.occluder_depth)
    mask_ref = np.zeros(ctx.out.visibility_mask_words, dtype=np.uint32)
    mask_flat = np.zeros_like(mask_ref)
    lod_matters = False
    for f in range(2):
        cam = sc.camera(2.0 * f)
        ref = orc.frame(hs, cam, w, h, mask_ref, sc.occluder_depth, materials=tab)
        lod_matters = lod_matters or not np.array_equal(ref["vis64"], orc.frame(orc.HostScene(sc), cam, w, h, mask_flat, sc.occluder_depth, materials=flat)["vis64"])
        got = _frame_gpu(capi, ctx, sc, cam, occ_dev, vis_dev)
        assert (got["early"], got["late"]) == (ref["early"], ref["late"]), f"frame {f}"
        np.testing.assert_array_equal(got["mask"], mask_ref)
        np.testing.assert_array_equal(got["vis64"], ref["vis64"])
        assert got["ntri"] == ref["ntri_early"] + ref["ntri_late"]
        assert ctx.check_status() == 0
    assert lod_matters  # the chains are read: the level-0-only table gives another image
    for d in ptrs + [vis_dev, occ_dev]:
        ctx.free(d)
    ctx.close()
    # (2) level bands on the ground plane
    n = 256
    levels = [np.full((max(1, n >> l), max(1, n >> l)), 255 if l % 2 == 0 else 0, dtype=np.uint8) for l in range(9)]
    for cells, mode in ((1, abi.MIPMAP_NEAREST), (24, abi.MIPMAP_LINEAR)):
        sc = textured_ground(cells, width=640, height=360)
        sc.mesh_instances["material_index"] = 0
        hs = orc.HostScene(sc)
        cam = sc.camera()
        w, h = sc.width, sc.height
        mats = np.array([material(image=0, cutoff=0.5)], dtype=abi.MATERIAL_DT)
        smp = np.array([abi.sampler(mip=mode)], dtype=abi.SAMPLER_DT)
        tab = orc.MaterialTable(mats, [(levels, abi.IMAGE_R8_UNORM)], smp)
        mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
        visible, cmd = orc.cull_meshlets(hs, mi, vis, cam)
        visible = visible[: int(cmd["x"][0])]
        ref = orc.clear_visbuffer(w, h)
        ntri, nalpha = orc.raster_alpha(hs, mi, visible, 0, len(visible), cam, ref, tab)
        assert nalpha == ntri > 0
        ctx = make_ctx(capi, sc)
        dev, ptrs = tab.device_images(ctx)
        ctx.set_materials(mats, dev, smp)
        vis_dev = ctx.alloc(w * h * 8)
        ctx.clear_visbuffer(vis_dev, w, h)
        ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
        ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, False)
        ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis_dev)
        got = ctx.download(vis_dev, np.uint64, w * h).reshape(h, w)
        np.testing.assert_array_equal(got, ref)
        kept = ((ref & 0xFFFFFFFF) != 0xFFFFFFFF)
        assert 0.05 * kept.size < kept.sum() < 0.45 * kept.size
        with pytest.raises(capi.OxcError):  # more levels than the image can have
            ctx.set_materials(mats, [(dev[0][0], 4, 4, abi.IMAGE_R8_UNORM, 4)], smp)
        for d in ptrs + [vis_dev]:
            ctx.free(d)
        ctx.close()


def test_golden_alpha_frames(capi, orc):
    """the CUDA path against the committed fixture tests/golden/alpha_small.json (two-pass frames with a single-level and a
    mip-mapped material table; the fixture is what the oracle computes, test_oracle_alpha.py::test_golden_alpha_fixture)"""
    from tests.test_oracle_alpha import load_golden_alpha

    import os

    mg, want = load_golden_alpha()
    if os.environ.get("OXC_TEST_HOSTILE_SCENES"):  # the CPU tier's hostile pass mutates every scene: the fixture no longer applies,
        want = mg.generate()                       # the oracle on the mutated scene does
    state = {}

    def frame_fn(name, parts, sc, cam, f):
        mats, images, smp, tab = parts
        if f == 0:
            for st in state.values():
                st["ctx"].close()
            state.clear()
            ctx = make_ctx(capi, sc)
            dev, ptrs = tab.device_images(ctx)
            ctx.set_materials(mats, dev, smp)
            vis_dev, occ_dev = ctx.alloc(sc.width * sc.height * 8), ctx.alloc(sc.width * sc.height * 4)
            ctx.upload(occ_dev, sc.occluder_depth)
            state[name] = dict(ctx=ctx, vis=vis_dev, occ=occ_dev)
        st = state[name]
        got = _frame_gpu(capi, st["ctx"], sc, cam, st["occ"], st["vis"])
        assert st["ctx"].check_status() == 0
        return dict(vis64=got["vis64"], early=got["early"], late=got["late"], ntri=got["ntri"])

    got = mg.generate(frame_fn)
    for st in state.values():
        st["ctx"].close()
    assert got == want


def test_alpha_discard_random_triangles(capi, orc):
    """fuzz: meshes of random triangles around and through the camera (slivers, sub-pixel and screen-filling ones, vertices behind
    the near plane, uv from tiny to huge), random images (with / without mip chains, RGBA8 / R8), random sampler modes and cutoffs:
    the CUDA raster's image equals the oracle's bit for bit — small path, whole-warp path, clip path and level selection under
    inputs no scene generator produces.  The plain raster (no table) is checked on the same triangles first."""
    from oxylus_b200 import capi as capi_mod
    from tests.test_oracle_alpha import material

    import os

    n_seeds = int(os.environ.get("OXC_ALPHA_FUZZ_SEEDS", "6"))  # more seeds: OXC_ALPHA_FUZZ_SEEDS=400 on the emulated library
    discarding = 0
    for seed in range(n_seeds):
        rng = np.random.default_rng(100 + seed)
        n_tri = 192
        centre = np.stack([rng.uniform(-3, 3, n_tri), rng.uniform(-2, 2, n_tri), rng.uniform(-8, 0.5, n_tri)], axis=1)
        size = 10.0 ** rng.uniform(-2.5, 0.8, n_tri)
        pos = (centre[:, None, :] + rng.normal(0, 1, (n_tri, 3, 3)) * size[:, None, None]).astype(np.float32)
        sliver = rng.random(n_tri) < 0.15
        pos[sliver, 2] = pos[sliver, 1] + (pos[sliver, 2] - pos[sliver, 1]) * np.float32(1e-3)
        uv = (rng.normal(0, 1, (n_tri, 3, 2)) * (10.0 ** rng.uniform(-2, 1.5, n_tri))[:, None, None]).astype(np.float32)
        idx = np.arange(n_tri * 3, dtype=np.uint32)
        built = [capi_mod.BuiltMesh(pos.reshape(-1, 3), [(idx, 0.0)], texcoords=uv.reshape(-1, 2))]
        sc = capi_mod.assemble_scene(built, np.arange(1), np.eye(4, dtype=np.float32).reshape(1, 16), 320, 200)
        sc.mesh_instances["material_index"] = 0
        n = int(2 ** rng.integers(0, 6))
        fmt = abi.IMAGE_R8_UNORM if rng.random() < 0.5 else abi.IMAGE_RGBA8_UNORM
        tex = rng.integers(0, 256, (n, max(1, n // int(2 ** rng.integers(0, 2)))) + ((4,) if fmt == abi.IMAGE_RGBA8_UNORM else ()), dtype=np.uint8)
        img = (orc.mip_chain(tex) if seed % 2 == 0 else tex, fmt)
        smp = np.array([abi.sampler(int(rng.integers(2)), int(rng.integers(2)), int(rng.integers(2)), int(rng.integers(3)), int(rng.integers(3)))], dtype=abi.SAMPLER_DT)
        mats = np.array([material(image=0, cutoff=float(rng.uniform(0.2, 0.8)), albedo_a=float(rng.uniform(0.7, 1.0)))], dtype=abi.MATERIAL_DT)
        tab = orc.MaterialTable(mats, [img], smp)
        hs = orc.HostScene(sc)
        cam = sc.camera()
        w, h = sc.width, sc.height
        mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
        visible, cmd = orc.cull_meshlets(hs, mi, vis, cam)
        visible = visible[: int(cmd["x"][0])]
        ref = orc.clear_visbuffer(w, h)
        ntri, nalpha = orc.raster_alpha(hs, mi, visible, 0, len(visible), cam, ref, tab)
        plain = orc.clear_visbuffer(w, h)
        _, nclip = orc.raster_clip(hs, mi, visible, 0, len(visible), cam, plain)
        assert ntri > 20 and nalpha == ntri and nclip > 0, (seed, ntri, nclip)
        assert ((plain & 0xFFFFFFFF) != 0xFFFFFFFF).sum() > 200, seed
        discarding += int(not np.array_equal(ref, plain))
        ctx = make_ctx(capi, sc)
        vis_dev = ctx.alloc(w * h * 8)
        ctx.clear_visbuffer(vis_dev, w, h)
        ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
        ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, False)
        ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis_dev)  # no table yet: the plain raster on the same triangles
        np.testing.assert_array_equal(ctx.download(vis_dev, np.uint64, w * h).reshape(h, w), plain, err_msg=f"seed {seed} (plain)")
        dev, ptrs = tab.device_images(ctx)
        ctx.set_materials(mats, dev, smp)
        ctx.clear_visbuffer(vis_dev, w, h)
        ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis_dev)
        got = ctx.download(vis_dev, np.uint64, w * h).reshape(h, w)
        np.testing.assert_array_equal(got, ref, err_msg=f"seed {seed}")
        assert ctx.raster_triangle_count() == ntri and ctx.check_status() == 0
        for d in ptrs + [vis_dev]:
            ctx.free(d)
        ctx.close()
    assert discarding >= n_seeds // 2  # (a random image can lie entirely above or below the cutoff)


def test_overdraw_counter_parity(capi, orc):
    """oxc_raster_overdraw (RENDER_OVERDRAW of the encode pass, visbuffer_encode.slang:68-70): the fragment counter of both passes of
    a two-pass frame, without and with a material table, equals the oracle's counter pixel for pixel; the frame's own outputs are
    untouched by the extra launches; clipped screen-filling triangles count too"""
    from tests.test_oracle_alpha import checker, material, textured_ground

    sc = synth.make_scene(config_index=2, **SCENES["small"])
    sc.mesh_instances["material_index"] = np.arange(sc.mesh_instance_count) % 4
    w, h = sc.width, sc.height
    for with_table in (False, True):
        hs = orc.HostScene(sc)
        ctx = make_ctx(capi, sc)
        tab, ptrs = _alpha_tables(capi, orc, ctx) if with_table else (None, [])
        vis_dev, occ_dev, over_dev = ctx.alloc(w * h * 8), ctx.alloc(w * h * 4), ctx.alloc(w * h * 4)
        ctx.upload(occ_dev, sc.occluder_depth)
        mask_ref = np.zeros(ctx.out.visibility_mask_words, dtype=np.uint32)
        for f in range(2):
            cam = sc.camera(2.0 * f)
            ref = orc.frame(hs, cam, w, h, mask_ref, sc.occluder_depth, materials=tab)
            e, l = ref["early"], ref["late"]
            want = np.zeros((h, w), dtype=np.uint32)
            orc.raster_overdraw(hs, ref["meshlet_instances"], ref["visible"], 0, e, cam, want, tab)
            orc.raster_overdraw(hs, ref["meshlet_instances"], ref["visible"], e, l, cam, want, tab)
            # the frame, with the counter launched after each raster
            ctx.clear_visbuffer(vis_dev, w, h)
            ctx.clear_overdraw(over_dev, w, h)
            ctx.clear_hiz()
            ctx.merge_depth(vis_dev, occ_dev, w, h)
            ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
            ctx.cull_meshlets(cam, abi.CULL_TEST_ALL, True)
            ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis_dev)
            ctx.raster_overdraw(cam, abi.CULL_TEST_ALL, w, h, over_dev)
            ctx.build_hiz_packed(vis_dev, w, h)
            ctx.cull_meshlets(cam, abi.CULL_TEST_ALL | abi.CULL_LATE_PASS, True)
            ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL | abi.CULL_LATE_PASS, w, h, vis_dev)
            ctx.raster_overdraw(cam, abi.CULL_TEST_ALL | abi.CULL_LATE_PASS, w, h, over_dev)
            np.testing.assert_array_equal(ctx.download(over_dev, np.uint32, w * h).reshape(h, w), want, err_msg=f"table {with_table} frame {f}")
            # the same counter issued after the frame (the dispatch command now holds the late count: ranges from the visibility record)
            ctx.clear_overdraw(over_dev, w, h)
            ctx.raster_overdraw(cam, abi.CULL_TEST_ALL, w, h, over_dev, after_frame=True)
            ctx.raster_overdraw(cam, abi.CULL_TEST_ALL | abi.CULL_LATE_PASS, w, h, over_dev, after_frame=True)
            np.testing.assert_array_equal(ctx.download(over_dev, np.uint32, w * h).reshape(h, w), want, err_msg=f"after frame, table {with_table} frame {f}")
            np.testing.assert_array_equal(ctx.download(vis_dev, np.uint64, w * h).reshape(h, w), ref["vis64"])
            np.testing.assert_array_equal(ctx.mask(), mask_ref)
            assert ctx.raster_triangle_count() == ref["ntri_early"] + ref["ntri_late"] and ctx.check_status() == 0
            assert want.max() >= 2 and (want > 0).sum() >= ((ref["vis64"] & 0xFFFFFFFF) != 0xFFFFFFFF).sum()
        for d in ptrs + [vis_dev, occ_dev, over_dev]:
            ctx.free(d)
        ctx.close()
    # the host mirror: oxr_overdraw after a rendered frame == the oracle's counter over that frame's two passes
    sc = synth.make_scene(config_index=2, **SCENES["small"])
    hs = orc.HostScene(sc)
    r = capi.Renderer(0, sc)
    mask_ref = np.zeros((sc.max_meshlet_instance_count + 31) // 32, dtype=np.uint32)
    for f in range(2):
        cam = sc.camera(3.0 * f)
        ref = orc.frame(hs, cam, sc.width, sc.height, mask_ref, sc.occluder_depth)
        got = r.render(cam, sc.occluder_depth)
        assert (got["early"], got["late"]) == (ref["early"], ref["late"])
        want = np.zeros((sc.height, sc.width), dtype=np.uint32)
        orc.raster_overdraw(hs, ref["meshlet_instances"], ref["visible"], 0, ref["early"], cam, want)
        orc.raster_overdraw(hs, ref["meshlet_instances"], ref["visible"], ref["early"], ref["late"], cam, want)
        np.testing.assert_array_equal(r.overdraw(cam), want)
    r.close()
    # clipped, screen-filling triangles (whole-warp path) with a checker material
    sc = textured_ground(1, width=640, height=360)
    sc.mesh_instances["material_index"] = 0
    hs = orc.HostScene(sc)
    cam = sc.camera()
    w, h = sc.width, sc.height
    tex = checker(4, 1, rgba=False)
    mats = np.array([material(image=0, cutoff=0.5)], dtype=abi.MATERIAL_DT)
    tab = orc.MaterialTable(mats, [(tex, abi.IMAGE_R8_UNORM)])
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    visible, cmd = orc.cull_meshlets(hs, mi, vis, cam)
    visible = visible[: int(cmd["x"][0])]
    want = np.zeros((h, w), dtype=np.uint32)
    orc.raster_overdraw(hs, mi, visible, 0, len(visible), cam, want, tab)
    assert 0.05 * want.size < (want > 0).sum() < 0.45 * want.size
    ctx = make_ctx(capi, sc)
    dev, ptrs = tab.device_images(ctx)
    ctx.set_materials(mats, dev)
    over_dev = ctx.alloc(w * h * 4)
    ctx.clear_overdraw(over_dev, w, h)
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, False)
    ctx.raster_overdraw(cam, abi.CULL_TEST_ALL, w, h, over_dev)
    np.testing.assert_array_equal(ctx.download(over_dev, np.uint32, w * h).reshape(h, w), want)
    for d in ptrs + [over_dev]:
        ctx.free(d)
    ctx.close()


def test_alpha_clip_pass_leaves_alpha_meshlets_alone(capi, orc):
    """the stand-alone clip pass after a raster with a material table: alpha-tested meshlets were clipped (with the test) by the
    raster itself, so the pass must not draw their clipped triangles again without the test"""
    from tests.test_oracle_alpha import checker, material, textured_ground

    sc = textured_ground(1, width=640, height=360)
    sc.mesh_instances["material_index"] = 0
    hs = orc.HostScene(sc)
    cam = sc.camera()
    w, h = sc.width, sc.height
    tex = checker(4, 1, rgba=False)
    mats = np.array([material(image=0, cutoff=0.5)], dtype=abi.MATERIAL_DT)
    tab = orc.MaterialTable(mats, [(tex, abi.IMAGE_R8_UNORM)])
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    visible, cmd = orc.cull_meshlets(hs, mi, vis, cam)
    visible = visible[: int(cmd["x"][0])]
    ref = orc.clear_visbuffer(w, h)
    orc.raster_alpha(hs, mi, visible, 0, len(visible), cam, ref, tab)
    ctx = make_ctx(capi, sc)
    dev, ptrs = tab.device_images(ctx)
    ctx.set_materials(mats, dev)
    vis_dev = ctx.alloc(w * h * 8)
    ctx.clear_visbuffer(vis_dev, w, h)
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, False)
    ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis_dev)
    ctx.raster_visbuffer_clip_pass(cam, abi.CULL_TEST_ALL, w, h, vis_dev)
    np.testing.assert_array_equal(ctx.download(vis_dev, np.uint64, w * h).reshape(h, w), ref)
    for d in ptrs + [vis_dev]:
        ctx.free(d)
    ctx.close()


def test_plain_c_host_alpha_runs(capi, tmp_path):
    """examples/host_min.c alpha: oxc_set_materials from plain C — the 2x2 checker material discards two quadrants of the quad (the same
    binary linked with the emulated library prints the same in the CPU tier)"""
    from tests.test_abi_cpu import _build_host_min
    import subprocess

    res = subprocess.run([_build_host_min(tmp_path), "alpha"], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "alpha-tested: 384 of 768 quad pixels kept, 0 pixels differ" in res.stdout
