"""The VSM shadow raster on the device (oxc_vsm_draw_pages, oxr_vsm_draw_shadows) against the CPU oracle
(oracle/oxc_oracle_vsm_draw.c orc_vsm_draw_pages), the physical atlas compared bit for bit in every case."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_vsm_pages import LIGHT, Dev, _sequence_frames, clipmaps, physical_count, vsm_context

pytestmark = pytest.mark.gpu

B, D, V = abi.VSM_PAGE_BACKED, abi.VSM_PAGE_DIRTY, abi.VSM_PAGE_VISIBLE
CENTER = (6.0, -2.0, -115.0)  # middle of the synthetic scenes' instances: the fine clipmaps see casters


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def vd():
    """the shadow-raster oracle (oracle/pyoracle_vsm_draw.py)"""
    import pyoracle_vsm_draw

    pyoracle_vsm_draw.build()
    return pyoracle_vsm_draw


@pytest.fixture(scope="module")
def scene():
    return synth.make_scene(3000, config_index=2, width=640, height=360, n_unique_meshes=8)


@pytest.fixture(scope="module")
def ctx(capi, scene):
    hw, hh = scene.hiz_extent()
    c = capi.Context(0, scene.mesh_instance_count, scene.max_meshlet_instance_count, hw, hh, max_views=10)
    c.set_scene(scene)
    yield c
    c.close()


def coarse_camera(n_instances, center=(0.0, 0.0, -60.0)):
    """clipmap 9's view as the coarse camera (Shadowmaps.cpp:433-463): position = -light direction"""
    cam = synth.make_ortho_view(LIGHT, center, 10.0 * 2 ** 9, 2000.0, n_instances)
    cam["position"][0] = -np.asarray(LIGHT) / np.linalg.norm(LIGHT)
    return cam


def dirty_table(rng, vsm, density):
    """random states in which Backed && Dirty does not imply Visible, about `density` of the entries Backed && Dirty, physical
    addresses anywhere in the atlas (and a few beyond it)"""
    layers, size, p = int(vsm["clipmap_count"][0]), int(vsm["page_table_size"][0]), physical_count(vsm)
    shape = (layers, size, size)
    state = rng.integers(0, 32, size=shape).astype(np.uint32) & ~np.uint32(B | D)
    bd = rng.random(shape) < density
    state[bd] |= B | D
    other = ~bd & (rng.random(shape) < 0.3)
    state[other] |= rng.choice([B, D], int(other.sum())).astype(np.uint32)
    phys = rng.integers(0, p + p // 16, size=shape).astype(np.uint32)
    return (state | (phys << 16)).astype(np.uint32)


def start_atlas(rng, P):
    """1.0 (a cleared page) almost everywhere, random depths below it in a few rows"""
    a = np.ones((P, P), dtype=np.float32)
    rows = rng.choice(P, max(1, P // 16), replace=False)
    a[rows] = rng.random((len(rows), P)).astype(np.float32)
    return a


def draw_case(ctx, orc, vd, scene, vsm, cm, pt, flags, atlas, coarse, materials=None, hpb_all=True):
    """device: cull_meshes + HPB cull on device flags (an all-ones HPB: every caster in a dirty clipmap's frustum survives) + draw;
    oracle: the same three.  Returns (device atlas as u32, oracle atlas as u32, fragments the oracle wrote, draw stats)"""
    hs = orc.HostScene(scene)
    layers, size = int(vsm["clipmap_count"][0]), int(vsm["page_table_size"][0])
    levels = int(np.log2(size)) + 1 if size & (size - 1) == 0 else 1
    hpb = np.ones(orc.hpb_layout(size, layers, levels)[1], dtype=np.uint8)
    mi, vis, _ = orc.cull_meshes(hs, coarse, abi.CULL_TEST_ALL)
    ref, _ = orc.cull_meshlets_hpb(hs, mi, vis, coarse, cm, flags, hpb, size, levels)
    want = atlas.copy()
    written = vd.vsm_draw_pages(hs, mi, ref, coarse, vsm, cm, flags, pt, want, materials)
    d = Dev(ctx)
    d_pt, d_flags, d_atlas, d_hpb = d.put(pt), d.put(np.uint32(flags)), d.put(atlas), d.put(hpb)
    ctx.cull_meshes(coarse, abi.CULL_TEST_ALL)
    ctx.cull_meshlets_hpb_dirty_dev(coarse, cm, d_flags, d_hpb, size, levels)
    n = int(ctx.cull_triangles_cmd()["x"][0])
    np.testing.assert_array_equal(np.sort(ctx.visible_indices(n)), np.sort(ref))
    ctx.vsm_draw_pages(vsm, coarse, cm, d_flags, d_pt, d_atlas)
    got = d.get(d_atlas, atlas).view(np.uint32)
    stats = ctx.vsm_draw_stats()
    d.free()
    return got, want.view(np.uint32), written, stats


@pytest.mark.parametrize("which", ["one", "all", "none"])
def test_random_tables(ctx, orc, vd, scene, which):
    """random tables (Backed && Dirty independent of Visible, addresses beyond the atlas included), one dirty clipmap, all ten, or
    none (the atlas is untouched)"""
    rng = np.random.default_rng({"one": 1, "all": 2, "none": 3}[which])
    vsm = vsm_context(size=64, page_size=32, physical=2048)
    cm = clipmaps(10, rng, center=CENTER)
    flags = {"one": [0] * 10, "all": [1] * 10, "none": [0] * 10}[which]
    if which == "one":
        flags[1] = 1
    pt = dirty_table(rng, vsm, 0.5)
    atlas = start_atlas(rng, 2048)
    got, want, written, stats = draw_case(ctx, orc, vd, scene, vsm, cm, pt, flags, atlas, coarse_camera(scene.mesh_instance_count))
    np.testing.assert_array_equal(got, want)
    if which == "none":
        assert written == 0 and (got == atlas.view(np.uint32)).all() and stats["items"] == 0
    else:
        assert written > 1000 and (got != atlas.view(np.uint32)).sum() > 500 and stats["items"] > 0
    print(which, "fragments", written, stats)


def test_clip_path_in_the_finest_clipmap(ctx, orc, vd, scene):
    """clipmaps of half-size 0.25, 1 and 4 around a caster with a 4096^2 target: its vertices are tens of thousands of pixels outside
    the viewport and take the clipper; every page of those three clipmaps dirty"""
    rng = np.random.default_rng(4)
    vsm = vsm_context(size=64, page_size=64, physical=4096)
    center = tuple(float(x) for x in scene.transforms["world"][int(scene.mesh_instances["transform_index"][0]), 12:15])
    cm = np.zeros(10, dtype=abi.CLIPMAP_DT)
    for k in range(10):
        v = synth.make_ortho_view(LIGHT, center, 0.25 * (4 ** k), 2000.0, 1)
        cm["projection_view_mat"][k] = v["projection_view"][0]
    cm["page_offset"] = rng.integers(-70, 70, size=(10, 2))
    pt = np.zeros((10, 64, 64), dtype=np.uint32)
    pt[:3] = (B | D) | (rng.integers(0, 4096, size=(3, 64, 64)).astype(np.uint32) << 16)
    flags = [1, 1, 1] + [0] * 7
    atlas = np.ones((4096, 4096), dtype=np.float32)
    got, want, written, stats = draw_case(ctx, orc, vd, scene, vsm, cm, pt, flags, atlas, coarse_camera(scene.mesh_instance_count, center))
    np.testing.assert_array_equal(got, want)
    assert written > 100000, written
    print("clip path: fragments", written, stats)


@pytest.mark.parametrize("capacity", [7, 5000])
def test_queue_overflow_drawn_inline(capi, orc, vd, capacity):
    """OXC_VSM_DRAW_CAPACITY: a work queue of 7 or 5000 items under a tessellated ground caster with half the pages of two clipmaps
    dirty — more items than the queue holds, so most are drawn inline by the lane that found them (reservations straddle the
    capacity in the second case); the atlas still equals the oracle bit for bit"""
    import os

    sc = synth.with_ground_caster(synth.make_scene(600, config_index=2, width=640, height=360, n_unique_meshes=8), center=CENTER, grid=8)
    hw, hh = sc.hiz_extent()
    os.environ["OXC_VSM_DRAW_CAPACITY"] = str(capacity)
    try:
        c = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh, max_views=10)
    finally:
        os.environ.pop("OXC_VSM_DRAW_CAPACITY", None)
    c.set_scene(sc)
    rng = np.random.default_rng(capacity)
    vsm = vsm_context(size=64, page_size=32, physical=2048)
    cm = clipmaps(10, rng, center=CENTER)
    pt = dirty_table(rng, vsm, 0.5)
    flags = [0, 0, 1, 0, 1, 0, 0, 0, 0, 0]
    atlas = start_atlas(rng, 2048)
    got, want, written, stats = draw_case(c, orc, vd, sc, vsm, cm, pt, flags, atlas, coarse_camera(sc.mesh_instance_count, CENTER))
    np.testing.assert_array_equal(got, want)
    assert stats["items"] > 2 * capacity and written > 100000, (stats, written)
    print("capacity", capacity, "fragments", written, stats)
    c.close()


def checker_materials(orc):
    """material 0 opaque, material 1 an RGBA8 checker (linear + repeat) with cutoff 0.5 (tests/test_oracle_alpha.py helpers)"""
    from tests.test_oracle_alpha import checker, material

    mats = np.array([material(), material(image=0, cutoff=0.5)], dtype=abi.MATERIAL_DT)
    smp = np.array([abi.sampler()], dtype=abi.SAMPLER_DT)
    return orc.MaterialTable(mats, [(checker(16, 2), abi.IMAGE_RGBA8_UNORM)], smp)


def test_alpha_tested_casters(capi, orc, vd):
    """a material table with every other instance alpha tested: the discarded samples are not written, on the device as in the
    oracle (uv through the clipper included)"""
    sc = synth.make_scene(1500, config_index=2, width=640, height=360, n_unique_meshes=8)
    sc.mesh_instances["material_index"] = np.arange(sc.mesh_instance_count) % 2
    hw, hh = sc.hiz_extent()
    c = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh, max_views=10)
    c.set_scene(sc)
    table = checker_materials(orc)
    images, ptrs = table.device_images(c)
    c.set_materials(table.materials, images, table.samplers)
    rng = np.random.default_rng(5)
    vsm = vsm_context(size=64, page_size=32, physical=2048)
    cm = clipmaps(10, rng, center=CENTER)
    pt = dirty_table(rng, vsm, 0.5)
    flags = [1] * 10
    atlas = np.ones((2048, 2048), dtype=np.float32)
    got, want, written, _ = draw_case(c, orc, vd, sc, vsm, cm, pt, flags, atlas, coarse_camera(sc.mesh_instance_count), materials=table)
    np.testing.assert_array_equal(got, want)
    opaque = atlas.copy()
    vd.vsm_draw_pages(orc.HostScene(sc), *_survivors(orc, sc, vsm, cm, flags), vsm, cm, flags, pt, opaque, None)
    assert (opaque.view(np.uint32) != want).sum() > 20  # the test discarded samples
    for p in ptrs:
        c.free(p)
    c.close()


def _survivors(orc, sc, vsm, cm, flags):
    hs = orc.HostScene(sc)
    coarse = coarse_camera(sc.mesh_instance_count)
    layers, size = int(vsm["clipmap_count"][0]), int(vsm["page_table_size"][0])
    levels = int(np.log2(size)) + 1
    mi, vis, _ = orc.cull_meshes(hs, coarse, abi.CULL_TEST_ALL)
    ref, _ = orc.cull_meshlets_hpb(hs, mi, vis, coarse, cm, flags, np.ones(orc.hpb_layout(size, layers, levels)[1], np.uint8), size, levels)
    return mi, ref, coarse


def test_atlas_shape_not_reference(ctx, orc, vd, scene):
    """24 x 24 pages per clipmap, 3 clipmaps, 16-texel pages in a 400^2 atlas: 16.67 pixels per virtual page, page boundaries fall
    between pixel centres at uneven places"""
    rng = np.random.default_rng(6)
    vsm = vsm_context(size=24, layers=3, page_size=16, physical=400)
    cm = clipmaps(3, rng, center=CENTER)
    pt = dirty_table(rng, vsm, 0.5)
    flags = [1, 0, 1]
    atlas = start_atlas(rng, 400)
    got, want, written, _ = draw_case(ctx, orc, vd, scene, vsm, cm, pt, flags, atlas, coarse_camera(scene.mesh_instance_count))
    np.testing.assert_array_equal(got, want)
    assert written > 100


def test_argument_refusals(capi, ctx, scene):
    vsm = vsm_context()
    d = Dev(ctx)
    buf = d.put(np.zeros(1 << 16, np.uint32))
    cam = coarse_camera(scene.mesh_instance_count)

    def refused(fn, match, code="(-1)"):
        with pytest.raises(capi.OxcError, match=match) as e:
            fn()
        assert code in str(e.value)

    def bad(**kw):
        v = vsm.copy()
        for k, x in kw.items():
            v[k] = x
        return v

    for v, match in ((bad(clipmap_count=0), "clipmap_count"), (bad(clipmap_count=11), "clipmap_count"), (bad(page_size=100), "does not divide"),
                     (bad(page_size=16), "65536"), (bad(page_table_size=0), "page_table_size"),
                     (bad(physical_page_table_size=32768, page_size=512), "snap range")):
        refused(lambda: ctx.vsm_draw_pages(v, cam, clipmaps(10), buf, buf, buf), match)
    refused(lambda: ctx.vsm_draw_pages(vsm, cam, clipmaps(10), None, buf, buf), "null")
    refused(lambda: ctx.vsm_draw_pages(vsm, cam, clipmaps(10), buf, None, buf), "null")
    refused(lambda: ctx.vsm_draw_pages(vsm, cam, clipmaps(10), buf, buf, None), "null")
    refused(lambda: ctx.vsm_draw_pages(vsm, None, clipmaps(10), buf, buf, buf), "null")
    hw, hh = scene.hiz_extent()
    empty = capi.Context(0, scene.mesh_instance_count, scene.max_meshlet_instance_count, hw, hh, max_views=10)
    refused(lambda: empty.vsm_draw_pages(vsm, cam, clipmaps(10), buf, buf, buf), "oxc_set_scene", "(-5)")
    empty.close()
    d.free()


def test_graph_capture_equals_eager(capi, ctx, scene):
    """page update + shadow cull + draw captured into one CUDA graph and replayed twice (a new depth image before the second replay)
    equals the same calls run eagerly, atlas and page table for both frames"""
    import torch
    from tests.test_oracle_units import make_vsm_case

    inv_pv, res, cm6, vsm, depth0, _ = make_vsm_case(640, 360, size=64, clipmaps=6)
    vsm["page_size"], vsm["physical_page_table_size"] = 64, 4096
    cm = clipmaps(6, np.random.default_rng(8))
    cm["page_offset"] = cm6["page_offset"]
    for k in range(6):
        cm6["projection_view_mat"][k] = cm["projection_view_mat"][k]
    depth1 = np.roll(depth0, 37, axis=1)
    p = physical_count(vsm)
    entries = 6 * 64 * 64
    coarse = coarse_camera(scene.mesh_instance_count)

    def buffers():
        d = Dev(ctx)
        b = dict(depth=d.put(depth0), pt=d.put(np.zeros(entries, np.uint32)), occ=d.put(np.zeros(p, np.uint32)), req=d.put(np.zeros((entries, 3), np.int32)),
                 al=d.put(np.zeros(1, abi.VSM_ALLOCATOR_DT)), fl=d.put(np.zeros(p, np.uint32)), coords=d.put(np.zeros((entries, 2), np.uint32)),
                 flags=d.put(np.zeros(6, np.uint32)), hpb=d.put(np.zeros(6 * sum(max(1, 64 >> l) ** 2 for l in range(7)), np.uint8)),
                 atlas=d.put(np.zeros((4096, 4096), np.float32)))
        return d, b

    def enqueue(c, b):
        c.vsm_begin_frame(vsm, False, b["pt"], b["occ"], p, b["al"])
        c.mark_visible_pages(inv_pv, res, cm6, vsm, b["depth"], b["pt"], b["occ"], b["al"], b["req"], entries)
        c.vsm_allocate_pages(vsm, b["pt"], b["occ"], p, b["req"], entries, b["al"], b["fl"], b["coords"], b["flags"])
        c.build_hpb(b["pt"], 64, 6, b["hpb"], 7)
        c.vsm_clear_dirty_pages(vsm, b["al"], b["coords"], b["atlas"])
        c.cull_meshes(coarse, abi.CULL_TEST_ALL)
        c.cull_meshlets_hpb_dirty_dev(coarse, cm6, b["flags"], b["hpb"], 64, 7)
        c.vsm_draw_pages(vsm, coarse, cm6, b["flags"], b["pt"], b["atlas"])

    def snapshot(b):
        return [ctx.download(b["pt"], np.uint32, entries), ctx.download(b["atlas"], np.uint32, 4096 * 4096)]

    de, be = buffers()
    eager = []
    for dep in (depth0, depth1):
        ctx.upload(be["depth"], dep)
        enqueue(ctx, be)
        eager.append(snapshot(be))
    dg, bg = buffers()
    s = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
        enqueue(gctx, bg)
    for k, dep in enumerate((depth0, depth1)):
        ctx.upload(bg["depth"], dep)
        g.replay()
        torch.cuda.synchronize()
        for a, b_ in zip(snapshot(bg), eager[k]):
            np.testing.assert_array_equal(a, b_)
    drawn = eager[0][1]
    assert ((drawn != 0x3F800000) & (drawn != 0)).sum() > 1000  # the draw wrote depth below the clear value
    del g
    de.free()
    dg.free()


def test_sequence_through_renderer_full_size(capi, orc, vd):
    """the eight frames of test_vsm_sequence_through_renderer_full_size (64 x 64 pages x 10 clipmaps, 8192^2 atlas, camera moving,
    offsets scrolling, sun_moved at frame 3, instances moved at frames 5-6) with oxr_vsm_draw_shadows after every update: the atlas
    equals the oracle's after every frame, accumulated across frames (clean pages keep last frame's depth, re-dirtied pages are
    cleared and redrawn)"""
    import pyoracle_vsm

    sc = synth.make_scene(20000, config_index=2, width=1920, height=1080, n_unique_meshes=32)
    hs = orc.HostScene(sc)
    hs.transforms = hs.transforms.copy()
    hs.desc.transforms = hs.transforms.ctypes.data
    r = capi.Renderer(0, sc)
    vsm = vsm_context()
    st = pyoracle_vsm.VsmState(vsm, 7)
    atlas = np.zeros((8192, 8192), dtype=np.float32)  # the renderer's atlas starts zeroed
    prev = hs.transforms.copy()
    coarse = coarse_camera(sc.mesh_instance_count)
    drawn_total = 0
    for f, fr in enumerate(_sequence_frames(sc)):
        if len(fr["movers"]):
            prev = hs.transforms.copy()
            for i in fr["movers"]:
                ti = int(sc.mesh_instances["transform_index"][i])
                hs.transforms["world"][ti, 12:15] += np.float32([3.0, 0.0, -2.0])
                r.update_transforms(np.ascontiguousarray(hs.transforms[ti: ti + 1]), first=ti)
        cam = sc.camera(fr["yaw"])
        out = r.render(cam, want_indices=False)
        inv_pv = np.linalg.inv(cam["projection_view"][0].reshape(4, 4).T.astype(np.float64)).T.astype(np.float32).reshape(16)
        res = cam["resolution"][0]
        pg = r.vsm_update_pages(vsm, fr["clip"], inv_pv, res, sun_moved=fr["sun_moved"], dirty_mesh_instances=fr["movers"], hpb_levels=7)
        r.vsm_draw_shadows(coarse)
        st.frame(fr["clip"], fr["sun_moved"], hs, fr["movers"], prev, inv_pv, res, out["depth"], atlas)
        mi, vis, _ = orc.cull_meshes(hs, coarse, abi.CULL_TEST_ALL)
        ref, _ = orc.cull_meshlets_hpb(hs, mi, vis, coarse, fr["clip"], st.dirty_flags, st.hpb, 64, 7)
        drawn = vd.vsm_draw_pages(hs, mi, ref, coarse, vsm, fr["clip"], st.dirty_flags, st.page_tables, atlas)
        got = r.ctx.download(pg.physical_atlas, np.uint32, 8192 * 8192).reshape(8192, 8192)
        np.testing.assert_array_equal(got, atlas.view(np.uint32), err_msg=f"frame {f}")
        drawn_total += drawn
        print(f"frame {f}: dirty pages {len(st.dirty())}, survivors {len(ref)}, fragments {drawn}")
    assert drawn_total > 100000
    r.close()


def test_next_camera_frame_unchanged(capi):
    """oxr_render and oxr_submit after oxr_vsm_draw_shadows give bit for bit what they give without it, and oxr_overdraw still sees
    the last frame"""
    sc = synth.make_scene(4000, config_index=2, width=640, height=360, n_unique_meshes=8)
    vsm = vsm_context(width=640, height=360)
    coarse = coarse_camera(sc.mesh_instance_count)
    outs = []
    for draw in (False, True):
        r = capi.Renderer(0, sc)
        o = []
        for f, fr in enumerate(_sequence_frames(sc, 3)):
            cam = sc.camera(fr["yaw"])
            out = r.render(cam)
            inv_pv = np.linalg.inv(cam["projection_view"][0].reshape(4, 4).T.astype(np.float64)).T.astype(np.float32).reshape(16)
            r.vsm_update_pages(vsm, fr["clip"], inv_pv, cam["resolution"][0], sun_moved=fr["sun_moved"], hpb_levels=7)
            if draw:
                r.vsm_draw_shadows(coarse)
            o.append((out["vis32"].copy(), out["depth"].copy(), np.sort(out["visible"]), r.overdraw(cam)))  # list order: atomics
        bufs = dict(vis32=np.empty((360, 640), np.uint32), depth=np.empty((360, 640), np.float32), idx=np.empty(max(1, sc.max_meshlet_instance_count), np.uint32))
        for yaw in (7.0, 9.0):
            t = r.submit(sc.camera(yaw), bufs)
            res = r.wait(t)
            o.append((bufs["vis32"].copy(), bufs["depth"].copy(), np.sort(bufs["idx"][: res["early"] + res["late"]]), None))
            if draw:
                r.vsm_draw_shadows(coarse)
        outs.append(o)
        r.close()
    for a, b in zip(*outs):
        for x, y in zip(a, b):
            if x is not None:
                np.testing.assert_array_equal(x, y)
