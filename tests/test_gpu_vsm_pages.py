"""VSM page bookkeeping on the device (oxc_vsm_*, oxc_cull_meshlets_hpb_dirty_dev, oxr_vsm_update_pages) against the CPU oracle
(oracle/oxc_oracle_vsm.c orc_vsm_*), bit for bit: page tables, occupancy, free list, allocator counters, dirty list and flags, the HPB,
the physical atlas and the shadow cull's survivors."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth

pytestmark = pytest.mark.gpu

V, D, B, I, F = abi.VSM_PAGE_VISIBLE, abi.VSM_PAGE_DIRTY, abi.VSM_PAGE_BACKED, abi.VSM_PAGE_INVALIDATED, abi.VSM_PAGE_ALLOCATION_FAILED
LIGHT = (0.3, -1.0, 0.2)


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def vo():
    """the VSM oracle (oracle/pyoracle_vsm.py)"""
    import pyoracle_vsm

    pyoracle_vsm.build()
    return pyoracle_vsm


@pytest.fixture(scope="module")
def scene():
    return synth.make_scene(4000, config_index=2, width=640, height=360, n_unique_meshes=8)


@pytest.fixture(scope="module")
def ctx(capi, scene):
    hw, hh = scene.hiz_extent()
    c = capi.Context(0, scene.mesh_instance_count, scene.max_meshlet_instance_count, hw, hh, max_views=10)
    c.set_scene(scene)
    yield c
    c.close()


def vsm_context(size=64, layers=10, page_size=128, physical=8192, width=1920, height=1080):
    vsm = np.zeros(1, dtype=abi.VSM_CONTEXT_DT)
    vsm["page_size"], vsm["page_table_size"], vsm["physical_page_table_size"], vsm["clipmap_count"] = page_size, size, physical, layers
    vsm["depth_extent"][0] = (width, height)
    vsm["first_clipmap_width"], vsm["clipmap_selection_bias"], vsm["virtual_extent"], vsm["z_length"] = 10.0, 0.25, float(physical), 2000.0
    vsm["directional_light_dir"][0] = LIGHT
    return vsm


def clipmaps(n, rng=None, offsets=None, center=(0.0, 0.0, -60.0)):
    cm = np.zeros(n, dtype=abi.CLIPMAP_DT)
    for k in range(n):
        v = synth.make_ortho_view(LIGHT, center, 10.0 * (2 ** k), 2000.0, 1)
        cm["projection_view_mat"][k] = v["projection_view"][0]
        cm["page_offset"][k] = offsets[k] if offsets is not None else (rng.integers(-90, 90, size=2) if rng is not None else (0, 0))
    return cm


def physical_count(vsm):
    n = int(vsm["physical_page_table_size"][0]) // int(vsm["page_size"][0])
    return n * n


def random_table(rng, vsm):
    layers, size, p = int(vsm["clipmap_count"][0]), int(vsm["page_table_size"][0]), physical_count(vsm)
    shape = (layers, size, size)
    state = rng.integers(0, 32, size=shape).astype(np.uint32) | (rng.integers(0, 2, size=shape).astype(np.uint32) << rng.integers(5, 16, size=shape).astype(np.uint32))
    phys = np.where(state & B, rng.integers(0, p, size=shape), rng.integers(0, 65536, size=shape)).astype(np.uint32)
    return (state | (phys << 16)).astype(np.uint32)


def random_requests(rng, vsm, n):
    layers, size = int(vsm["clipmap_count"][0]), int(vsm["page_table_size"][0])
    req = np.stack([rng.integers(0, size, n), rng.integers(0, size, n), rng.integers(0, layers, n)], axis=1).astype(np.int32)
    dup = rng.random(n) < 0.2
    req[dup] = req[rng.integers(0, max(1, n // 8), int(dup.sum()))]  # duplicates of a few early requests
    bad = rng.random(n) < 0.05
    req[bad, rng.integers(0, 3, int(bad.sum()))] = rng.choice([-1, size, layers, 1 << 20], int(bad.sum()))
    return req


class Dev:
    """device copies of host arrays on one context, freed together"""

    def __init__(self, ctx):
        self.ctx, self.ptrs = ctx, []

    def put(self, a, extra=0):
        a = np.ascontiguousarray(a)
        p = self.ctx.alloc(a.nbytes + extra)
        self.ctx.upload(p, a)
        self.ptrs.append(p)
        return p

    def get(self, p, like):
        return self.ctx.download(p, like.dtype, like.size).reshape(like.shape)

    def free(self):
        for p in self.ptrs:
            self.ctx.free(p)


def test_begin_frame(ctx, vo):
    rng = np.random.default_rng(1)
    vsm = vsm_context()
    for sun_moved in (False, True):
        pt = random_table(rng, vsm)
        occ = rng.integers(0, 3, physical_count(vsm)).astype(np.uint32)
        d = Dev(ctx)
        d_pt, d_occ, d_cnt = d.put(pt), d.put(occ), d.put(np.uint32([12345]))
        ctx.vsm_begin_frame(vsm, sun_moved, d_pt, d_occ, len(occ), d_cnt)
        want = pt.copy()
        vo.vsm_reset_page_visibility(vsm, sun_moved, want)
        np.testing.assert_array_equal(d.get(d_pt, pt), want)
        assert not d.get(d_occ, occ).any() and int(ctx.download(d_cnt, np.uint32, 1)[0]) == 0
        assert sun_moved == (not want.any())
        d.free()


def test_invalidate_pages(ctx, orc, scene, vo):
    """previous and current boxes of dirty instances over random tables with wrapped (negative) page offsets; one clipmap whose
    projection fails, a dirty index outside the table"""
    rng = np.random.default_rng(2)
    vsm = vsm_context()
    hs = orc.HostScene(scene)
    prev = scene.transforms.copy()
    prev["world"][:, 12:15] += rng.normal(0.0, 4.0, size=(len(prev), 3)).astype(np.float32)
    d = Dev(ctx)
    d_prev = d.put(prev)
    for trial in range(3):
        cm = clipmaps(10, rng)
        cm["z_near"][3] = 2.0  # reverse-Z ortho: w = 1 < z_near, project_aabb fails, nothing is invalidated there
        dirty = np.concatenate([rng.choice(scene.mesh_instance_count, 5 + 5 * trial, replace=False), [scene.mesh_instance_count + 7]]).astype(np.uint32)
        pt = random_table(rng, vsm)
        d_pt, d_dirty = d.put(pt), d.put(dirty)
        ctx.vsm_invalidate_pages(vsm, cm, d_dirty, len(dirty), d_prev, d_pt)
        want = pt.copy()
        vo.vsm_invalidate_pages(vsm, cm, hs, dirty, prev, want)
        got = d.get(d_pt, pt)
        np.testing.assert_array_equal(got, want)
        assert (want == I).sum() > (pt == I).sum() and (want[3] == pt[3]).all()
    # without previous-transform boxes fewer pages go: the previous transform is read
    pt = random_table(rng, vsm)
    d_pt = d.put(pt)
    ctx.vsm_invalidate_pages(vsm, cm, d_dirty, len(dirty), d.put(scene.transforms), d_pt)
    only_current = pt.copy()
    vo.vsm_invalidate_pages(vsm, cm, hs, dirty, scene.transforms, only_current)
    np.testing.assert_array_equal(d.get(d_pt, pt), only_current)
    both = pt.copy()
    vo.vsm_invalidate_pages(vsm, cm, hs, dirty, prev, both)
    assert (both == I).sum() > (only_current == I).sum()
    d.free()


def oracle_allocate(vo, vsm, pt, occ, req, capacity, active):
    al = np.zeros(1, dtype=abi.VSM_ALLOCATOR_DT)
    al["active_request_count"] = active
    fl = np.zeros(len(occ), dtype=np.uint32)
    coords = np.zeros((pt.size, 2), dtype=np.uint32)
    flags = np.zeros(int(vsm["clipmap_count"][0]), dtype=np.uint32)
    vo.vsm_free_invisible_pages(vsm, pt)
    vo.vsm_build_free_page_list(occ, al, fl)
    vo.vsm_allocate_pages(vsm, req, capacity, al, fl, pt)
    vo.vsm_mark_dirty_pages(vsm, pt, al, coords, flags)
    return al, fl, coords, flags


def run_allocate(ctx, vsm, pt, occ, req, capacity, active):
    d = Dev(ctx)
    al = np.zeros(1, dtype=abi.VSM_ALLOCATOR_DT)
    al["active_request_count"] = active
    al["dirty_physical_page_count"], al["free_page_count"], al["alloc_cursor"] = 77, 77, 77
    req_buf = np.zeros((max(capacity, len(req)), 3), dtype=np.int32)
    req_buf[: len(req)] = req
    d_pt, d_occ, d_req, d_al = d.put(pt), d.put(occ), d.put(req_buf), d.put(al)
    d_fl, d_coords = d.put(np.full(len(occ), 0xEEEEEEEE, np.uint32)), d.put(np.full((pt.size, 2), 0xEEEEEEEE, np.uint32))
    d_flags = d.put(np.full(int(vsm["clipmap_count"][0]), 9, np.uint32))
    ctx.vsm_allocate_pages(vsm, d_pt, d_occ, len(occ), d_req, capacity, d_al, d_fl, d_coords, d_flags)
    out = dict(pt=d.get(d_pt, pt), al=ctx.download(d_al, abi.VSM_ALLOCATOR_DT, 1), fl=ctx.download(d_fl, np.uint32, len(occ)),
               coords=ctx.download(d_coords, np.uint32, pt.size * 2).reshape(-1, 2), flags=ctx.download(d_flags, np.uint32, int(vsm["clipmap_count"][0])),
               ptrs=(d_req, d_coords, d_fl))
    d.free()
    return out


def assert_allocate_equal(got, pt_want, al, fl, coords, flags):
    np.testing.assert_array_equal(got["pt"], pt_want)
    for k in ("active_request_count", "dirty_physical_page_count", "free_page_count", "alloc_cursor"):
        assert int(got["al"][k][0]) == int(al[k][0]), k
    assert (int(got["al"]["requests"][0]), int(got["al"]["dirty_physical_page_coords"][0]), int(got["al"]["free_page_list"][0])) == got["ptrs"]
    nf, nd = int(al["free_page_count"][0]), int(al["dirty_physical_page_count"][0])
    np.testing.assert_array_equal(got["fl"][:nf], fl[:nf])
    np.testing.assert_array_equal(got["coords"][:nd], coords[:nd])
    np.testing.assert_array_equal(got["flags"], flags)


@pytest.mark.parametrize("case", ["plenty", "exhausted", "capacity", "small_table"])
def test_allocate_pages(ctx, case, vo):
    """free invisible pages, free list, allocation (duplicates, out-of-range requests) and the dirty list over random tables"""
    rng = np.random.default_rng(hash(case) & 0xFFFF)
    vsm = vsm_context(size=24, layers=3, page_size=16, physical=256) if case == "small_table" else vsm_context()
    pt = random_table(rng, vsm)
    p = physical_count(vsm)
    occ = (rng.random(p) < (0.97 if case == "exhausted" else 0.3)).astype(np.uint32) * rng.integers(1, 4, p).astype(np.uint32)
    n = {"plenty": 3000, "exhausted": 3000, "capacity": 5000, "small_table": 900}[case]
    req = random_requests(rng, vsm, n)
    capacity, active = (2000, n) if case == "capacity" else (n + 100, n)
    got = run_allocate(ctx, vsm, pt, occ, req, capacity, active)
    want = pt.copy()
    al, fl, coords, flags = oracle_allocate(vo, vsm, want, occ, req, capacity, active)
    assert_allocate_equal(got, want, al, fl, coords, flags)
    assert int(al["dirty_physical_page_count"][0]) > 0 and int(al["alloc_cursor"][0]) > 0
    if case == "exhausted":
        assert int(al["alloc_cursor"][0]) > int(al["free_page_count"][0])


def test_allocation_exhaustion_through_marking(ctx, vo):
    """a ground-plane frame that wants more pages than there are free: exactly free_count entries are backed, on distinct
    physical pages, in address order; the other requested entries stay as the marking left them (no AllocationFailed)"""
    from tests.test_oracle_units import make_vsm_case

    inv_pv, res, cm, vsm, depth, _ = make_vsm_case(1920, 1080, size=64, clipmaps=6)
    vsm["page_size"], vsm["physical_page_table_size"] = 128, 1024  # 8 x 8 = 64 physical pages
    p = physical_count(vsm)
    st = vo.VsmState(vsm, 7)
    st.frame(cm, True, None, [], None, inv_pv, res, depth)
    n = int(st.allocator["active_request_count"][0])
    assert n > 2 * p
    d = Dev(ctx)
    d_depth = d.put(depth)
    d_pt, d_occ = d.put(np.zeros_like(st.page_tables)), d.put(np.zeros(p, np.uint32))
    d_al = d.put(np.zeros(1, abi.VSM_ALLOCATOR_DT))
    cap = st.request_capacity
    d_req, d_fl, d_coords, d_flags = d.put(np.zeros((cap, 3), np.int32)), d.put(np.zeros(p, np.uint32)), d.put(np.zeros((st.page_tables.size, 2), np.uint32)), d.put(np.zeros(6, np.uint32))
    d_hpb = d.put(np.zeros_like(st.hpb))
    ctx.vsm_begin_frame(vsm, True, d_pt, d_occ, p, d_al)
    ctx.mark_visible_pages(inv_pv, res, cm, vsm, d_depth, d_pt, d_occ, d_al, d_req, cap)
    ctx.vsm_allocate_pages(vsm, d_pt, d_occ, p, d_req, cap, d_al, d_fl, d_coords, d_flags)
    ctx.build_hpb(d_pt, 64, 6, d_hpb, 7)
    pt = d.get(d_pt, st.page_tables)
    np.testing.assert_array_equal(pt, st.page_tables)
    np.testing.assert_array_equal(d.get(d_hpb, st.hpb), st.hpb)
    backed = (pt & B) != 0
    assert backed.sum() == p and len(np.unique(pt[backed] >> 16)) == p
    requested = (pt & V) != 0
    flat = np.flatnonzero(requested.reshape(-1))
    assert (np.flatnonzero(backed.reshape(-1)) == flat[:p]).all()  # the p lowest requested addresses
    assert (pt.reshape(-1)[flat[p:]] == V).all() and not (pt & F).any()
    # request capacity overflow: which requests are kept is atomics order; check only that nothing lands out of bounds and
    # that every backed entry has a page of its own
    small = 40
    sentinel = np.full((small + 64, 3), -7, np.int32)
    d_req2 = d.put(sentinel)
    ctx.vsm_begin_frame(vsm, True, d_pt, d_occ, p, d_al)
    ctx.mark_visible_pages(inv_pv, res, cm, vsm, d_depth, d_pt, d_occ, d_al, d_req2, small)
    ctx.vsm_allocate_pages(vsm, d_pt, d_occ, p, d_req2, small, d_al, d_fl, d_coords, d_flags)
    req = d.get(d_req2, sentinel)
    assert (req[small:] == -7).all() and (req[:small] >= 0).all()
    al = ctx.download(d_al, abi.VSM_ALLOCATOR_DT, 1)
    assert int(al["active_request_count"][0]) == n and int(al["alloc_cursor"][0]) == small
    pt = d.get(d_pt, st.page_tables)
    backed = (pt & B) != 0
    assert backed.sum() == len(np.unique(pt[backed] >> 16)) <= small
    d.free()


@pytest.mark.parametrize("atlas_size", [2048, 8192])
def test_clear_dirty_pages(ctx, atlas_size, vo):
    """128-px pages: the whole 2048^2 atlas against the oracle; at the reference's 8192^2, every page by itself and a checksum of
    the texels no dirty page covers (page coordinates outside the atlas are not written)"""
    rng = np.random.default_rng(atlas_size)
    vsm = vsm_context(physical=atlas_size)
    n = atlas_size // 128
    k = n * n // 3
    pages = rng.choice(n * n, k, replace=False)
    coords = np.stack([pages % n, pages // n], axis=1).astype(np.uint32)
    coords = np.concatenate([coords, [[n, 0], [0, n + 3]]]).astype(np.uint32)
    al = np.zeros(1, dtype=abi.VSM_ALLOCATOR_DT)
    al["dirty_physical_page_count"] = len(coords)
    atlas = rng.integers(0, 1 << 30, size=(atlas_size, atlas_size), dtype=np.uint32).view(np.float32)
    d = Dev(ctx)
    d_atlas, d_al, d_coords = d.put(atlas), d.put(al), d.put(coords)
    ctx.vsm_clear_dirty_pages(vsm, d_al, d_coords, d_atlas)
    got = d.get(d_atlas, atlas).view(np.uint32)
    if atlas_size <= 2048:
        want = atlas.copy()
        vo.vsm_clear_dirty_pages(vsm, al, coords, want)
        np.testing.assert_array_equal(got, want.view(np.uint32))
    else:
        g = got.reshape(n, 128, n, 128).transpose(0, 2, 1, 3).reshape(n * n, -1)
        a = atlas.view(np.uint32).reshape(n, 128, n, 128).transpose(0, 2, 1, 3).reshape(n * n, -1)
        dirty = np.zeros(n * n, dtype=bool)
        dirty[pages] = True
        assert (g[dirty] == 0x3F800000).all()
        assert int(g[~dirty].astype(np.uint64).sum()) == int(a[~dirty].astype(np.uint64).sum()) and (g[~dirty] == a[~dirty]).all()
    d.free()


def test_hpb_dirty_dev_equals_host_flags(ctx, orc, scene):
    """oxc_cull_meshlets_hpb_dirty_dev with the flags in device memory == oxc_cull_meshlets_hpb with equal host flags == oracle"""
    rng = np.random.default_rng(5)
    hs = orc.HostScene(scene)
    cam0 = scene.camera()
    mi, vis, _ = orc.cull_meshes(hs, cam0, abi.CULL_TEST_ALL)
    ctx.cull_meshes(cam0, abi.CULL_TEST_ALL)
    cm = clipmaps(10, rng, center=(0.0, 0.0, -200.0))
    coarse = synth.make_ortho_view(LIGHT, (0.0, 0.0, -200.0), 10.0 * 2 ** 9, 2000.0, scene.mesh_instance_count)
    coarse["position"][0] = -np.asarray(LIGHT) / np.linalg.norm(LIGHT)
    lv = [(rng.random((10, 64, 64)) < 0.1).astype(np.uint8)]
    for l in range(1, 7):
        q = lv[-1]
        lv.append(np.maximum(np.maximum(q[:, 0::2, 0::2], q[:, 0::2, 1::2]), np.maximum(q[:, 1::2, 0::2], q[:, 1::2, 1::2])))
    hpb = np.concatenate([a.reshape(-1) for a in lv])
    d = Dev(ctx)
    d_hpb = d.put(hpb)
    seen = 0
    for flags in ([1] * 10, [0, 1, 0, 0, 1, 0, 0, 0, 0, 3], [0] * 10):
        d_flags = d.put(np.uint32(flags))
        ref, cmd = orc.cull_meshlets_hpb(hs, mi, vis, coarse, cm, flags, hpb, 64, 7)
        ctx.cull_meshlets_hpb(coarse, cm, flags, d_hpb, 64, 7)
        n = int(ctx.cull_triangles_cmd()["x"][0])
        host = np.sort(ctx.visible_indices(n))
        ctx.cull_meshlets_hpb_dirty_dev(coarse, cm, d_flags, d_hpb, 64, 7)
        assert int(ctx.cull_triangles_cmd()["x"][0]) == n == int(cmd["x"][0])
        np.testing.assert_array_equal(np.sort(ctx.visible_indices(n)), host)
        np.testing.assert_array_equal(host, np.sort(ref))
        seen += n
    assert seen > 0
    d.free()


def test_argument_refusals(capi, ctx):
    vsm = vsm_context()
    d = Dev(ctx)
    buf = d.put(np.zeros(1 << 20, np.uint32))
    p = physical_count(vsm)

    def refused(fn, match):
        with pytest.raises(capi.OxcError, match=match) as e:
            fn()
        assert "(-1)" in str(e.value)

    def bad(**kw):
        v = vsm.copy()
        for k, x in kw.items():
            v[k] = x
        return v

    for v, match in ((bad(clipmap_count=0), "clipmap_count"), (bad(clipmap_count=11), "clipmap_count"), (bad(page_size=100), "does not divide"),
                     (bad(page_size=16), "65536"), (bad(page_table_size=0), "page_table_size")):
        refused(lambda: ctx.vsm_begin_frame(v, False, buf, buf, physical_count(v) if int(v["page_size"][0]) else p, buf), match)
        refused(lambda: ctx.vsm_allocate_pages(v, buf, buf, p, buf, 16, buf, buf, buf, buf), match)
        refused(lambda: ctx.vsm_clear_dirty_pages(v, buf, buf, buf), match)
        refused(lambda: ctx.vsm_invalidate_pages(v, clipmaps(10), buf, 1, buf, buf), match)
    refused(lambda: ctx.vsm_begin_frame(vsm, False, buf, buf, p - 1, buf), "physical_page_count")
    refused(lambda: ctx.vsm_allocate_pages(vsm, buf, buf, p + 1, buf, 16, buf, buf, buf, buf), "physical_page_count")
    refused(lambda: ctx.vsm_begin_frame(vsm, False, None, buf, p, buf), "null")
    refused(lambda: ctx.vsm_allocate_pages(vsm, buf, buf, p, buf, 16, buf, buf, None, buf), "null")
    refused(lambda: ctx.vsm_clear_dirty_pages(vsm, buf, buf, None), "null")
    refused(lambda: ctx.vsm_invalidate_pages(vsm, clipmaps(10), buf, 1, None, buf), "null")
    refused(lambda: ctx.cull_meshlets_hpb_dirty_dev(synth.make_ortho_view(LIGHT, (0, 0, 0), 10.0, 100.0, 1), clipmaps(10), None, buf, 64, 7), "null")
    d.free()


def _sequence_frames(sc, n_frames=8):
    """camera yaw / position per frame, the clipmaps (stable matrices, page offsets scrolling with the camera), sun_moved and
    the transform moves of frames 5-6 (five mesh instances)"""
    rng = np.random.default_rng(11)
    movers = rng.choice(sc.mesh_instance_count, 5, replace=False).astype(np.uint32)
    frames = []
    for f in range(n_frames):
        offsets = [(f * (k + 1) % 64 - 3 * f, (2 * f) % 7 - k) for k in range(10)]
        frames.append(dict(yaw=1.5 * f, clip=clipmaps(10, offsets=offsets), sun_moved=(f == 3),
                           movers=movers if f in (5, 6) else np.zeros(0, np.uint32)))
    return frames


def test_vsm_sequence_through_renderer_full_size(capi, orc, vo):
    """eight frames through oxr_vsm_update_pages at the reference's sizes (64 x 64 pages x 10 clipmaps, 4096 physical pages, 8192^2
    atlas) from the depth the library renders: camera moving, page offsets scrolling, sun_moved at frame 3, five instances moved and
    invalidated at frames 5-6.  Every frame: page table, occupancy, free list, counters, dirty list, flags, HPB, atlas and the
    shadow cull's survivors (oxc_cull_meshlets_hpb_dirty_dev on the device flags) equal the oracle.  Frame 2 repeated with no
    change leaves every visible page resident on the same physical page and clean."""
    sc = synth.make_scene(20000, config_index=2, width=1920, height=1080, n_unique_meshes=32)
    hs = orc.HostScene(sc)
    hs.transforms = hs.transforms.copy()
    hs.desc.transforms = hs.transforms.ctypes.data
    r = capi.Renderer(0, sc)
    hw, hh = sc.hiz_extent()
    cull = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh, max_views=10)
    cull.set_scene(sc)
    vsm = vsm_context()
    st = vo.VsmState(vsm, 7)
    atlas_dirty = np.zeros((64, 64), dtype=bool)
    prev = hs.transforms.copy()
    coarse = synth.make_ortho_view(LIGHT, (0.0, 0.0, -60.0), 10.0 * 2 ** 9, 2000.0, sc.mesh_instance_count)
    coarse["position"][0] = -np.asarray(LIGHT) / np.linalg.norm(LIGHT)
    stats = []
    for f, fr in enumerate(_sequence_frames(sc)):
        if len(fr["movers"]):
            prev = hs.transforms.copy()
            for i in fr["movers"]:
                ti = int(sc.mesh_instances["transform_index"][i])
                hs.transforms["world"][ti, 12:15] += np.float32([3.0, 0.0, -2.0])
                r.update_transforms(np.ascontiguousarray(hs.transforms[ti: ti + 1]), first=ti)
                cull.update_transforms(np.ascontiguousarray(hs.transforms[ti: ti + 1]), first=ti)
        cam = sc.camera(fr["yaw"])
        out = r.render(cam, want_indices=False)
        inv_pv = np.linalg.inv(cam["projection_view"][0].reshape(4, 4).T.astype(np.float64)).T.astype(np.float32).reshape(16)
        res = cam["resolution"][0]
        reps = 2 if f == 2 else 1
        for rep in range(reps):
            before = st.page_tables.copy()
            pg = r.vsm_update_pages(vsm, fr["clip"], inv_pv, res, sun_moved=fr["sun_moved"], dirty_mesh_instances=fr["movers"], hpb_levels=7)
            st.frame(fr["clip"], fr["sun_moved"], hs, fr["movers"], prev, inv_pv, res, out["depth"])
            al = _compare_state(r.ctx, pg, st, f"frame {f}.{rep}")
            atlas_dirty[st.dirty()[:, 1], st.dirty()[:, 0]] = True
            atlas = r.ctx.download(pg.physical_atlas, np.uint32, 8192 * 8192).reshape(64, 128, 64, 128).transpose(0, 2, 1, 3).reshape(64, 64, -1)
            assert (atlas[atlas_dirty] == 0x3F800000).all() and not atlas[~atlas_dirty].any()
            nd = int(al["dirty_physical_page_count"][0])
            stats.append((f, int(al["active_request_count"][0]), nd, int((st.page_tables == I).sum())))
            if f == 0 or fr["sun_moved"]:
                assert nd > 50 and nd == int(al["alloc_cursor"][0])
            if rep == 1:  # nothing changed since the previous update
                vis_pages = (before & V) != 0
                assert nd == 0 and vis_pages.sum() > 50
                assert ((st.page_tables[vis_pages] & (V | B | D)) == (V | B)).all()
                assert ((st.page_tables[vis_pages] >> 16) == (before[vis_pages] >> 16)).all()
            # the shadow cull on the new bitmap, flags read from the device
            mi, vis, _ = orc.cull_meshes(hs, coarse, abi.CULL_TEST_ALL)
            ref, cmd = orc.cull_meshlets_hpb(hs, mi, vis, coarse, fr["clip"], st.dirty_flags, st.hpb, 64, 7)
            cull.cull_meshes(coarse, abi.CULL_TEST_ALL)
            cull.cull_meshlets_hpb_dirty_dev(coarse, fr["clip"], pg.clipmap_dirty_flags, pg.hpb, 64, 7)
            n = int(cull.cull_triangles_cmd()["x"][0])
            assert n == int(cmd["x"][0]), f
            np.testing.assert_array_equal(np.sort(cull.visible_indices(n)), np.sort(ref))
    # frames 5-6 invalidated pages (only resident pages can be invalidated, so their count shows up after the reset)
    assert any(s[0] in (5, 6) for s in stats)
    print("vsm sequence (frame, requests, dirty pages, invalidated entries):", stats)
    cull.close()
    r.close()


def _compare_state(ctx, pg, st, what):
    np.testing.assert_array_equal(ctx.download(pg.page_tables, np.uint32, st.page_tables.size).reshape(st.page_tables.shape), st.page_tables, err_msg=what)
    np.testing.assert_array_equal(ctx.download(pg.page_occupancy, np.uint32, len(st.occupancy)), st.occupancy, err_msg=what)
    al = ctx.download(pg.allocator, abi.VSM_ALLOCATOR_DT, 1)
    for k in ("active_request_count", "dirty_physical_page_count", "free_page_count", "alloc_cursor"):
        assert int(al[k][0]) == int(st.allocator[k][0]), (what, k)
    nf, nd = int(al["free_page_count"][0]), int(al["dirty_physical_page_count"][0])
    np.testing.assert_array_equal(ctx.download(pg.free_page_list, np.uint32, nf), st.free_list[:nf], err_msg=what)
    np.testing.assert_array_equal(ctx.download(pg.dirty_physical_page_coords, np.uint32, 2 * nd).reshape(-1, 2), st.dirty(), err_msg=what)
    np.testing.assert_array_equal(ctx.download(pg.clipmap_dirty_flags, np.uint32, len(st.dirty_flags)), st.dirty_flags, err_msg=what)
    np.testing.assert_array_equal(ctx.download(pg.hpb, np.uint8, st.hpb.size), st.hpb, err_msg=what)
    return al


def test_graph_capture_equals_eager(capi, ctx, scene, vo):
    """the whole sequence (begin, invalidate, mark, allocate, HPB, clear) captured once into a CUDA graph and replayed twice, with a
    new depth image uploaded before the second replay, equals the same calls run eagerly, buffer for buffer"""
    import torch
    from tests.test_oracle_units import make_vsm_case

    inv_pv, res, cm, vsm, depth0, _ = make_vsm_case(640, 360, size=64, clipmaps=6)
    vsm["page_size"], vsm["physical_page_table_size"] = 64, 4096  # 4096 physical pages: the second frame still finds free ones
    depth1 = np.roll(depth0, 37, axis=1)
    p = physical_count(vsm)
    entries = 6 * 64 * 64
    st = vo.VsmState(vsm, 7)
    prev = scene.transforms.copy()
    prev["world"][:, 12] += np.float32(5.0)

    def buffers():
        d = Dev(ctx)
        b = dict(depth=d.put(depth0), pt=d.put(st.page_tables), occ=d.put(np.zeros(p, np.uint32)), req=d.put(np.zeros((entries, 3), np.int32)),
                 al=d.put(np.zeros(1, abi.VSM_ALLOCATOR_DT)), fl=d.put(np.zeros(p, np.uint32)), coords=d.put(np.zeros((entries, 2), np.uint32)),
                 flags=d.put(np.zeros(6, np.uint32)), hpb=d.put(np.zeros_like(st.hpb)), atlas=d.put(np.zeros((4096, 4096), np.float32)),
                 dirty=d.put(np.uint32([0, 1, 2, 3])), prev=d.put(prev))
        return d, b

    def enqueue(c, b):
        c.vsm_begin_frame(vsm, False, b["pt"], b["occ"], p, b["al"])
        c.vsm_invalidate_pages(vsm, cm, b["dirty"], 4, b["prev"], b["pt"])
        c.mark_visible_pages(inv_pv, res, cm, vsm, b["depth"], b["pt"], b["occ"], b["al"], b["req"], entries)
        c.vsm_allocate_pages(vsm, b["pt"], b["occ"], p, b["req"], entries, b["al"], b["fl"], b["coords"], b["flags"])
        c.build_hpb(b["pt"], 64, 6, b["hpb"], 7)
        c.vsm_clear_dirty_pages(vsm, b["al"], b["coords"], b["atlas"])

    def snapshot(d, b):
        return [ctx.download(b[k], dt, n) for k, dt, n in (("pt", np.uint32, entries), ("occ", np.uint32, p), ("al", np.uint32, 4), ("fl", np.uint32, p),
                                                           ("coords", np.uint32, 2 * entries), ("flags", np.uint32, 6), ("hpb", np.uint8, st.hpb.size),
                                                           ("atlas", np.uint32, 4096 * 4096))]

    de, be = buffers()
    eager = []
    for dep in (depth0, depth1):
        ctx.upload(be["depth"], dep)
        enqueue(ctx, be)
        eager.append(snapshot(de, be))
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
        for a, b_ in zip(snapshot(dg, bg), eager[k]):
            np.testing.assert_array_equal(a, b_)
    assert int(eager[0][2][1]) > 20 and int(eager[1][2][1]) > 0  # both frames allocated and cleared pages
    del g
    de.free()
    dg.free()
