"""Known-answer tests of the oracle's VSM page bookkeeping (oracle/oxc_oracle_vsm.c orc_vsm_*, the passes of
Passes/Shadowmaps.cpp:100-430).  Every expected value below is worked out by hand from the shaders' text and the canonical
orders include/oxcull.h commits to (free list ascending, requests ranked by page table address, dirty list ascending)."""
import types

import numpy as np
import pytest

from oxylus_b200 import abi


@pytest.fixture(scope="module")
def vo():
    """the VSM oracle (oracle/pyoracle_vsm.py)"""
    import pyoracle_vsm

    pyoracle_vsm.build()
    return pyoracle_vsm


V, D, B, I, F = abi.VSM_PAGE_VISIBLE, abi.VSM_PAGE_DIRTY, abi.VSM_PAGE_BACKED, abi.VSM_PAGE_INVALIDATED, abi.VSM_PAGE_ALLOCATION_FAILED


def small_vsm(size=4, layers=2, page_size=4, physical=16):
    vsm = np.zeros(1, dtype=abi.VSM_CONTEXT_DT)
    vsm["page_size"], vsm["page_table_size"], vsm["physical_page_table_size"], vsm["clipmap_count"] = page_size, size, physical, layers
    return vsm


def entry(bits, phys=0):
    return np.uint32(bits | (phys << 16))


def alloc_state(vsm, free_list, active):
    al = np.zeros(1, dtype=abi.VSM_ALLOCATOR_DT)
    al["free_page_count"], al["active_request_count"] = len(free_list), active
    fl = np.zeros(64, dtype=np.uint32)
    fl[: len(free_list)] = free_list
    return al, fl


def test_reset_page_visibility(vo):
    """rmvsm_reset_page_visibility: Visible, Dirty and Invalidated cleared, Backed, AllocationFailed, other metadata bits and the
    address kept; sun_moved clears every entry (vuk::clear_image, Shadowmaps.cpp:143-148)"""
    vsm = small_vsm()
    pt = np.zeros((2, 4, 4), dtype=np.uint32)
    pt[0, 0, 0] = entry(V | D | B | I | F | 0x20, 0xABCD)
    pt[1, 3, 2] = entry(V | I, 7)
    pt[1, 1, 1] = entry(D)
    vo.vsm_reset_page_visibility(vsm, False, pt)
    assert pt[0, 0, 0] == entry(B | F | 0x20, 0xABCD)
    assert pt[1, 3, 2] == entry(0, 7) and pt[1, 1, 1] == 0
    pt[0, 1, 0] = entry(B, 3)
    vo.vsm_reset_page_visibility(vsm, True, pt)
    assert not pt.any()


def test_free_invisible_pages_and_free_list(vo):
    """rmvsm_free_invisible_pages: only !Visible && Backed loses Backed (address stays); rmvsm_build_free_page_list: the physical
    pages with occupancy 0, ascending"""
    vsm = small_vsm()
    pt = np.zeros((2, 4, 4), dtype=np.uint32)
    pt[0, 0, 1] = entry(B | D, 9)
    pt[0, 0, 2] = entry(V | B, 4)
    pt[0, 0, 3] = entry(V, 5)
    vo.vsm_free_invisible_pages(vsm, pt)
    assert pt[0, 0, 1] == entry(D, 9) and pt[0, 0, 2] == entry(V | B, 4) and pt[0, 0, 3] == entry(V, 5)
    occ = np.ones(16, dtype=np.uint32)
    occ[[0, 3, 4, 15]] = 0
    al = np.zeros(1, dtype=abi.VSM_ALLOCATOR_DT)
    fl = np.full(16, 99, dtype=np.uint32)
    vo.vsm_build_free_page_list(occ, al, fl)
    assert int(al["free_page_count"][0]) == 4 and fl[:4].tolist() == [0, 3, 4, 15]


def test_allocate_ranks_by_address(vo):
    """requests in any order take free-list slots in page table address order; the entry keeps its low 16 bits and gains the
    physical address, Dirty and Backed"""
    vsm = small_vsm()
    pt = np.zeros((2, 4, 4), dtype=np.uint32)
    pt[1, 0, 0] = entry(V | 0x20, 0x3FF)  # stale address bits are replaced
    pt[0, 2, 1] = entry(V)
    req = np.array([[0, 0, 1], [1, 2, 0]], dtype=np.int32)  # layer 1 first in the list, but address 16 > 9
    al, fl = alloc_state(vsm, [2, 5, 7], 2)
    vo.vsm_allocate_pages(vsm, req, 8, al, fl, pt)
    assert pt[0, 2, 1] == entry(V | D | B, 2) and pt[1, 0, 0] == entry(V | D | B | 0x20, 5)
    assert int(al["alloc_cursor"][0]) == 2


def test_allocate_duplicates_out_of_range_and_capacity(vo):
    """d requests for one entry consume d consecutive slots and the entry takes the highest of them below the free count;
    requests outside the table are skipped and take no slot; only the first min(count, capacity) requests are read"""
    vsm = small_vsm()
    pt = np.zeros((2, 4, 4), dtype=np.uint32)
    req = np.array([[1, 0, 0], [-1, 0, 0], [0, 0, 0], [4, 0, 0], [0, 0, 0], [0, 0, 2], [0, 4, 1], [2, 0, 0]], dtype=np.int32)
    al, fl = alloc_state(vsm, [2, 5, 7, 11], 8)
    vo.vsm_allocate_pages(vsm, req, 8, al, fl, pt)
    # address 0 (x=0): slots 0, 1 -> free_list[1] = 5; address 1: slot 2 -> 7; address 2: slot 3 -> 11
    assert pt[0, 0, 0] == entry(D | B, 5) and pt[0, 0, 1] == entry(D | B, 7) and pt[0, 0, 2] == entry(D | B, 11)
    assert int(al["alloc_cursor"][0]) == 4 and np.count_nonzero(pt) == 3
    # capacity 3 of active 8: [1,0,0], [-1,0,0], [0,0,0] are read
    pt[:] = 0
    al, fl = alloc_state(vsm, [2, 5, 7, 11], 8)
    vo.vsm_allocate_pages(vsm, req, 3, al, fl, pt)
    assert pt[0, 0, 0] == entry(D | B, 2) and pt[0, 0, 1] == entry(D | B, 5) and np.count_nonzero(pt) == 2
    assert int(al["alloc_cursor"][0]) == 2


def test_allocation_failed_quirk(vo):
    """a request whose slot is past the free count leaves its entry exactly as it was: the shader sets AllocationFailed on its
    local copy and returns without storing (rmvsm_allocate_pages.slang:32-35); duplicates straddling the free count still take
    the highest slot below it"""
    vsm = small_vsm()
    pt = np.zeros((2, 4, 4), dtype=np.uint32)
    pt[0, 0, 0] = entry(V, 3)
    pt[0, 0, 1] = entry(V, 3)
    pt[0, 1, 0] = entry(V | 0x40, 0x1234)
    req = np.array([[0, 1, 0], [0, 0, 0], [1, 0, 0], [0, 0, 0], [0, 0, 0]], dtype=np.int32)
    al, fl = alloc_state(vsm, [6, 9], 5)
    vo.vsm_allocate_pages(vsm, req, 5, al, fl, pt)
    # address 0 has three requests: slots 0..2, highest below 2 is 1 -> 9; address 1 (slot 3) and address 4 (slot 4) fail
    assert pt[0, 0, 0] == entry(V | D | B, 9)
    assert pt[0, 0, 1] == entry(V, 3) and pt[0, 1, 0] == entry(V | 0x40, 0x1234)
    assert not (pt & F).any()
    assert int(al["alloc_cursor"][0]) == 5


def test_mark_dirty_and_clear(vo):
    """rmvsm_mark_dirty_pages: Backed && Dirty entries in address order push (address % n, address / n), the layer's flag is 1,
    the others 0; rmvsm_clear_dirty_pages writes 1.0 into exactly those pages (a page outside the atlas is not written)"""
    vsm = small_vsm()
    pt = np.zeros((2, 4, 4), dtype=np.uint32)
    pt[1, 0, 0] = entry(B | D, 6)     # address 16
    pt[0, 3, 3] = entry(B | D | V, 1)  # address 15
    pt[0, 0, 0] = entry(D, 2)          # not backed
    pt[0, 0, 1] = entry(B, 3)          # not dirty
    pt[1, 1, 1] = entry(B | D, 17)     # physical address past the atlas (4 x 4 pages)
    al = np.zeros(1, dtype=abi.VSM_ALLOCATOR_DT)
    coords = np.zeros((32, 2), dtype=np.uint32)
    flags = np.full(2, 7, dtype=np.uint32)
    vo.vsm_mark_dirty_pages(vsm, pt, al, coords, flags)
    assert int(al["dirty_physical_page_count"][0]) == 3
    assert coords[:3].tolist() == [[1, 0], [2, 1], [1, 4]] and flags.tolist() == [1, 1]
    pt[1] = 0
    vo.vsm_mark_dirty_pages(vsm, pt, al, coords, flags)
    assert flags.tolist() == [1, 0]
    atlas = np.zeros((16, 16), dtype=np.float32)
    al["dirty_physical_page_count"] = 3
    coords[:3] = [[1, 0], [2, 1], [1, 4]]
    vo.vsm_clear_dirty_pages(vsm, al, coords, atlas)
    want = np.zeros((16, 16), dtype=np.float32)
    want[0:4, 4:8] = 1.0
    want[4:8, 8:12] = 1.0
    np.testing.assert_array_equal(atlas, want)


def _one_instance_scene(world, center=(0.0, 0.0, 0.0), extent=(1.0, 1.0, 1.0)):
    meshes = np.zeros(1, dtype=abi.MESH_DT)
    meshes["bounds"]["aabb_center"][0], meshes["bounds"]["aabb_extent"][0] = center, extent
    inst = np.zeros(1, dtype=abi.MESH_INSTANCE_DT)
    xf = np.zeros(1, dtype=abi.TRANSFORM_DT)
    xf["world"][0] = np.asarray(world, dtype=np.float32).reshape(16)
    return types.SimpleNamespace(meshes=meshes, mesh_instances=inst, transforms=xf, blob=np.zeros(16, dtype=np.uint8), max_meshlet_instance_count=1)


def _translate(tx):
    m = np.eye(4, dtype=np.float32).T.reshape(16).copy()
    m[12] = tx
    return m


def test_invalidate_pages(vo):
    """rmvsm_invalidate_pages with identity clipmaps: the unit box at the origin covers uv [0.25, 0.75] -> pages 1..2; the previous
    transform (x + 1) covers uv [0.75, 1] -> page 3.  Backed entries there become exactly Invalidated, others stay; the page
    offset wraps the columns; a failed projection (z_near above w) and an out-of-range dirty index invalidate nothing"""
    vsm = small_vsm()
    hs = vo.HostScene(_one_instance_scene(np.eye(4, dtype=np.float32).reshape(16)))
    prev = np.zeros(1, dtype=abi.TRANSFORM_DT)
    prev["world"][0] = _translate(1.0)
    cm = np.zeros(2, dtype=abi.CLIPMAP_DT)
    cm["projection_view_mat"][:] = np.eye(4, dtype=np.float32).reshape(16)
    cm["page_offset"][1] = (1, 0)
    cm["z_near"][1] = 0.0
    cm["z_near"][0] = 2.0  # w = 1 < z_near: project_aabb fails -> layer 0 untouched
    pt = np.full((2, 4, 4), entry(B | V | D, 0x55), dtype=np.uint32)
    pt[1, 1, 0] = entry(V, 0x55)  # wrapped column 0 (virtual 3) not backed: unchanged
    vo.vsm_invalidate_pages(vsm, cm, hs, [0, 5], prev, pt)
    want = np.full((2, 4, 4), entry(B | V | D, 0x55), dtype=np.uint32)
    want[1, 1, 0] = entry(V, 0x55)
    for y in (1, 2):
        for x in (1, 2, 3):
            wx = (x + 1) % 4
            if not (y == 1 and wx == 0):
                want[1, y, wx] = I
    np.testing.assert_array_equal(pt, want)
    # without the previous-transform box only virtual columns 1..2 (wrapped 2..3)
    pt[:] = entry(B, 1)
    vo.vsm_invalidate_pages(vsm, cm, hs, [0], hs.transforms, pt)
    assert sorted(zip(*np.nonzero(pt[1] == I))) == [(1, 2), (1, 3), (2, 2), (2, 3)] and not (pt[0] == I).any()


def _sequence_case():
    from tests.test_oracle_units import make_vsm_case

    inv_pv, res, cm, vsm, depth, _ = make_vsm_case(160, 90, size=64, clipmaps=6)
    vsm["page_size"], vsm["physical_page_table_size"] = 128, 8192  # 64 x 64 = 4096 physical pages (RendererInstance.hpp:262-267)
    return inv_pv, res, cm, vsm, depth


def test_two_frame_sequence_keeps_resident_pages(vo):
    """orc_vsm_frame twice on the same view: frame 1 (sun_moved) allocates a physical page for every visible page and clears it;
    frame 2 finds them backed, requests nothing, keeps every page on its physical page and dirties none"""
    inv_pv, res, cm, vsm, depth = _sequence_case()
    st = vo.VsmState(vsm, 7)
    atlas = np.zeros((8192, 8192), dtype=np.float32)
    st.frame(cm, True, None, [], None, inv_pv, res, depth, atlas)
    n = int(st.allocator["active_request_count"][0])
    visible = (st.page_tables & V) != 0
    assert n > 20 and n == int(visible.sum()) == int(st.allocator["dirty_physical_page_count"][0]) == int(st.allocator["alloc_cursor"][0])
    assert ((st.page_tables[visible] & (B | D)) == (B | D)).all()
    phys = st.page_tables[visible] >> 16
    assert sorted(phys.tolist()) == list(range(n))  # ascending free list, all pages free after the clear
    assert st.dirty_flags.tolist() == [int(visible[l].any()) for l in range(6)]
    pages = atlas.reshape(64, 128, 64, 128).transpose(0, 2, 1, 3).reshape(64, 64, -1)
    cleared = np.zeros((64, 64), dtype=bool)
    cleared[st.dirty()[:, 1], st.dirty()[:, 0]] = True
    assert (pages[cleared] == 1.0).all() and (pages[~cleared] == 0.0).all()
    first = st.page_tables.copy()
    st.frame(cm, False, None, [], None, inv_pv, res, depth, atlas)
    assert int(st.allocator["active_request_count"][0]) == 0 and int(st.allocator["dirty_physical_page_count"][0]) == 0
    np.testing.assert_array_equal(st.page_tables, first & ~np.uint32(D))
    assert st.dirty_flags.tolist() == [0] * 6 and int(st.allocator["free_page_count"][0]) == 4096 - n
    assert not vo.build_hpb(st.page_tables, 7).any() and not st.hpb.any()  # nothing dirty: the shadow cull has nothing to redraw
