"""The oracle's shadow-clipmap, multi-view and terrain culls against the independent float64 reference of tests/test_gpu_culls.py,
on the oracle alone (no GPU): every decision equals the float64 one unless a float64 quantity lies within the stated margin of its
edge, and such excused decisions stay under 1 % of all."""
import numpy as np
import pytest

from oxylus_b200 import abi
from tests.test_gpu_culls import (EXCUSED_BOUND, _views, assert_f64_agrees, box_scene, clipmaps_for, coarse_view, f64_hpb,
                                  f64_multiview, f64_terrain, mask_bits, offset_patterns, perspective_views, random_page_table,
                                  survivors_to_mask, terrain_cameras, terrain_minmax, terrain_pyramids, terrain_record, DIRTY,
                                  FLAG_SUBSETS, OCC, LATE, TERRAIN_W, TERRAIN_H)


@pytest.fixture(scope="module")
def box(orc):
    sc = box_scene()
    hs = orc.HostScene(sc)
    mi, vis, _ = orc.cull_meshes(hs, sc.camera(), abi.CULL_TEST_ALL)
    return sc, hs, mi, vis


def test_hpb_oracle_matches_float64(orc, box):
    sc, hs, mi, vis = box
    total = int(vis["total"][0])
    rng = np.random.default_rng(5)
    excused = decisions = 0
    for size, levels, count in ((16, 5, 16), (48, 3, 5), (64, 7, 10), (128, 16, 3), (1, 1, 1)):
        hpb = orc.build_hpb(random_page_table(rng, size, count), levels)
        for k, mk in enumerate(DIRTY.values()):
            clip = clipmaps_for(sc, count, offset_patterns(size, rng)[k + 2], z_near_every=3 if k == 3 else 0)
            dirty = mk(count)
            ref, _ = orc.cull_meshlets_hpb(hs, mi, vis, coarse_view(sc), clip, dirty, hpb, size, levels)
            want, near = f64_hpb(hs, mi, total, coarse_view(sc), clip, dirty, hpb, size, levels)
            excused += assert_f64_agrees(f"size {size} levels {levels} clipmaps {count}", survivors_to_mask(ref, total), want, near)
            decisions += total
    print(f"hpb: {excused} of {decisions} float64 decisions excused")
    assert excused <= EXCUSED_BOUND * decisions


@pytest.mark.parametrize("directional", [1, 0])
def test_multiview_oracle_matches_float64(orc, box, directional):
    sc, hs, mi, vis = box
    total = int(vis["total"][0])
    views = _views(sc, abi.MAX_VIEWS, 2) if directional else perspective_views(sc, abi.MAX_VIEWS)
    bits, counts = orc.cull_meshlets_multiview(hs, mi, total, views, directional)
    got = ((bits[:, None] >> np.arange(abi.MAX_VIEWS, dtype=np.uint32)) & 1).astype(bool)
    want, near = f64_multiview(hs, mi, total, views, directional)
    excused = assert_f64_agrees(f"multiview directional {directional}", got, want, near)
    np.testing.assert_array_equal(counts, got.sum(0))
    print(f"multiview directional {directional}: {excused} of {got.size} float64 decisions excused")
    assert excused <= EXCUSED_BOUND * got.size and got.any()


def test_terrain_oracle_matches_float64(orc):
    rng = np.random.default_rng(77)
    hw, hh = abi.hiz_extent(TERRAIN_W, TERRAIN_H)
    pyramids, _ = terrain_pyramids(orc, rng)
    excused = decisions = 0
    for nx, ny, hscale in ((33, 31, 40.0), (7, 5, 0.0), (96, 80, -25.0)):
        n = nx * ny
        t = terrain_record(nx, ny, hscale)
        mm = terrain_minmax(rng, n)
        for cam in terrain_cameras().values():
            for pyr in pyramids.values():
                levels = [pyr.level(l) for l in range(pyr.levels)]
                for flags in FLAG_SUBSETS:
                    mask = rng.integers(0, 2**32, size=(n + 31) // 32, dtype=np.uint64).astype(np.uint32)
                    before = mask.copy()
                    ref, _ = orc.cull_terrain(t, mm, cam, flags, pyr, mask)
                    emit, visible, near = f64_terrain(t, mm, cam, flags, levels, hw, hh, before)
                    tag = f"{nx}x{ny} flags {flags:#x}"
                    excused += assert_f64_agrees(tag, survivors_to_mask(ref, n), emit, near)
                    assert_f64_agrees(tag + ": mask", mask_bits(mask, n), visible if flags & (OCC | LATE) else mask_bits(before, n), near)
                    decisions += n
    print(f"terrain: {excused} of {decisions} float64 decisions excused")
    assert excused <= EXCUSED_BOUND * decisions
