"""ctypes wrapper of the VSM page-bookkeeping oracle (oracle/oxc_oracle_vsm.c, built with oxc_oracle.c into
oracle/liboxc_oracle_vsm.so).  TEST INFRASTRUCTURE ONLY: tests/ import it; the product package never does.

Page tables are (layers, size, size) u32 arrays and every other array is updated in place.  Scenes are pyoracle.HostScene
objects (the same OrcScene layout)."""
import ctypes as C

import numpy as np

import pyoracle
from pyoracle import HostScene, _p, hpb_layout  # noqa: F401  (HostScene: re-exported for the tests)
from oxylus_b200 import abi

_LIB = None
SOURCES = ("oxc_oracle.c", "oxc_oracle.h", "oxc_oracle_math.inc", "oxc_oracle_vsm.c", "oxc_oracle_vsm.h")


def build(force=False):
    """compiles liboxc_oracle_vsm.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_vsm.so", ["oxc_oracle.c", "oxc_oracle_vsm.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
    return _LIB


def build_hpb(page_table, levels):
    return pyoracle.build_hpb(page_table, levels)


# ---- VSM page bookkeeping (orc_vsm_*): page tables (layers, size, size) u32 and the other arrays are updated in place ----
def vsm_reset_page_visibility(vsm, sun_moved, page_tables):
    lib().orc_vsm_reset_page_visibility(_p(np.ascontiguousarray(vsm)), C.c_int(int(bool(sun_moved))), _p(page_tables))


def vsm_invalidate_pages(vsm, clipmaps, hs, dirty, previous_transforms, page_tables):
    d = np.ascontiguousarray(dirty, dtype=np.uint32)
    lib().orc_vsm_invalidate_pages(_p(np.ascontiguousarray(vsm)), _p(np.ascontiguousarray(clipmaps)), hs.ref, _p(d), C.c_uint32(len(d)),
                                   _p(np.ascontiguousarray(previous_transforms)), _p(page_tables))


def vsm_free_invisible_pages(vsm, page_tables):
    lib().orc_vsm_free_invisible_pages(_p(np.ascontiguousarray(vsm)), _p(page_tables))


def vsm_build_free_page_list(occupancy, allocator, free_list):
    occ = np.ascontiguousarray(occupancy, dtype=np.uint32)
    lib().orc_vsm_build_free_page_list(_p(occ), C.c_uint32(len(occ)), _p(allocator), _p(free_list))


def vsm_allocate_pages(vsm, requests, request_capacity, allocator, free_list, page_tables):
    req = np.ascontiguousarray(requests, dtype=np.int32).reshape(-1)
    if req.size < 3 * request_capacity:
        req = np.concatenate([req, np.zeros(3 * request_capacity - req.size, dtype=np.int32)])
    lib().orc_vsm_allocate_pages(_p(np.ascontiguousarray(vsm)), _p(req), C.c_uint32(request_capacity), _p(allocator), _p(free_list), _p(page_tables))


def vsm_mark_dirty_pages(vsm, page_tables, allocator, dirty_coords, dirty_flags):
    lib().orc_vsm_mark_dirty_pages(_p(np.ascontiguousarray(vsm)), _p(page_tables), _p(allocator), _p(dirty_coords), _p(dirty_flags))


def vsm_clear_dirty_pages(vsm, allocator, dirty_coords, atlas):
    lib().orc_vsm_clear_dirty_pages(_p(np.ascontiguousarray(vsm)), _p(allocator), _p(dirty_coords), _p(atlas))


class VsmState:
    """Everything one VSM frame reads and writes (host arrays), sized from an abi.VSM_CONTEXT_DT record."""

    def __init__(self, vsm, hpb_levels, request_capacity=None):
        v = vsm[0] if vsm.shape else vsm
        self.vsm = np.ascontiguousarray(vsm, dtype=abi.VSM_CONTEXT_DT).reshape(1)
        layers, size = int(v["clipmap_count"]), int(v["page_table_size"])
        n = int(v["physical_page_table_size"]) // int(v["page_size"])
        self.page_tables = np.zeros((layers, size, size), dtype=np.uint32)
        self.occupancy = np.zeros(n * n, dtype=np.uint32)
        self.request_capacity = request_capacity or layers * size * size
        self.requests = np.zeros((self.request_capacity, 3), dtype=np.int32)
        self.allocator = np.zeros(1, dtype=abi.VSM_ALLOCATOR_DT)
        self.free_list = np.zeros(n * n, dtype=np.uint32)
        self.dirty_coords = np.zeros((layers * size * size, 2), dtype=np.uint32)
        self.dirty_flags = np.zeros(layers, dtype=np.uint32)
        self.hpb_levels = hpb_levels
        self.hpb = np.zeros(hpb_layout(size, layers, hpb_levels)[1], dtype=np.uint8)

    def dirty(self):
        return self.dirty_coords[: int(self.allocator["dirty_physical_page_count"][0])]

    def frame(self, clipmaps, sun_moved, hs, dirty, previous_transforms, inv_pv, resolution, depth, atlas=None):
        """orc_vsm_frame: steps 0-10 of Shadowmaps.cpp:100-430 (atlas: float32 array updated in place, or None)"""
        d = np.ascontiguousarray(dirty, dtype=np.uint32)
        prev = np.ascontiguousarray(previous_transforms) if previous_transforms is not None else np.zeros(1, dtype=abi.TRANSFORM_DT)
        lib().orc_vsm_frame(_p(self.vsm), _p(np.ascontiguousarray(clipmaps)), C.c_int(int(bool(sun_moved))), hs.ref if hs is not None else None,
                            _p(d), C.c_uint32(len(d)), _p(prev), _p(np.ascontiguousarray(inv_pv, dtype=np.float32)),
                            _p(np.ascontiguousarray(resolution, dtype=np.float32)), _p(np.ascontiguousarray(depth, dtype=np.float32)),
                            _p(self.page_tables), _p(self.occupancy), C.c_uint32(len(self.occupancy)), _p(self.requests),
                            C.c_uint32(self.request_capacity), _p(self.allocator), _p(self.free_list), _p(self.dirty_coords), _p(self.dirty_flags),
                            _p(self.hpb), C.c_uint32(self.hpb_levels), _p(atlas) if atlas is not None else None)
