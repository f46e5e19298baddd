"""ctypes wrapper of the VSM shadow-raster oracle (oracle/oxc_oracle_vsm_draw.c, one translation unit with oxc_oracle.c and
oxc_oracle_vsm.c, built into oracle/liboxc_oracle_vsm_draw.so).  TEST INFRASTRUCTURE ONLY: tests/ import it; the product package
never does."""
import ctypes as C

import numpy as np

import pyoracle
from pyoracle import _p

_LIB = None
SOURCES = ("oxc_oracle.c", "oxc_oracle.h", "oxc_oracle_math.inc", "oxc_oracle_vsm.c", "oxc_oracle_vsm.h", "oxc_oracle_vsm_draw.c",
           "oxc_oracle_vsm_draw.h")


def build(force=False):
    """compiles liboxc_oracle_vsm_draw.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_vsm_draw.so", ["oxc_oracle_vsm_draw.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.orc_vsm_draw_pages.restype = C.c_uint64
    return _LIB


def vsm_draw_pages(hs, meshlet_instances, survivors, coarse, vsm, clipmaps, dirty_flags, page_tables, atlas, materials=None):
    """orc_vsm_draw_pages: atlas (P x P float32) is updated in place; materials = a pyoracle.MaterialTable or None.  Returns the
    fragments that reached the sink."""
    s = np.ascontiguousarray(survivors, dtype=np.uint32)
    flags = np.ascontiguousarray(dirty_flags, dtype=np.uint32)
    pt = np.ascontiguousarray(page_tables, dtype=np.uint32)
    assert atlas.dtype == np.float32 and atlas.flags.c_contiguous
    table = C.byref(materials.ref) if materials is not None else None
    return int(lib().orc_vsm_draw_pages(hs.ref, _p(np.ascontiguousarray(meshlet_instances)), _p(s), C.c_uint32(len(s)),
                                        _p(np.ascontiguousarray(coarse)), _p(np.ascontiguousarray(vsm)), _p(np.ascontiguousarray(clipmaps)),
                                        _p(flags), _p(pt), table, _p(atlas)))


__all__ = ["build", "lib", "vsm_draw_pages", "pyoracle"]
