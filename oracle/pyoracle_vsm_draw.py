"""ctypes wrapper of the VSM shadow-raster oracle (oracle/oxc_oracle_vsm_draw.c, one translation unit with oxc_oracle.c and
oxc_oracle_vsm.c, built into oracle/liboxc_oracle_vsm_draw.so).  TEST INFRASTRUCTURE ONLY: tests/ import it; the product package
never does."""
import ctypes as C
import os
import subprocess

import numpy as np

import pyoracle
from pyoracle import _p
from pyoracle_vsm import CFLAGS

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
SOURCES = ("oxc_oracle.c", "oxc_oracle.h", "oxc_oracle_math.inc", "oxc_oracle_vsm.c", "oxc_oracle_vsm.h", "oxc_oracle_vsm_draw.c",
           "oxc_oracle_vsm_draw.h")


def build(force=False):
    """compiles liboxc_oracle_vsm_draw.so next to the sources when it is missing or older than them"""
    so = os.path.join(_HERE, "liboxc_oracle_vsm_draw.so")
    srcs = [os.path.join(_HERE, f) for f in SOURCES] + [os.path.join(os.path.dirname(_HERE), "include", "oxcull.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        tmp = so + f".{os.getpid()}.tmp"
        subprocess.check_call([os.environ.get("CC", "gcc")] + CFLAGS + ["-shared", "-o", tmp, os.path.join(_HERE, "oxc_oracle_vsm_draw.c"),
                                                                         "-lm", "-lpthread"])
        os.replace(tmp, so)
    return so


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
