"""ctypes wrapper of the terrain-draw oracle (oracle/oxc_oracle_terrain_draw.c, one translation unit with oxc_oracle_vsm_resolve.c and the
sources it includes, built into oracle/liboxc_oracle_terrain_draw.so).  TEST INFRASTRUCTURE ONLY: tests/ and tools/ import it; the product
package never does.  Heightmaps are uint16 [res_y, res_x]; settings are abi.TERRAIN_DRAW_SETTINGS_DT records."""
import ctypes as C

import numpy as np

import pyoracle
from pyoracle import _p
from pyoracle_vsm_resolve import SOURCES as _RESOLVE_SOURCES

_LIB = None
SOURCES = _RESOLVE_SOURCES + ("oxc_oracle_terrain_draw.c", "oxc_oracle_terrain_draw.h")
MAX_PATCH_TRIANGLES = 8192


class Patch(C.Structure):
    """OrcTerrainPatch"""

    _fields_ = [("corner", (C.c_float * 3) * 4), ("factor", C.c_float * 6), ("pinned", C.c_float * 6), ("n", C.c_int32 * 6),
                ("triangles", C.c_uint32)]


def build(force=False):
    """compiles liboxc_oracle_terrain_draw.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_terrain_draw.so", ["oxc_oracle_terrain_draw.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        f, u32, i32, vp = C.c_float, C.c_uint32, C.c_int32, C.c_void_p
        _LIB.orc_terrain_projection_scale.restype, _LIB.orc_terrain_projection_scale.argtypes = f, [f, f]
        _LIB.orc_terrain_factor_clamp.restype, _LIB.orc_terrain_factor_clamp.argtypes = f, [f]
        _LIB.orc_terrain_round_odd.restype, _LIB.orc_terrain_round_odd.argtypes = i32, [f]
        _LIB.orc_terrain_edge_points.argtypes = [f, i32, vp]
        _LIB.orc_terrain_patch.argtypes = [vp, u32, u32, vp, vp, u32, vp]
        _LIB.orc_terrain_patch_domain.restype, _LIB.orc_terrain_patch_domain.argtypes = u32, [vp, vp, u32]
        _LIB.orc_draw_terrain.restype = C.c_uint64
        _LIB.orc_draw_terrain.argtypes = [vp, u32, u32, vp, vp, u32, vp, u32, u32, u32, vp]
    return _LIB


def projection_scale(fov, resolution_y):
    return np.float32(lib().orc_terrain_projection_scale(float(np.float32(fov)), float(np.float32(resolution_y))))


def factor_clamp(f):
    return np.float32(lib().orc_terrain_factor_clamp(float(np.float32(f))))


def round_odd(f):
    return int(lib().orc_terrain_round_odd(float(np.float32(f))))


def edge_points(f, n):
    out = np.zeros(n + 1, np.float32)
    lib().orc_terrain_edge_points(float(np.float32(f)), int(n), _p(out))
    return out


def _hm(heightmap):
    hm = np.ascontiguousarray(heightmap, dtype=np.uint16)
    assert hm.ndim == 2
    return hm


def patch(heightmap, settings, cam, patch_index):
    """items 1-2 of one patch: a Patch (corner, factor, pinned, n, triangles)"""
    hm = _hm(heightmap)
    st = np.ascontiguousarray(settings)
    out = Patch()
    lib().orc_terrain_patch(_p(hm), hm.shape[1], hm.shape[0], _p(st), _p(np.ascontiguousarray(cam)), int(patch_index), C.byref(out))
    return out


def patch_domain(p):
    """item 3: float32 [triangles, 3, 2] domain points in the raster's order"""
    tris = np.zeros((MAX_PATCH_TRIANGLES, 3, 2), np.float32)
    n = lib().orc_terrain_patch_domain(C.byref(p), _p(tris), MAX_PATCH_TRIANGLES)
    return tris[:n]


def draw_terrain(heightmap, settings, visible_patches, instance_count, cam, vis, prim_bits=8):
    """the pass into vis (uint64 [H, W], updated in place); returns the triangles emitted"""
    hm = _hm(heightmap)
    st = np.ascontiguousarray(settings)
    vp = np.ascontiguousarray(visible_patches, dtype=np.uint32)
    assert vis.dtype == np.uint64 and vis.flags.c_contiguous
    h, w = vis.shape
    return int(lib().orc_draw_terrain(_p(hm), hm.shape[1], hm.shape[0], _p(st), _p(vp) if vp.size else None, int(instance_count),
                                      _p(np.ascontiguousarray(cam)), int(prim_bits), w, h, _p(vis)))


__all__ = ["build", "lib", "projection_scale", "factor_clamp", "round_odd", "edge_points", "patch", "patch_domain", "draw_terrain",
           "Patch", "MAX_PATCH_TRIANGLES", "pyoracle"]
