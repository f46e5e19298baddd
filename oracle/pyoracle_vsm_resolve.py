"""ctypes wrapper of the VSM shadow-resolve oracle (oracle/oxc_oracle_vsm_resolve.c, one translation unit with oxc_oracle.c and
oxc_oracle_vsm.c, built into oracle/liboxc_oracle_vsm_resolve.so).  TEST INFRASTRUCTURE ONLY: tests/ and tools/ import it; the
product package never does."""
import ctypes as C

import numpy as np

import pyoracle
from pyoracle import _p

_LIB = None
SOURCES = ("oxc_oracle.c", "oxc_oracle.h", "oxc_oracle_math.inc", "oxc_oracle_vsm.c", "oxc_oracle_vsm.h", "oxc_oracle_vsm_resolve.c",
           "oxc_oracle_vsm_resolve.h")


def build(force=False):
    """compiles liboxc_oracle_vsm_resolve.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_vsm_resolve.so", ["oxc_oracle_vsm_resolve.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.orc_vsm_resolve_shadows.restype = C.c_uint64
        _LIB.orc_vsm_base_bias.restype = C.c_float
        _LIB.orc_vsm_base_bias.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        _LIB.orc_round_to_half.restype = C.c_float
        _LIB.orc_round_to_half.argtypes = [C.c_float]
        _LIB.orc_vsm_hash2.argtypes = [C.c_float, C.c_float, C.c_void_p]
        _LIB.orc_sincos_canonical.argtypes = [C.c_float, C.c_void_p, C.c_void_p]
        _LIB.orc_sincos_error_scan.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
        _LIB.orc_sincos_error_list.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
    return _LIB


def vsm_resolve_shadows(vsm, inv_pv, resolution, clipmaps, depth, normals, page_tables, atlas):
    """orc_vsm_resolve_shadows: returns (shadow [H, W] float32, pcf [H, W] bool: the pixels that ran the PCF loop)"""
    v = np.ascontiguousarray(vsm)
    w, h = int(v["depth_extent"].reshape(-1)[0]), int(v["depth_extent"].reshape(-1)[1])
    shadow = np.zeros((h, w), np.float32)
    pcf = np.zeros((h, w), np.uint8)
    lib().orc_vsm_resolve_shadows(_p(v), _p(np.ascontiguousarray(inv_pv, dtype=np.float32)), _p(np.ascontiguousarray(resolution, dtype=np.float32)),
                                  _p(np.ascontiguousarray(clipmaps)), _p(np.ascontiguousarray(depth, dtype=np.float32)),
                                  _p(np.ascontiguousarray(normals, dtype=np.float32)), _p(np.ascontiguousarray(page_tables, dtype=np.uint32)),
                                  _p(np.ascontiguousarray(atlas, dtype=np.float32)), _p(shadow), _p(pcf))
    return shadow, pcf.astype(bool)


def sincos(x):
    """orc_sincos_canonical of a binary32 value: (sin, cos) as float32"""
    s, c = C.c_float(), C.c_float()
    lib().orc_sincos_canonical(C.c_float(float(x)), C.byref(s), C.byref(c))
    return np.float32(s.value), np.float32(c.value)


def sincos_error_scan(lo_bits, hi_bits, stride=1):
    """max (abs sin error, abs cos error, sin ulps, cos ulps) against binary64 libm over the binary32 bit patterns lo, lo + stride, ...
    <= hi"""
    out = np.zeros(4, np.float64)
    lib().orc_sincos_error_scan(lo_bits, hi_bits, stride, _p(out))
    return out


def sincos_error_list(x):
    """the same maxima over the given binary32 values"""
    v = np.ascontiguousarray(x, dtype=np.float32)
    out = np.zeros(4, np.float64)
    lib().orc_sincos_error_list(_p(v), v.size, _p(out))
    return out


def hammersley2d(i, n):
    out = np.zeros(2, np.float32)
    lib().orc_hammersley2d(C.c_uint32(i), C.c_uint32(n), _p(out))
    return out


def hash2(px, py):
    out = np.zeros(2, np.float32)
    lib().orc_vsm_hash2(float(px), float(py), _p(out))
    return out


def perpendicular_basis(light):
    out = np.zeros(6, np.float32)
    lib().orc_vsm_perpendicular_basis(_p(np.ascontiguousarray(light, dtype=np.float32)), _p(out))
    return out[:3], out[3:]


def base_bias(vsm, clipmap_index, normal):
    return np.float32(lib().orc_vsm_base_bias(_p(np.ascontiguousarray(vsm)), int(clipmap_index), _p(np.ascontiguousarray(normal, dtype=np.float32))))


def round_to_half(x):
    return np.float32(lib().orc_round_to_half(float(x)))


__all__ = ["build", "lib", "vsm_resolve_shadows", "sincos", "sincos_error_scan", "sincos_error_list", "hammersley2d", "hash2", "perpendicular_basis", "base_bias",
           "round_to_half", "pyoracle"]
