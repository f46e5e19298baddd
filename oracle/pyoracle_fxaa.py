"""ctypes wrapper of the FXAA oracle (oracle/oxc_oracle_fxaa.c, one translation unit with oxc_oracle_post.c and the sources it includes,
built into oracle/liboxc_oracle_fxaa.so).  TEST INFRASTRUCTURE ONLY: tests/ and tools/ import it; the product package never does.  Frames
are float32 [H, W, 4]."""
import ctypes as C

import numpy as np

import pyoracle
from pyoracle import _p
from pyoracle_post import SOURCES as _POST_SOURCES

_LIB = None
SOURCES = _POST_SOURCES + ("oxc_oracle_fxaa.c", "oxc_oracle_fxaa.h")
CONSTANTS = 4  # ORC_FXAA_CONSTANTS: EDGE_THRESHOLD_MIN, EDGE_THRESHOLD_MAX, SUBPIXEL_QUALITY, 1.0 / 12.0
EARLY_EXIT_TAPS, MAX_TAPS = 5, 32


def build(force=False):
    """compiles liboxc_oracle_fxaa.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_fxaa.so", ["oxc_oracle_fxaa.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        f, u32, i32, vp = C.c_float, C.c_uint32, C.c_int32, C.c_void_p
        _LIB.orc_fxaa_constants.argtypes = [vp]
        _LIB.orc_fxaa_quality.restype, _LIB.orc_fxaa_quality.argtypes = f, [i32]
        _LIB.orc_fxaa_luma.restype, _LIB.orc_fxaa_luma.argtypes = f, [vp]
        _LIB.orc_fxaa_tap.argtypes = [vp, u32, u32, f, f, i32, i32, vp]
        _LIB.orc_fxaa.argtypes = [vp, u32, u32, vp, vp]
    return _LIB


def _plane(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.ndim == 3 and a.shape[2] == 4
    return a


def constants():
    out = np.zeros(CONSTANTS, np.float32)
    lib().orc_fxaa_constants(_p(out))
    return out


def quality(i):
    return lib().orc_fxaa_quality(int(i))


def luma(rgb):
    a = np.ascontiguousarray(rgb, dtype=np.float32)
    return np.float32(lib().orc_fxaa_luma(_p(a)))


def tap(plane, u, v, dx=0, dy=0):
    a = _plane(plane)
    out = np.zeros(4, np.float32)
    lib().orc_fxaa_tap(_p(a), a.shape[1], a.shape[0], float(np.float32(u)), float(np.float32(v)), int(dx), int(dy), _p(out))
    return out


def fxaa(frame, with_taps=False):
    """float32 [H, W, 4] -> float32 [H, W, 4]; with_taps also returns each pixel's bilinear tap count (uint8 [H, W])"""
    a = _plane(frame)
    h, w = a.shape[:2]
    out = np.zeros_like(a)
    taps = np.zeros((h, w), np.uint8)
    lib().orc_fxaa(_p(a), w, h, _p(out), _p(taps))
    return (out, taps) if with_taps else out


__all__ = ["build", "lib", "constants", "quality", "luma", "tap", "fxaa", "CONSTANTS", "EARLY_EXIT_TAPS", "MAX_TAPS"]
