"""ctypes wrapper of the post-processing oracle (oracle/oxc_oracle_post.c, one translation unit with oxc_oracle_atmosphere.c and the sources
it includes, built into oracle/liboxc_oracle_post.so).  TEST INFRASTRUCTURE ONLY: tests/ and tools/ import it; the product package never
does.  Frames are float32 [H, W, 4]; a bloom chain is float32 [texels, 4], its levels packed in order (oxylus_b200.abi.bloom_levels)."""
import ctypes as C

import numpy as np

import pyoracle
from pyoracle import _p
from pyoracle_atmosphere import SOURCES as _ATMOSPHERE_SOURCES

_LIB = None
SOURCES = _ATMOSPHERE_SOURCES + ("oxc_oracle_post.c", "oxc_oracle_post.h")


def build(force=False):
    """compiles liboxc_oracle_post.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_post.so", ["oxc_oracle_post.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        from oxylus_b200 import abi

        _LIB = C.CDLL(build())
        f, u32, vp = C.c_float, C.c_uint32, C.c_void_p
        _LIB.orc_eye_adaptation_constants.argtypes = [C.POINTER(abi.EyeAdaptationSettings), u32, u32, f, vp]
        _LIB.orc_histogram_bin.restype, _LIB.orc_histogram_bin.argtypes = u32, [C.POINTER(abi.EyeAdaptationSettings), f, f, f]
        _LIB.orc_histogram_average.argtypes = [vp, vp, f, C.POINTER(abi.Exposure)]
        _LIB.orc_eye_adaptation.argtypes = [vp, u32, u32, C.POINTER(abi.EyeAdaptationSettings), f, C.POINTER(abi.Exposure), vp]
        _LIB.orc_bloom_level_count.restype, _LIB.orc_bloom_level_count.argtypes = u32, [u32, u32]
        _LIB.orc_bloom_tap.argtypes = [vp, u32, u32, f, f, C.c_int, vp]
        _LIB.orc_bloom.argtypes = [vp, u32, u32, C.POINTER(abi.BloomSettings), C.POINTER(abi.Exposure), vp, vp]
    return _LIB


def _frame(frame):
    a = np.ascontiguousarray(frame, dtype=np.float32)
    assert a.ndim == 3 and a.shape[2] == 4
    return a


def constants(settings, width, height, delta_time):
    """item 1: float32 [pixel_count, exposure_range, time_coeff, bias_scale]"""
    out = np.zeros(4, np.float32)
    lib().orc_eye_adaptation_constants(C.byref(settings), width, height, float(np.float32(delta_time)), _p(out))
    return out


def histogram_bin(settings, r, g, b):
    return int(lib().orc_histogram_bin(C.byref(settings), float(np.float32(r)), float(np.float32(g)), float(np.float32(b))))


def histogram_average(bins, consts, min_exposure, record):
    """item 3: the record (abi.Exposure, not modified) after one frame with u32 bins [256]"""
    from oxylus_b200 import abi

    b = np.ascontiguousarray(bins, dtype=np.uint32)
    assert b.shape == (256,)
    out = abi.Exposure.from_buffer_copy(record)
    lib().orc_histogram_average(_p(b), _p(np.ascontiguousarray(consts, np.float32)), float(np.float32(min_exposure)), C.byref(out))
    return out


def eye_adaptation(frame, settings, delta_time, record):
    """(record after the call, u32 histogram [256]); `record` is not modified"""
    from oxylus_b200 import abi

    a = _frame(frame)
    out, hist = abi.Exposure.from_buffer_copy(record), np.zeros(256, np.uint32)
    lib().orc_eye_adaptation(_p(a), a.shape[1], a.shape[0], C.byref(settings), float(np.float32(delta_time)), C.byref(out), _p(hist))
    return out, hist


def level_count(width, height):
    return int(lib().orc_bloom_level_count(width, height))


def tap(plane, u, v, border):
    """item 1's tap (rgb) of a float32 [H, W, 4] plane"""
    a = _frame(plane)
    out = np.zeros(3, np.float32)
    lib().orc_bloom_tap(_p(a), a.shape[1], a.shape[0], float(np.float32(u)), float(np.float32(v)), int(bool(border)), _p(out))
    return out


def bloom(frame, settings, record=None, upsampled=None):
    """(downsampled, upsampled) chains, float32 [texels, 4].  `upsampled` (copied) is the chain's content before the call, which its
    level n-1 keeps (zeros when None); record: abi.Exposure, read under HasEyeAdaptation"""
    from oxylus_b200 import abi

    a = _frame(frame)
    h, w = a.shape[:2]
    n = abi.bloom_chain_texels(w, h)
    down = np.zeros((n, 4), np.float32)
    up = np.zeros((n, 4), np.float32) if upsampled is None else np.array(upsampled, dtype=np.float32, copy=True).reshape(n, 4)
    rec = record if record is not None else abi.Exposure(1.0, 1.0)
    lib().orc_bloom(_p(a), w, h, C.byref(settings), C.byref(rec), _p(down), _p(up))
    return down, up


__all__ = ["build", "lib", "constants", "histogram_bin", "histogram_average", "eye_adaptation", "level_count", "tap", "bloom"]
