"""ctypes wrapper of the tonemap oracle (oracle/oxc_oracle_tonemap.c, one translation unit with oxc_oracle_post.c and the sources it
includes, built into oracle/liboxc_oracle_tonemap.so).  TEST INFRASTRUCTURE ONLY: tests/ and tools/ import it; the product package
never does.  Frames and the bloom image are float32 [H, W, 4]."""
import ctypes as C

import numpy as np

import pyoracle
from pyoracle import _p
from pyoracle_post import SOURCES as _POST_SOURCES

_LIB = None
SOURCES = _POST_SOURCES + ("oxc_oracle_tonemap.c", "oxc_oracle_tonemap.h")
CONSTANTS = 33  # ORC_TM_CONSTANTS
# item 9's table, by name: (first index, count)
CONSTANT_NAMES = {"agx": (0, 9), "agx_inv": (9, 9), "agx_s": (18, 1), "agx_c": (19, 1), "agx_peak_s": (20, 1), "gt7_ka": (21, 1),
                  "gt7_kb": (22, 1), "gt7_kc": (23, 1), "gt7_linear_peak": (24, 1), "gt7_target": (25, 1), "gt7_target_ucs": (26, 1),
                  "gt7_sdr": (27, 1), "gt7_one_minus_blend": (28, 1), "pq_inv_m1": (29, 1), "pq_inv_m2": (30, 1), "simplex_f2": (31, 1),
                  "simplex_g2": (32, 1)}


def build(force=False):
    """compiles liboxc_oracle_tonemap.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_tonemap.so", ["oxc_oracle_tonemap.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        from oxylus_b200 import abi

        _LIB = C.CDLL(build())
        f, u32, vp = C.c_float, C.c_uint32, C.c_void_p
        _LIB.orc_tonemap_constants.argtypes = [vp]
        _LIB.orc_tonemap_rg_mag.argtypes = [f, vp]
        _LIB.orc_tonemap_curve.argtypes = [u32, vp, vp]
        _LIB.orc_tonemap_gt7_rec2020.argtypes = [vp, vp]
        _LIB.orc_tonemap_tap.argtypes = [vp, u32, u32, f, f, vp]
        _LIB.orc_tonemap.argtypes = [vp, u32, u32, C.POINTER(abi.TonemapSettings), C.POINTER(abi.Exposure), vp, vp]
    return _LIB


def _plane(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.ndim == 3 and a.shape[2] == 4
    return a


def constants():
    """item 9's table, float32 [CONSTANTS]"""
    out = np.zeros(CONSTANTS, np.float32)
    lib().orc_tonemap_constants(_p(out))
    return out


def rg_mag(amount):
    out = np.zeros(2, np.float32)
    lib().orc_tonemap_rg_mag(float(np.float32(amount)), _p(out))
    return out


def curve(tonemap_type, rgb):
    """item 3 on float32 [..., 3] colours (a loop over them)"""
    a = np.ascontiguousarray(rgb, dtype=np.float32).reshape(-1, 3)
    out = np.zeros_like(a)
    for i in range(len(a)):
        lib().orc_tonemap_curve(int(tonemap_type), _p(a[i]), _p(out[i]))
    return out.reshape(np.shape(rgb))


def gt7_rec2020(rgb):
    a = np.ascontiguousarray(rgb, dtype=np.float32).reshape(-1, 3)
    out = np.zeros_like(a)
    for i in range(len(a)):
        lib().orc_tonemap_gt7_rec2020(_p(a[i]), _p(out[i]))
    return out.reshape(np.shape(rgb))


def tap(plane, u, v):
    a = _plane(plane)
    out = np.zeros(4, np.float32)
    lib().orc_tonemap_tap(_p(a), a.shape[1], a.shape[0], float(np.float32(u)), float(np.float32(v)), _p(out))
    return out


def tonemap(frame, settings, record=None, bloom=None):
    """float32 [H, W, 4]; record (abi.Exposure) is read under HasEyeAdaptation, bloom (float32 [H // 2, W // 2, 4]) under HasBloom"""
    from oxylus_b200 import abi

    a = _plane(frame)
    h, w = a.shape[:2]
    out = np.zeros_like(a)
    rec = record if record is not None else abi.Exposure(1.0, 1.0)
    b = _plane(bloom) if bloom is not None else np.zeros((max(h // 2, 1), max(w // 2, 1), 4), np.float32)
    if settings.scene_flags & abi.SCENE_HAS_BLOOM:
        assert b.shape == (h // 2, w // 2, 4)
    lib().orc_tonemap(_p(a), w, h, C.byref(settings), C.byref(rec), _p(b), _p(out))
    return out


__all__ = ["build", "lib", "constants", "rg_mag", "curve", "gt7_rec2020", "tap", "tonemap", "CONSTANTS", "CONSTANT_NAMES"]
