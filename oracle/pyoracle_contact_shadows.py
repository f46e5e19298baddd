"""ctypes wrapper of the contact-shadow oracle (oracle/oxc_oracle_contact_shadows.c, one translation unit with oxc_oracle_pbr.c and the
sources it includes, built into oracle/liboxc_oracle_contact_shadows.so).  TEST INFRASTRUCTURE ONLY: tests/ and tools/ import it; the
product package never does."""
import ctypes as C

import numpy as np

import pyoracle
from pyoracle import _p
from pyoracle_pbr import SOURCES as _PBR_SOURCES

_LIB = None
SOURCES = _PBR_SOURCES + ("oxc_oracle_contact_shadows.c", "oxc_oracle_contact_shadows.h")


def build(force=False):
    """compiles liboxc_oracle_contact_shadows.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_contact_shadows.so", ["oxc_oracle_contact_shadows.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        f, u32, vp = C.c_float, C.c_uint32, C.c_void_p
        _LIB.orc_cs_bias_factor.restype, _LIB.orc_cs_bias_factor.argtypes = f, []
        _LIB.orc_cs_nearest.restype, _LIB.orc_cs_nearest.argtypes = f, [vp, u32, u32, f, f]
        _LIB.orc_cs_bilinear.restype, _LIB.orc_cs_bilinear.argtypes = f, [vp, u32, u32, f, f]
        _LIB.orc_cs_clip_ray.argtypes = [vp, vp, vp]
        _LIB.orc_cs_step_count.restype, _LIB.orc_cs_step_count.argtypes = u32, [vp, u32, u32, u32]
        _LIB.orc_cs_pixel.restype, _LIB.orc_cs_pixel.argtypes = f, [vp, vp, vp, u32, u32, u32, u32, vp]
        _LIB.orc_contact_shadows.argtypes = [vp, vp, vp, u32, u32, vp]
        _LIB.orc_pbr_smoothstep.restype, _LIB.orc_pbr_smoothstep.argtypes = f, [f, f, f]
    return _LIB


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def contact_shadows(camera, settings, depth):
    """orc_contact_shadows: camera abi.ContactShadowCamera, settings abi.ContactShadowSettings, depth [H, W] -> float32 [H, W]"""
    d = _f32(depth)
    h, w = d.shape
    out = np.zeros((h, w), np.float32)
    lib().orc_contact_shadows(C.byref(camera), C.byref(settings), _p(d), w, h, _p(out))
    return out


def pixel(camera, settings, depth, x, y):
    """orc_cs_pixel: (1 - shadow, step count, hit step or -1, in contact) of pixel (x, y)"""
    d = _f32(depth)
    h, w = d.shape
    m = np.zeros(3, np.int32)
    v = lib().orc_cs_pixel(C.byref(camera), C.byref(settings), _p(d), w, h, x, y, _p(m))
    return np.float32(v), int(m[0]), int(m[1]), bool(m[2])


def bias_factor():
    return np.float32(lib().orc_cs_bias_factor())


def nearest(depth, u, v):
    d = _f32(depth)
    h, w = d.shape
    return np.float32(lib().orc_cs_nearest(_p(d), w, h, float(u), float(v)))


def bilinear(depth, u, v):
    d = _f32(depth)
    h, w = d.shape
    return np.float32(lib().orc_cs_bilinear(_p(d), w, h, float(u), float(v)))


def clip_ray(start_cs, end_cs):
    """the clipped ray (start[3], end[3]) of to_cs(end_cs) from start_cs"""
    out = np.zeros(6, np.float32)
    s, e = _f32(start_cs), _f32(end_cs)
    lib().orc_cs_clip_ray(_p(s), _p(e), _p(out))
    return out[:3], out[3:]


def step_count(start, end, w, h, steps):
    ray = _f32(np.concatenate([np.asarray(start, np.float32), np.asarray(end, np.float32)]))
    return int(lib().orc_cs_step_count(_p(ray), w, h, steps))


def smoothstep(e0, e1, x):
    return np.float32(lib().orc_pbr_smoothstep(float(e0), float(e1), float(x)))


__all__ = ["build", "lib", "contact_shadows", "pixel", "bias_factor", "nearest", "bilinear", "clip_ray", "step_count", "smoothstep"]
