"""ctypes wrapper of the sky IBL oracle (oracle/oxc_oracle_sky_ibl.c, one translation unit with oxc_oracle_atmosphere.c and the sources it
includes, built into oracle/liboxc_oracle_sky_ibl.so).  TEST INFRASTRUCTURE ONLY: tests/ and tools/ import it; the product package never
does.  The cube is a float16 array [6, 32, 32, 4]; the LUTs are float16 [H, W, 4]."""
import ctypes as C

import numpy as np

import pyoracle
from pyoracle import _p
from pyoracle_atmosphere import SOURCES as _ATMOSPHERE_SOURCES

_LIB = None
SOURCES = _ATMOSPHERE_SOURCES + ("oxc_oracle_sky_ibl.c", "oxc_oracle_sky_ibl.h")
CUBE_SHAPE = (6, 32, 32, 4)


def build(force=False):
    """compiles liboxc_oracle_sky_ibl.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_sky_ibl.so", ["oxc_oracle_sky_ibl.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        f, u32, u64, vp = C.c_float, C.c_uint32, C.c_uint64, C.c_void_p
        _LIB.orc_atan2_canonical.restype, _LIB.orc_atan2_canonical.argtypes = f, [f, f]
        _LIB.orc_atan2_canonical_array.argtypes = [vp, vp, vp, u64]
        _LIB.orc_acos_canonical_array.argtypes = [vp, vp, u64]
        _LIB.orc_sky_ibl_tap4.argtypes = [vp, u32, u32, f, f, vp]
        _LIB.orc_sky_ibl_dir.argtypes = [u32, u32, u32, vp]
        _LIB.orc_sky_ibl_radical_inverse.restype, _LIB.orc_sky_ibl_radical_inverse.argtypes = f, [u32]
        _LIB.orc_sky_ibl_ign.restype, _LIB.orc_sky_ibl_ign.argtypes = f, [f, f]
        _LIB.orc_sky_ibl_local_sample.argtypes = [u32, f, vp]
        _LIB.orc_sky_ibl_illuminance.argtypes = [vp, f, vp, vp, vp, vp]
        _LIB.orc_atmosphere_sky_ibl.argtypes = [vp, vp, vp, f, f, u32, vp, vp, vp]
    return _LIB


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def atan2(y, x):
    """orc_atan2_canonical elementwise (float32 in, float32 out)"""
    y, x = np.broadcast_arrays(_f32(y), _f32(x))
    y, x = _f32(y), _f32(x)
    out = np.empty_like(y)
    lib().orc_atan2_canonical_array(_p(y), _p(x), _p(out), y.size)
    return out


def acos(x):
    x = _f32(x)
    out = np.empty_like(x)
    lib().orc_acos_canonical_array(_p(x), _p(out), x.size)
    return out


def tap4(lut, u, v):
    """the linear-clamp tap (rgba) of a float16 [H, W, 4] plane"""
    t = np.ascontiguousarray(lut, dtype=np.float16)
    out = np.zeros(4, np.float32)
    lib().orc_sky_ibl_tap4(_p(t), t.shape[1], t.shape[0], float(u), float(v), _p(out))
    return out


def direction(face, x, y):
    out = np.zeros(3, np.float32)
    lib().orc_sky_ibl_dir(face, x, y, _p(out))
    return out


def radical_inverse(i):
    return np.float32(lib().orc_sky_ibl_radical_inverse(i))


def ign(px, py):
    return np.float32(lib().orc_sky_ibl_ign(float(px), float(py)))


def local_sample(i, rotation):
    out = np.zeros(3, np.float32)
    lib().orc_sky_ibl_local_sample(i, float(rotation), _p(out))
    return out


def illuminance(atmosphere, camera_y, sun_direction, sky_view, eye_dir):
    """get_atmosphere_illuminance_along_ray over a float16 sky-view LUT at atmosphere.sky_view_lut_size"""
    sv = np.ascontiguousarray(sky_view, dtype=np.float16)
    assert sv.shape == (atmosphere.sky_view_lut_size[1], atmosphere.sky_view_lut_size[0], 4)
    out = np.zeros(3, np.float32)
    lib().orc_sky_ibl_illuminance(C.byref(atmosphere), float(camera_y), _p(_f32(sun_direction)), _p(sv), _p(_f32(eye_dir)), _p(out))
    return out


def sky_ibl(atmosphere, camera, sun_direction, sun_intensity, sun_ambient_strength, frame_index, transmittance_lut, sky_view_lut, cube=None):
    """orc_atmosphere_sky_ibl: the next cube (float16 [6, 32, 32, 4]) from `cube` (zeros when None), which is not modified"""
    t = np.ascontiguousarray(transmittance_lut, dtype=np.float16)
    sv = np.ascontiguousarray(sky_view_lut, dtype=np.float16)
    assert t.shape == (atmosphere.transmittance_lut_size[1], atmosphere.transmittance_lut_size[0], 4)
    assert sv.shape == (atmosphere.sky_view_lut_size[1], atmosphere.sky_view_lut_size[0], 4)
    out = np.zeros(CUBE_SHAPE, np.float16) if cube is None else np.array(cube, dtype=np.float16, copy=True).reshape(CUBE_SHAPE)
    lib().orc_atmosphere_sky_ibl(C.byref(atmosphere), C.byref(camera), _p(_f32(sun_direction)), float(np.float32(sun_intensity)),
                                 float(np.float32(sun_ambient_strength)), int(frame_index), _p(t), _p(sv), _p(out))
    return out


__all__ = ["build", "lib", "atan2", "acos", "tap4", "direction", "radical_inverse", "ign", "local_sample", "illuminance", "sky_ibl",
           "CUBE_SHAPE"]
