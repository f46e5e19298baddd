"""ctypes wrapper of the atmospheric PBR apply oracle (oracle/oxc_oracle_pbr_atmosphere.c, one translation unit with the PBR and sky IBL
oracles and the sources they include, built into oracle/liboxc_oracle_pbr_atmosphere.so).  TEST INFRASTRUCTURE ONLY: tests/ and tools/
import it; the product package never does.  LUTs are float16 [H, W, 4] (the aerial perspective [D, H, W, 4]), the cube [6, 32, 32, 4]."""
import ctypes as C

import numpy as np

import pyoracle
from pyoracle import _p
from pyoracle_pbr import SOURCES as _PBR_SOURCES
from pyoracle_pbr import _plane
from pyoracle_sky_ibl import SOURCES as _SKY_IBL_SOURCES

_LIB = None
SOURCES = tuple(dict.fromkeys(_PBR_SOURCES + _SKY_IBL_SOURCES + ("oxc_oracle_pbr_atmosphere.c", "oxc_oracle_pbr_atmosphere.h")))


def build(force=False):
    """compiles liboxc_oracle_pbr_atmosphere.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_pbr_atmosphere.so", ["oxc_oracle_pbr_atmosphere.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        f, u32, i32, vp = C.c_float, C.c_uint32, C.c_int32, C.c_void_p
        _LIB.orc_pbra_constants.argtypes = [vp]
        _LIB.orc_pbra_draw_sun.restype, _LIB.orc_pbra_draw_sun.argtypes = f, [f]
        _LIB.orc_pbra_cube_face.restype, _LIB.orc_pbra_cube_face.argtypes = C.c_int, [vp, vp]
        _LIB.orc_pbra_cube_remap.restype, _LIB.orc_pbra_cube_remap.argtypes = u32, [u32, i32, i32]
        _LIB.orc_pbra_cube_tap.argtypes = [vp, vp, vp]
        _LIB.orc_pbra_tap3.argtypes = [vp, vp, f, f, f, vp]
        _LIB.orc_pbra_aerial.argtypes = [vp, vp, f, f, vp, vp]
        _LIB.orc_apply_pbr_atmosphere.argtypes = [vp] * 13 + [u32, u32, vp]
    return _LIB


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _h(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float16)
    assert shape is None or a.shape == tuple(shape), (a.shape, shape)
    return a


def pass_constants():
    """the constants the pass reads, float32: (radius * PI / 180, min_cos, half_slice_depth, near_depth_fade_out)"""
    out = np.zeros(4, np.float32)
    lib().orc_pbra_constants(_p(out))
    return out


def draw_sun(cos_theta):
    return np.float32(lib().orc_pbra_draw_sun(float(np.float32(cos_theta))))


def cube_face(r):
    """(face, [sc, tc, ma])"""
    o = np.zeros(3, np.float32)
    return lib().orc_pbra_cube_face(_p(_f32(r)), _p(o)), o


def cube_remap(face, i, j):
    """the texel index (face * 32 + y) * 32 + x that texel (i, j) of `face` (one coordinate off the face) reads"""
    return int(lib().orc_pbra_cube_remap(face, i, j))


def cube_tap(cube, r):
    c = _h(cube, (6, 32, 32, 4))
    out = np.zeros(4, np.float32)
    lib().orc_pbra_cube_tap(_p(c), _p(_f32(r)), _p(out))
    return out


def _ap_shape(atmosphere):
    s = atmosphere.aerial_perspective_lut_size
    return (s[2], s[1], s[0], 4)


def tap3(atmosphere, lut, u, v, w):
    t = _h(lut, _ap_shape(atmosphere))
    out = np.zeros(4, np.float32)
    lib().orc_pbra_tap3(C.byref(atmosphere), _p(t), float(np.float32(u)), float(np.float32(v)), float(np.float32(w)), _p(out))
    return out


def aerial(atmosphere, lut, u, v, d):
    t = _h(lut, _ap_shape(atmosphere))
    out = np.zeros(4, np.float32)
    lib().orc_pbra_aerial(C.byref(atmosphere), _p(t), float(np.float32(u)), float(np.float32(v)), _p(_f32(d)), _p(out))
    return out


def apply_pbr_atmosphere(camera, settings, atmosphere, lights, depth, albedo, normal, emissive, mro, ao, shadow, contact, transmittance, sky_view,
                         aerial_perspective, cube):
    """orc_apply_pbr_atmosphere: apply_pbr's arguments plus the record and the four sky planes (float16) -> float32 [H, W, 4]"""
    d = _plane(depth, 1)
    h, w = d.shape
    planes = [_plane(albedo, 4), _plane(normal, 4), _plane(emissive, 4), _plane(mro, 4), _plane(ao, 1), _plane(shadow, 1), _plane(contact, 1)]
    a = atmosphere
    sky = [_h(transmittance, (a.transmittance_lut_size[1], a.transmittance_lut_size[0], 4)),
           _h(sky_view, (a.sky_view_lut_size[1], a.sky_view_lut_size[0], 4)), _h(aerial_perspective, _ap_shape(a)), _h(cube, (6, 32, 32, 4))]

    class Sky(C.Structure):
        _fields_ = [(n, C.c_void_p) for n in ("transmittance", "sky_view", "aerial_perspective", "sky_cube")]

    k = Sky(*[s.ctypes.data for s in sky])
    out = np.zeros((h, w, 4), np.float32)
    lp = C.cast(lights, C.c_void_p) if lights is not None and len(lights) else None
    lib().orc_apply_pbr_atmosphere(C.byref(camera), C.byref(settings), C.byref(atmosphere), lp, _p(d),
                                   *[_p(p) if p is not None else None for p in planes], C.byref(k), w, h, _p(out))
    return out


__all__ = ["build", "lib", "pass_constants", "draw_sun", "cube_face", "cube_remap", "cube_tap", "tap3", "aerial", "apply_pbr_atmosphere"]
