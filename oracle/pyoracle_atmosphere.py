"""ctypes wrapper of the atmosphere oracle (oracle/oxc_oracle_atmosphere.c, one translation unit with oxc_oracle_gtao.c and the sources it
includes, built into oracle/liboxc_oracle_atmosphere.so).  TEST INFRASTRUCTURE ONLY: tests/ and tools/ import it; the product package
never does.  The LUTs are float16 arrays [H, W, 4] (transmittance, sky view) and [D, H, W, 4] (aerial perspective)."""
import ctypes as C

import numpy as np

import pyoracle
from pyoracle import _p
from pyoracle_gtao import SOURCES as _GTAO_SOURCES

_LIB = None
SOURCES = _GTAO_SOURCES + ("oxc_oracle_atmosphere.c", "oxc_oracle_atmosphere.h")


def build(force=False):
    """compiles liboxc_oracle_atmosphere.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_atmosphere.so", ["oxc_oracle_atmosphere.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        f, u32, u64, vp = C.c_float, C.c_uint32, C.c_uint64, C.c_void_p
        _LIB.orc_exp_canonical.restype, _LIB.orc_exp_canonical.argtypes = f, [f]
        _LIB.orc_exp_canonical_array.argtypes = [vp, vp, u64]
        _LIB.orc_acos_canonical.restype, _LIB.orc_acos_canonical.argtypes = f, [f]
        _LIB.orc_acos_canonical_array.argtypes = [vp, vp, u64]
        _LIB.orc_atm_half.restype, _LIB.orc_atm_half.argtypes = C.c_uint16, [f]
        _LIB.orc_atm_ray_sphere_nearest.restype, _LIB.orc_atm_ray_sphere_nearest.argtypes = C.c_int, [vp, vp, f, vp]
        _LIB.orc_atm_transmittance_uv.argtypes = [f, f, f, f, vp]
        _LIB.orc_atm_rayleigh_phase.restype, _LIB.orc_atm_rayleigh_phase.argtypes = f, [f]
        _LIB.orc_atm_hg_draine_constants.argtypes = [f, vp]
        _LIB.orc_atm_mie_phase.restype, _LIB.orc_atm_mie_phase.argtypes = f, [f, f]
        _LIB.orc_atm_medium_extinction.argtypes = [vp, f, vp]
        _LIB.orc_atm_tap.argtypes = [vp, u32, u32, f, f, vp]
        _LIB.orc_atm_eye_y.restype, _LIB.orc_atm_eye_y.argtypes = f, [vp, f]
        _LIB.orc_atm_sky_view_dir.argtypes = [vp, f, f, f, vp]
        _LIB.orc_atm_transmittance_params.argtypes = [vp, u32, u32, vp]
        _LIB.orc_atm_transmittance_ray.argtypes = [vp, f, f, vp]
        _LIB.orc_atmosphere_transmittance.argtypes = [vp, vp]
        _LIB.orc_atmosphere_sky_view.argtypes = [vp, vp, vp, f, vp, vp]
        _LIB.orc_atmosphere_aerial_perspective.argtypes = [vp, vp, vp, f, vp, vp]
    return _LIB


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def exp(x):
    """orc_exp_canonical elementwise (float32 in, float32 out)"""
    x = _f32(x)
    out = np.empty_like(x)
    lib().orc_exp_canonical_array(_p(x), _p(out), x.size)
    return out


def acos(x):
    x = _f32(x)
    out = np.empty_like(x)
    lib().orc_acos_canonical_array(_p(x), _p(out), x.size)
    return out


def half(x):
    return int(lib().orc_atm_half(float(x)))


def ray_sphere_nearest(origin, direction, radius):
    """the distance, or None for `none`"""
    o, d, t = _f32(origin), _f32(direction), np.zeros(1, np.float32)
    return t[0] if lib().orc_atm_ray_sphere_nearest(_p(o), _p(d), float(radius), _p(t)) else None


def transmittance_uv(atmos_radius, planet_radius, h, cos_theta):
    out = np.zeros(2, np.float32)
    lib().orc_atm_transmittance_uv(float(atmos_radius), float(planet_radius), float(h), float(cos_theta), _p(out))
    return out


def hg_draine_constants(g):
    out = np.zeros(4, np.float32)
    lib().orc_atm_hg_draine_constants(float(g), _p(out))
    return out


def mie_phase(g, cos_theta):
    return np.float32(lib().orc_atm_mie_phase(float(g), float(cos_theta)))


def rayleigh_phase(cos_theta):
    return np.float32(lib().orc_atm_rayleigh_phase(float(cos_theta)))


def medium_extinction(atmosphere, altitude):
    out = np.zeros(3, np.float32)
    lib().orc_atm_medium_extinction(C.byref(atmosphere), float(altitude), _p(out))
    return out


def tap(lut, u, v):
    """the linear-clamp tap (rgb) of a float16 [H, W, 4] LUT"""
    t = np.ascontiguousarray(lut, dtype=np.float16)
    out = np.zeros(3, np.float32)
    lib().orc_atm_tap(_p(t), t.shape[1], t.shape[0], float(u), float(v), _p(out))
    return out


def eye_y(atmosphere, camera_y):
    return np.float32(lib().orc_atm_eye_y(C.byref(atmosphere), float(camera_y)))


def sky_view_dir(atmosphere, u, v, altitude):
    out = np.zeros(3, np.float32)
    lib().orc_atm_sky_view_dir(C.byref(atmosphere), float(u), float(v), float(altitude), _p(out))
    return out


def transmittance_params(atmosphere, x, y):
    """the bake's (height, cos theta) of texel (x, y)"""
    out = np.zeros(2, np.float32)
    lib().orc_atm_transmittance_params(C.byref(atmosphere), x, y, _p(out))
    return out


def transmittance_ray(atmosphere, height, cos_theta):
    """exp(-optical depth) of the bake's 1000-step march from (height, cos theta), binary32"""
    out = np.zeros(3, np.float32)
    lib().orc_atm_transmittance_ray(C.byref(atmosphere), float(height), float(cos_theta), _p(out))
    return out


def transmittance(atmosphere):
    """orc_atmosphere_transmittance -> float16 [H, W, 4] at atmosphere.transmittance_lut_size"""
    w, h = atmosphere.transmittance_lut_size[0], atmosphere.transmittance_lut_size[1]
    out = np.zeros((h, w, 4), np.float16)
    lib().orc_atmosphere_transmittance(C.byref(atmosphere), _p(out))
    return out


def sky_luts(atmosphere, camera, sun_direction, sun_intensity, transmittance_lut):
    """(sky view float16 [H, W, 4], aerial perspective float16 [D, H, W, 4]) of the per-frame passes over transmittance_lut"""
    t = np.ascontiguousarray(transmittance_lut, dtype=np.float16)
    assert t.shape == (atmosphere.transmittance_lut_size[1], atmosphere.transmittance_lut_size[0], 4)
    sun = _f32(sun_direction)
    sv = np.zeros((atmosphere.sky_view_lut_size[1], atmosphere.sky_view_lut_size[0], 4), np.float16)
    ap = np.zeros((atmosphere.aerial_perspective_lut_size[2], atmosphere.aerial_perspective_lut_size[1],
                   atmosphere.aerial_perspective_lut_size[0], 4), np.float16)
    lib().orc_atmosphere_sky_view(C.byref(atmosphere), C.byref(camera), _p(sun), float(sun_intensity), _p(t), _p(sv))
    lib().orc_atmosphere_aerial_perspective(C.byref(atmosphere), C.byref(camera), _p(sun), float(sun_intensity), _p(t), _p(ap))
    return sv, ap


__all__ = ["build", "lib", "exp", "acos", "half", "ray_sphere_nearest", "transmittance_uv", "hg_draine_constants", "mie_phase",
           "rayleigh_phase", "medium_extinction", "tap", "transmittance_params", "transmittance_ray", "eye_y", "sky_view_dir", "transmittance", "sky_luts"]
