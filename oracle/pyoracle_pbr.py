"""ctypes wrapper of the PBR apply oracle (oracle/oxc_oracle_pbr.c, one translation unit with oxc_oracle_gtao.c and the sources it
includes, built into oracle/liboxc_oracle_pbr.so).  TEST INFRASTRUCTURE ONLY: tests/ and tools/ import it; the product package never
does."""
import ctypes as C

import numpy as np

import pyoracle
from pyoracle import _p
from pyoracle_gtao import SOURCES as _GTAO_SOURCES

_LIB = None
SOURCES = _GTAO_SOURCES + ("oxc_oracle_pbr.c", "oxc_oracle_pbr.h")


def build(force=False):
    """compiles liboxc_oracle_pbr.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_pbr.so", ["oxc_oracle_pbr.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        f, u32, vp = C.c_float, C.c_uint32, C.c_void_p
        _LIB.orc_pow5_canonical.restype, _LIB.orc_pow5_canonical.argtypes = f, [f]
        _LIB.orc_pow5_canonical_n.argtypes = [vp, vp, C.c_uint64]
        _LIB.orc_pbr_ggx_directional_albedo.argtypes = [f, f, vp]
        _LIB.orc_pbr_attenuate_point.restype, _LIB.orc_pbr_attenuate_point.argtypes = f, [f, f]
        _LIB.orc_pbr_spot_attenuation.restype, _LIB.orc_pbr_spot_attenuation.argtypes = f, [vp, vp, f, f]
        _LIB.orc_pbr_smoothstep.restype, _LIB.orc_pbr_smoothstep.argtypes = f, [f, f, f]
        _LIB.orc_pbr_oct_to_vec3.argtypes = [f, f, vp]
        _LIB.orc_apply_pbr.argtypes = [vp] * 11 + [u32, u32, vp]
        _LIB.orc_pow_canonical.restype, _LIB.orc_pow_canonical.argtypes = f, [f, f]
    return _LIB


def _plane(a, comps):
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.shape[-1] == comps if comps > 1 else a.ndim == 2, a.shape
    return a


def apply_pbr(camera, settings, lights, depth, albedo, normal, emissive, mro, ao=None, shadow=None, contact=None):
    """orc_apply_pbr: camera abi.PbrCamera, settings abi.PbrSettings, lights an abi.Light array (or None), depth [H, W], the four
    float4 planes [H, W, 4], ao / shadow / contact [H, W] or None -> float32 [H, W, 4]"""
    d = _plane(depth, 1)
    h, w = d.shape
    planes = [_plane(albedo, 4), _plane(normal, 4), _plane(emissive, 4), _plane(mro, 4), _plane(ao, 1), _plane(shadow, 1), _plane(contact, 1)]
    out = np.zeros((h, w, 4), np.float32)
    lp = C.cast(lights, C.c_void_p) if lights is not None and len(lights) else None
    lib().orc_apply_pbr(C.byref(camera), C.byref(settings), lp, _p(d), *[_p(p) if p is not None else None for p in planes], w, h, _p(out))
    return out


def pow5(x):
    """orc_pow5_canonical over an array of binary32 values"""
    a = np.ascontiguousarray(x, dtype=np.float32).reshape(-1)
    out = np.empty_like(a)
    lib().orc_pow5_canonical_n(_p(a), _p(out), a.size)
    return out.reshape(np.shape(x))


def pow_canonical(x, y):
    return np.float32(lib().orc_pow_canonical(float(x), float(y)))


def ggx_directional_albedo(NoV, alpha):
    out = np.zeros(2, np.float32)
    lib().orc_pbr_ggx_directional_albedo(float(NoV), float(alpha), _p(out))
    return out


def attenuate_point(dist, cutoff):
    return np.float32(lib().orc_pbr_attenuate_point(float(dist), float(cutoff)))


def spot_attenuation(L, spot_direction, inner, outer):
    return np.float32(lib().orc_pbr_spot_attenuation(_p(np.ascontiguousarray(L, dtype=np.float32)), _p(np.ascontiguousarray(spot_direction, dtype=np.float32)),
                                                     float(inner), float(outer)))


def smoothstep(e0, e1, x):
    return np.float32(lib().orc_pbr_smoothstep(float(e0), float(e1), float(x)))


def oct_to_vec3(ex, ey):
    out = np.zeros(3, np.float32)
    lib().orc_pbr_oct_to_vec3(float(ex), float(ey), _p(out))
    return out


__all__ = ["build", "lib", "apply_pbr", "pow5", "pow_canonical", "ggx_directional_albedo", "attenuate_point", "spot_attenuation", "smoothstep",
           "oct_to_vec3"]
