"""ctypes wrapper of the GTAO oracle (oracle/oxc_oracle_gtao.c, one translation unit with oxc_oracle_vsm_resolve.c, oxc_oracle.c and
oxc_oracle_vsm.c, built into oracle/liboxc_oracle_gtao.so).  TEST INFRASTRUCTURE ONLY: tests/ and tools/ import it; the product
package never does."""
import ctypes as C
import os

import numpy as np

import pyoracle
from pyoracle import _p
from pyoracle_vsm_resolve import SOURCES as _RESOLVE_SOURCES

_LIB = None
SOURCES = _RESOLVE_SOURCES + ("oxc_oracle_gtao.c", "oxc_oracle_gtao.h")


def build(force=False):
    """compiles liboxc_oracle_gtao.so next to the sources when it is missing or older than them"""
    return pyoracle.build_so("liboxc_oracle_gtao.so", ["oxc_oracle_gtao.c"], SOURCES, force)


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        f, u32, vp = C.c_float, C.c_uint32, C.c_void_p
        _LIB.orc_pow_canonical.restype, _LIB.orc_pow_canonical.argtypes = f, [f, f]
        _LIB.orc_gtao_hilbert_index.restype, _LIB.orc_gtao_hilbert_index.argtypes = u32, [u32, u32]
        _LIB.orc_gtao_noise.argtypes = [u32, u32, u32, vp]
        _LIB.orc_gtao_fast_acos.restype, _LIB.orc_gtao_fast_acos.argtypes = f, [f]
        _LIB.orc_gtao_update_sectors.restype, _LIB.orc_gtao_update_sectors.argtypes = u32, [f, f, u32]
        _LIB.orc_gtao_calc_sector_mask.restype, _LIB.orc_gtao_calc_sector_mask.argtypes = u32, [f, vp, vp, f, f]
        _LIB.orc_gtao_linearize.restype, _LIB.orc_gtao_linearize.argtypes = f, [vp, f]
        _LIB.orc_gtao_weighted_average.restype, _LIB.orc_gtao_weighted_average.argtypes = f, [f, f, f, f]
        _LIB.orc_gtao_mip_offset.restype, _LIB.orc_gtao_mip_offset.argtypes = C.c_uint64, [u32, u32, u32]
        _LIB.orc_gtao_sample_level.restype, _LIB.orc_gtao_sample_level.argtypes = f, [vp, u32, u32, f, f, f]
        _LIB.orc_gtao_denoise_pixel.restype, _LIB.orc_gtao_denoise_pixel.argtypes = f, [vp, vp, u32, u32, u32, u32, f]
        _LIB.orc_generate_ambient_occlusion.argtypes = [vp, vp, vp, vp, u32, u32, vp, vp, vp, vp]
    return _LIB


def generate_ambient_occlusion(gtao_camera, settings, depth, normals):
    """orc_generate_ambient_occlusion over depth [H, W] (D32F) and normals [H, W, 4]: dict(mips= packed float32, edges= uint32 [H, W],
    noisy= uint16 binary16 bits [H, W], ao= float32 [H, W])"""
    d = np.ascontiguousarray(depth, dtype=np.float32)
    n = np.ascontiguousarray(normals, dtype=np.float32)
    h, w = d.shape
    total = int(lib().orc_gtao_mip_offset(w, h, 5))
    mips = np.zeros(total, np.float32)
    edges = np.zeros((h, w), np.uint32)
    noisy = np.zeros((h, w), np.uint16)
    ao = np.zeros((h, w), np.float32)
    lib().orc_generate_ambient_occlusion(C.byref(gtao_camera), C.byref(settings), _p(d), _p(n), w, h, _p(mips), _p(edges), _p(noisy), _p(ao))
    return dict(mips=mips, edges=edges, noisy=noisy, ao=ao)


def pow_canonical(x, y):
    return np.float32(lib().orc_pow_canonical(float(x), float(y)))


def hilbert_index(x, y):
    return int(lib().orc_gtao_hilbert_index(x, y))


def noise(x, y, noise_index=0):
    out = np.zeros(2, np.float32)
    lib().orc_gtao_noise(x, y, noise_index, _p(out))
    return out


def fast_acos(x):
    return np.float32(lib().orc_gtao_fast_acos(float(x)))


def update_sectors(min_horizon, max_horizon, bitmask=0):
    return int(lib().orc_gtao_update_sectors(float(min_horizon), float(max_horizon), bitmask))


def calc_sector_mask(thickness, delta, view_dir, sampling_direction, n):
    return int(lib().orc_gtao_calc_sector_mask(float(thickness), _p(np.ascontiguousarray(delta, dtype=np.float32)),
                                               _p(np.ascontiguousarray(view_dir, dtype=np.float32)), float(sampling_direction), float(n)))


def linearize(projection, device_depth):
    return np.float32(lib().orc_gtao_linearize(_p(np.ascontiguousarray(projection, dtype=np.float32)), float(device_depth)))


def weighted_average(d0, d1, d2, d3):
    return np.float32(lib().orc_gtao_weighted_average(float(d0), float(d1), float(d2), float(d3)))


def mip_offset(w, h, level):
    return int(lib().orc_gtao_mip_offset(w, h, level))


def sample_level(mips, w, h, u, v, lam):
    return np.float32(lib().orc_gtao_sample_level(_p(np.ascontiguousarray(mips, dtype=np.float32)), w, h, float(u), float(v), float(lam)))


def denoise_pixel(noisy, edges, x, y, final_power):
    q = np.ascontiguousarray(noisy, dtype=np.uint16)
    e = np.ascontiguousarray(edges, dtype=np.uint32)
    h, w = q.shape
    return np.float32(lib().orc_gtao_denoise_pixel(_p(q), _p(e), w, h, x, y, float(final_power)))


__all__ = ["build", "lib", "generate_ambient_occlusion", "pow_canonical", "hilbert_index", "noise", "fast_acos", "update_sectors",
           "calc_sector_mask", "linearize", "weighted_average", "mip_offset", "sample_level", "denoise_pixel"]
