"""ctypes wrapper of the G-buffer decode oracle (oracle/oxc_oracle_gbuffer.c, one translation unit with oxc_oracle.c, built into
oracle/liboxc_oracle_gbuffer.so).  TEST INFRASTRUCTURE ONLY: tests/ and tools/ import it; the product package never does."""
import ctypes as C
import os
import subprocess

import numpy as np

import pyoracle
from pyoracle import _p
from pyoracle_vsm import CFLAGS

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
SOURCES = ("oxc_oracle.c", "oxc_oracle.h", "oxc_oracle_math.inc", "oxc_oracle_gbuffer.c", "oxc_oracle_gbuffer.h")
PLANES = ("albedo", "normal", "emissive", "metallic_roughness_occlusion")


def build(force=False):
    """compiles liboxc_oracle_gbuffer.so next to the sources when it is missing or older than them"""
    so = os.path.join(_HERE, "liboxc_oracle_gbuffer.so")
    srcs = [os.path.join(_HERE, f) for f in SOURCES] + [os.path.join(os.path.dirname(_HERE), "include", "oxcull.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        tmp = so + f".{os.getpid()}.tmp"
        subprocess.check_call([os.environ.get("CC", "gcc")] + CFLAGS + ["-shared", "-o", tmp, os.path.join(_HERE, "oxc_oracle_gbuffer.c"), "-lm", "-lpthread"])
        os.replace(tmp, so)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.orc_decode_gbuffer.restype = C.c_uint64
        _LIB.orc_gbuffer_shade.restype = C.c_int
        _LIB.orc_gbuffer_texel_fetches.restype = C.c_uint64
        _LIB.orc_gbuffer_texel_fetches.argtypes = [C.c_int]
        _LIB.orc_gbuffer_sample_level.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_float, C.c_float, C.c_void_p]
        _LIB.orc_gbuffer_sample_grad.argtypes = [C.c_void_p, C.c_void_p] + [C.c_float] * 6 + [C.c_void_p]
    return _LIB


def texel_fetches(reset=True):
    """texel fetches of the oracle's sampling since the last reset (the device reads one aligned 32-bit word per fetch)"""
    return int(lib().orc_gbuffer_texel_fetches(int(reset)))


def srgb_table():
    out = np.zeros(256, np.float32)
    lib().orc_srgb_table(_p(out))
    return out


def decode_gbuffer(hs, mi, total, cam, vis32, table, planes=PLANES, init=None):
    """orc_decode_gbuffer: dict plane -> float32 [H, W, 4] for the requested planes (discarded pixels keep `init`, default 0) and the
    number of decoded pixels whose material lies outside the table"""
    v = np.ascontiguousarray(vis32, dtype=np.uint32)
    h, w = v.shape
    out = {k: np.full((h, w, 4), 0.0 if init is None else init, np.float32) for k in planes}
    bad = lib().orc_decode_gbuffer(hs.ref, _p(mi), C.c_uint32(total), _p(cam), _p(v), C.c_uint32(w), C.c_uint32(h), C.byref(table.ref),
                                   *[_p(out.get(k)) for k in PLANES])
    return out, int(bad)


def decode_pixels(hs, mi, total, cam, vis32):
    """orc_decode_gbuffer_pixels: (records float32 [H, W, 24], material int32 [H, W]: -1 discarded, -2 vertex index out of range)"""
    v = np.ascontiguousarray(vis32, dtype=np.uint32)
    h, w = v.shape
    rec = np.zeros((h, w, 24), np.float32)
    mat = np.zeros((h, w), np.int32)
    lib().orc_decode_gbuffer_pixels(hs.ref, _p(mi), C.c_uint32(total), _p(cam), _p(v), C.c_uint32(w), C.c_uint32(h), _p(rec), _p(mat))
    return rec, mat


def tangent_frame(px, cam_pos):
    """orc_gbuffer_tangent_frame: (T, B) as float32 triples"""
    out = np.zeros(6, np.float32)
    lib().orc_gbuffer_tangent_frame(_p(np.ascontiguousarray(px, dtype=np.float32)), _p(np.ascontiguousarray(cam_pos, dtype=np.float32)), _p(out))
    return out[:3], out[3:]


def _image(texels, fmt):
    lv = texels if isinstance(texels, (list, tuple)) else [texels]
    t = np.ascontiguousarray(np.concatenate([np.ascontiguousarray(l, dtype=np.uint8).reshape(-1) for l in lv]))
    img = np.zeros(1, dtype=pyoracle.abi.ALPHA_IMAGE_DT)
    img[0] = (t.ctypes.data, lv[0].shape[1], lv[0].shape[0], fmt, len(lv))
    return img, t


def sample_level(texels, fmt, u, v, level=0, filt=0, sampler=None):
    img, keep = _image(texels, fmt)
    smp = None if sampler is None else np.array([sampler], dtype=pyoracle.abi.SAMPLER_DT)
    out = np.zeros(4, np.float32)
    lib().orc_gbuffer_sample_level(_p(img), _p(smp), level, filt, u, v, _p(out))
    return out


def sample_grad(texels, fmt, u, v, ddx, ddy, sampler=None):
    img, keep = _image(texels, fmt)
    smp = None if sampler is None else np.array([sampler], dtype=pyoracle.abi.SAMPLER_DT)
    out = np.zeros(4, np.float32)
    lib().orc_gbuffer_sample_grad(_p(img), _p(smp), u, v, ddx[0], ddx[1], ddy[0], ddy[1], _p(out))
    return out


def shade(table, material_index, px, cam_pos, want=15):
    """orc_gbuffer_shade on one pixel record (24 floats, see oxc_oracle_gbuffer.h): 16 floats or None (material out of range)"""
    p = np.ascontiguousarray(px, dtype=np.float32).reshape(24)
    out = np.zeros(16, np.float32)
    ok = lib().orc_gbuffer_shade(C.byref(table.ref), C.c_uint32(material_index), _p(p), _p(np.ascontiguousarray(cam_pos, dtype=np.float32)),
                                 C.c_uint32(want), _p(out))
    return out if ok else None


__all__ = ["build", "lib", "srgb_table", "decode_gbuffer", "decode_pixels", "tangent_frame", "texel_fetches", "sample_level", "sample_grad", "shade", "PLANES", "pyoracle"]
