"""The atmosphere's per-texel source (csrc/oxc_atmosphere.cuh), compiled for the HOST through tests/host_shim/ with the parameters of its
atmosphere_make_params, against the oracle (oracle/oxc_oracle_atmosphere.c) on every texel of the three LUTs: the default and random
atmospheres, cameras at 2 m, 10 km, 150 km and below the ground, the sun at the zenith, on the horizon, below it and at random, odd and
minimum sizes, and hostile NaN / Inf / denormal records, cameras and suns.  The GPU tier checks the same source as compiled by nvcc."""
import subprocess

import numpy as np
import pytest

from oxylus_b200 import abi
from tests.host_harness import compile_harness, skip_without_fma
from tests.test_gpu_atmosphere import HEIGHTS, SUNS, camera_for, hostile_atmospheres, lut_shapes, random_atmosphere


@pytest.fixture(scope="module")
def ao():
    import pyoracle_atmosphere

    pyoracle_atmosphere.build()
    return pyoracle_atmosphere


SMALL = dict(transmittance_lut_size=(48, 12, 1), sky_view_lut_size=(23, 13, 1), aerial_perspective_lut_size=(9, 5, 6))
MINIMUM = dict(transmittance_lut_size=(1, 1, 1), sky_view_lut_size=(2, 2, 1), aerial_perspective_lut_size=(1, 1, 1))


def _cases():
    """(label, bake record, frame record, camera, sun, intensity)"""
    out = []
    default = abi.atmosphere(**SMALL)
    for k, (hl, h) in enumerate(list(HEIGHTS.items()) + [("below", -500.0)]):
        for sl in ("zenith", "horizon", "below", "45deg"):
            out.append((f"default-{hl}-{sl}", default, default, camera_for(h, yaw=29.0 * k), SUNS[sl], 10.0))
    rng = np.random.default_rng(77)
    for k in range(4):
        a = random_atmosphere(rng, **SMALL)
        out.append((f"random{k}", default if k % 2 else a, a, camera_for(float(rng.uniform(-10, 20000)), yaw=float(rng.uniform(0, 360))),
                    tuple(rng.normal(size=3)), float(rng.uniform(1, 20))))
    nan, inf = float("nan"), float("inf")
    cams = [camera_for(0.2), abi.pbr_camera(np.full(16, nan, np.float32), (nan, nan, nan)),
            abi.pbr_camera(np.eye(4, dtype=np.float32).reshape(16), (0.0, inf, 1e-40))]
    for k, a in enumerate(hostile_atmospheres(**SMALL)):
        out.append((f"hostile{k}", a, a, cams[k % 3], ((nan, 1.0, 0.0), (0.0, 0.0, 0.0), (inf, 1e-40, -inf))[k % 3], (10.0, nan, inf)[k % 3]))
    m = abi.atmosphere(**MINIMUM)
    out.append(("minimum", m, m, camera_for(0.2), SUNS["45deg"], 10.0))
    return out


def _run(exe, tmp_path, case):
    label, bake, frame, cam, sun, intensity = case
    src, dst = tmp_path / f"{label}.in", tmp_path / f"{label}.out"
    with open(src, "wb") as f:
        f.write(bytes(bake))
        f.write(bytes(frame))
        f.write(bytes(cam))
        f.write(np.float32(list(sun) + [intensity]).tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = np.fromfile(dst, dtype=np.float16)
    ts, svs, aps = lut_shapes(frame)
    nt, nsv = int(np.prod(ts)), int(np.prod(svs))
    return raw[:nt].reshape(ts), raw[nt:nt + nsv].reshape(svs), raw[nt + nsv:].reshape(aps)


def _oracle(ao, case):
    _, bake, frame, cam, sun, intensity = case
    t = ao.transmittance(bake)
    sv, ap = ao.sky_luts(frame, cam, sun, intensity, t)
    return t, sv, ap


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_device_source_equals_the_oracle_on_the_host(ao, cases, tmp_path):
    exe = compile_harness(tmp_path, "atmosphere_vs_oracle")
    lit = 0
    for case in cases:
        got, want = _run(exe, tmp_path, case), _oracle(ao, case)
        for name, g, w in zip(("transmittance", "sky view", "aerial perspective"), got, want):
            bad = np.argwhere(g.view(np.uint16) != w.view(np.uint16))
            assert bad.size == 0, f"{case[0]} {name}: {len(bad)} channels differ, first at {bad[:3].tolist()}"
        lit += int((want[1][..., :3].astype(np.float32) > 0).sum())
    assert lit > 1000


def test_the_comparison_is_sensitive_to_contraction(ao, cases, tmp_path):
    """the same source built WITH fma contraction disagrees with the oracle: fused multiply-adds break the canonical order"""
    skip_without_fma()
    exe = compile_harness(tmp_path, "atmosphere_vs_oracle", contract=True)
    differ = 0
    for case in cases[:6]:
        got, want = _run(exe, tmp_path, case), _oracle(ao, case)
        differ += sum(int((g.view(np.uint16) != w.view(np.uint16)).sum()) for g, w in zip(got, want))
    assert differ > 0
