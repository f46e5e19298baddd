"""The atmospheric PBR apply's per-pixel source (csrc/oxc_pbr_atmosphere.cuh), compiled for the HOST through tests/host_shim/, against
the oracle (oracle/oxc_oracle_pbr_atmosphere.c) on every pixel, without a GPU: frames with 0, 17 and 256 mixed lights, every flag the
pass reads, NULL optional planes, random and oracle-made LUTs and cubes, and hostile planes, LUTs, cubes, records and lights.  The
constants the pass reads are pinned bit for bit.  The GPU tier checks the same source as compiled by nvcc."""
import subprocess

import numpy as np
import pytest

from oxylus_b200 import abi
from tests.host_harness import compile_harness, skip_without_fma
from tests.test_gpu_pbr import mixed_lights, random_planes
from tests.test_oracle_pbr_atmosphere import random_sky, small_atmosphere

OPTIONAL = ("ambient_occlusion", "shadow", "contact_shadow")
EVERY = abi.SCENE_HAS_ATMOSPHERE | abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_CONTACT_SHADOWS


@pytest.fixture(scope="module")
def pa():
    import pyoracle_pbr_atmosphere

    pyoracle_pbr_atmosphere.build()
    return pyoracle_pbr_atmosphere


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return compile_harness(tmp_path_factory.mktemp("pbra"), "pbr_atmosphere_vs_oracle")


def _cases():
    """(label, camera, settings, atmosphere, lights, planes, omitted planes, sky planes)"""
    out = []
    specs = [((1, 1), 1, EVERY, (), False, (8, 6, 4)), ((33, 17), 0, EVERY | abi.SCENE_HAS_SKY, (), True, (32, 32, 24)),
             ((64, 48), 17, EVERY, ("ambient_occlusion",), False, (8, 6, 5)),
             ((96, 54), 256, abi.SCENE_HAS_ATMOSPHERE, ("shadow", "contact_shadow"), True, (8, 6, 4)),
             ((80, 45), 17, EVERY | abi.SCENE_TRANSPARENT_BACKGROUND, (), True, (16, 8, 3))]
    for k, ((w, h), n, flags, omit, hostile, ap) in enumerate(specs):
        rng = np.random.default_rng(900 + k)
        at = small_atmosphere(ap)
        if k == 3:
            at.planet_radius, at.aerial_perspective_exposure = float("nan"), float("inf")
        pcam, planes = random_planes(rng, w, h, yaw=9.0 * k, hostile=hostile)
        pcam.position[1] = float(rng.choice([0.2, 1000.0, 20000.0]))
        lights = mixed_lights(rng, n, hostile=hostile)
        sun = [float(v) for v in rng.normal(size=3)] if k % 2 else [0.3, 0.8, 0.52]
        s = abi.pbr_settings(scene_flags=flags, sun_direction=sun, sun_intensity=float(rng.uniform(1, 12)), light_count=n)
        out.append((f"{w}x{h}_{n}", pcam, s, at, lights, planes, omit, random_sky(rng, at, hostile=hostile)))
    return out


def _run(exe, tmp_path, case):
    label, pcam, s, at, lights, planes, omit, sky = case
    h, w = planes["depth"].shape
    src, dst = tmp_path / f"{label}.in", tmp_path / f"{label}.out"
    mask = sum(1 << i for i, k in enumerate(OPTIONAL) if k not in omit)
    with open(src, "wb") as f:
        f.write(bytes(pcam))
        f.write(bytes(s))
        f.write(bytes(at))
        f.write(np.uint32([w, h, mask]).tobytes())
        if len(lights):
            f.write(bytes(lights))
        for k in abi.PBR_INPUTS:
            if k not in omit:
                f.write(np.ascontiguousarray(planes[k], dtype=np.float32).tobytes())
        for p in sky:
            f.write(np.ascontiguousarray(p, dtype=np.float16).tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout + r.stderr
    return np.fromfile(dst, dtype=np.float32).reshape(h, w, 4)


def _want(pa, case):
    _, pcam, s, at, lights, planes, omit, sky = case
    p = [None if k in omit else planes[k] for k in abi.PBR_INPUTS]
    return pa.apply_pbr_atmosphere(pcam, s, at, lights, *p, *sky)


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_constants_the_pass_reads(exe, pa, tmp_path):
    dst = tmp_path / "constants.out"
    subprocess.check_call([exe, "--constants", str(dst)])
    device = np.fromfile(dst, dtype=np.uint32)
    oracle = pa.pass_constants().view(np.uint32)
    assert device.tolist() == oracle.tolist()
    assert device[0] == 0x3C8EFA35 and device[2] == 0x3F3504F3 and device[3] == 0x4479FFFF
    # min_cos: canonical_cos of the argument, the correctly rounded cosine
    assert device[1] == np.float32(np.cos(np.float64(np.uint32(0x3C8EFA35).view(np.float32)))).view(np.uint32)


def test_device_source_equals_the_oracle_on_the_host(exe, pa, cases, tmp_path):
    for case in cases:
        got, want = _run(exe, tmp_path, case), _want(pa, case)
        bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
        assert bad.size == 0, f"{case[0]}: {len(bad)} values differ, first at {bad[:3].tolist()}"


def test_the_comparison_is_sensitive_to_contraction(pa, cases, tmp_path):
    """the same source built WITH fma contraction disagrees with the oracle: fused multiply-adds break the canonical order"""
    skip_without_fma()
    exe = compile_harness(tmp_path, "pbr_atmosphere_vs_oracle", contract=True)
    differ = 0
    for case in cases[2:]:
        differ += int((_run(exe, tmp_path, case).view(np.uint32) != _want(pa, case).view(np.uint32)).sum())
    assert differ > 0
