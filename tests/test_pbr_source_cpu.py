"""PBR apply's per-pixel source (csrc/oxc_pbr.cuh), compiled for the HOST through tests/host_shim/, against the oracle
(oracle/oxc_oracle_pbr.c) on every pixel, without a GPU: random frames with 0, 1, 17 and 256 mixed lights, every flag the pass reads,
NULL optional planes and hostile values.  The GPU tier checks the same source as compiled by nvcc, with the lights staged in shared
memory."""
import subprocess

import numpy as np
import pytest

from oxylus_b200 import abi
from tests.host_harness import compile_harness, skip_without_fma
from tests.test_gpu_pbr import mixed_lights, random_planes, settings_for

@pytest.fixture(scope="module")
def po():
    import pyoracle_pbr

    pyoracle_pbr.build()
    return pyoracle_pbr


def _cases():
    """(label, camera, settings, lights, planes, omitted planes)"""
    out = []
    every = abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_CONTACT_SHADOWS
    specs = [((1, 1), 1, every, ()), ((17, 9), 0, every | abi.SCENE_HAS_SKY, ()), ((64, 48), 17, every, ("ambient_occlusion",)),
             ((96, 54), 256, abi.SCENE_HAS_DIRECTIONAL_LIGHT, ("shadow", "contact_shadow")), ((80, 45), 17, every | abi.SCENE_TRANSPARENT_BACKGROUND, ()),
             ((120, 68), 256, every | abi.SCENE_HAS_SKY, ())]
    for k, ((w, h), n, flags, omit) in enumerate(specs):
        rng = np.random.default_rng(700 + k)
        pcam, planes = random_planes(rng, w, h, yaw=11.0 * k, hostile=k % 2 == 1)
        lights = mixed_lights(rng, n, hostile=k == 5)
        s = settings_for(flags, n, rng if k >= 3 else None)
        out.append((f"{w}x{h}_{n}", pcam, s, lights, planes, omit))
    return out


def _run(exe, tmp_path, case):
    label, pcam, s, lights, planes, omit = case
    h, w = planes["depth"].shape
    src, dst = tmp_path / f"{label}.in", tmp_path / f"{label}.out"
    mask = sum(1 << i for i, k in enumerate(("ambient_occlusion", "shadow", "contact_shadow")) if k not in omit)
    with open(src, "wb") as f:
        f.write(bytes(pcam))
        f.write(bytes(s))
        f.write(np.uint32([w, h, mask]).tobytes())
        if len(lights):
            f.write(bytes(lights))
        for k in ("depth", "albedo", "normal", "emissive", "metallic_roughness_occlusion", "ambient_occlusion", "shadow", "contact_shadow"):
            if k not in omit:
                f.write(np.ascontiguousarray(planes[k], dtype=np.float32).tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout + r.stderr
    return np.fromfile(dst, dtype=np.float32).reshape(h, w, 4)


def _want(po, case):
    _, pcam, s, lights, planes, omit = case
    p = {k: (None if k in omit else v) for k, v in planes.items()}
    return po.apply_pbr(pcam, s, lights, p["depth"], p["albedo"], p["normal"], p["emissive"], p["metallic_roughness_occlusion"], p["ambient_occlusion"],
                        p["shadow"], p["contact_shadow"])


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_device_source_equals_the_oracle_on_the_host(po, cases, tmp_path):
    exe = compile_harness(tmp_path, "pbr_vs_oracle")
    lit = 0
    for case in cases:
        got, want = _run(exe, tmp_path, case), _want(po, case)
        bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
        assert bad.size == 0, f"{case[0]}: {len(bad)} values differ, first at {bad[:3].tolist()}"
        lit += int((np.nan_to_num(want[..., :3], posinf=0.0, neginf=0.0).sum(-1, dtype=np.float64) > 0.05).sum())
    assert lit > 5000


def test_the_comparison_is_sensitive_to_contraction(po, cases, tmp_path):
    """the same source built WITH fma contraction disagrees with the oracle: fused multiply-adds break the canonical order"""
    skip_without_fma()
    exe = compile_harness(tmp_path, "pbr_vs_oracle", contract=True)
    differ = 0
    for case in cases[2:]:
        differ += int((_run(exe, tmp_path, case).view(np.uint32) != _want(po, case).view(np.uint32)).sum())
    assert differ > 0
