"""The contact-shadow pass's per-pixel source (csrc/oxc_contact_shadows.cuh), compiled for the HOST through tests/host_shim/, against
the oracle (oracle/oxc_oracle_contact_shadows.c) on every pixel, without a GPU: random frames with sky, NaN / Inf / denormal / negative
depth, steps 1 / 2 / 8 / 64, random and hostile settings, and odd sizes down to 1 x 1.  The nearest tap the header picks from the
bilinear tap's four texels is covered by the hostile frames.  The GPU tier checks the same source as compiled by nvcc."""
import subprocess

import numpy as np
import pytest

from tests.host_harness import compile_harness, skip_without_fma
from tests.test_gpu_contact_shadows import box_on_plane, contact_camera_for, random_depth, random_settings

@pytest.fixture(scope="module")
def co():
    import pyoracle_contact_shadows

    pyoracle_contact_shadows.build()
    return pyoracle_contact_shadows


def _cases():
    """(label, camera, settings, depth)"""
    out = []
    sizes = [(1, 1), (3, 2), (17, 9), (33, 65), (160, 90), (211, 97), (64, 48), (120, 68), (320, 180)]
    steps = [1, 2, 8, 64, None, None, None, None, None]
    for k, (w, h) in enumerate(sizes):
        rng = np.random.default_rng(500 + k)
        ccam, proj = contact_camera_for(w, h, yaw=23.0 * k)
        depth = random_depth(rng, w, h, proj, hostile=k % 2 == 0)
        out.append((f"{w}x{h}", ccam, random_settings(rng, steps=steps[k], hostile=k in (6, 7)), depth))
    ccam, _ = contact_camera_for(320, 180)
    from oxylus_b200 import abi

    out.append(("box", ccam, abi.contact_shadow_settings((0.3, 0.2, -1.0), 16, 0.1, 1.0), box_on_plane(320, 180)[0]))
    return out


def _run(exe, tmp_path, case):
    label, ccam, settings, depth = case
    h, w = depth.shape
    src, dst = tmp_path / f"{label}.in", tmp_path / f"{label}.out"
    with open(src, "wb") as f:
        f.write(bytes(ccam))
        f.write(bytes(settings))
        f.write(np.uint32([w, h]).tobytes())
        f.write(np.ascontiguousarray(depth, dtype=np.float32).tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    return np.fromfile(dst, dtype=np.float32).reshape(h, w)


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_device_source_equals_the_oracle_on_the_host(co, cases, tmp_path):
    exe = compile_harness(tmp_path, "contact_shadows_vs_oracle")
    contact = 0
    for case in cases:
        got = _run(exe, tmp_path, case)
        want = co.contact_shadows(case[1], case[2], case[3])
        bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
        assert bad.size == 0, f"{case[0]}: {len(bad)} pixels differ, first at {bad[:3].tolist()}"
        contact += int((want < 1).sum())
    assert contact > 1000


def test_the_comparison_is_sensitive_to_contraction(co, cases, tmp_path):
    """the same source built WITH fma contraction disagrees with the oracle: fused multiply-adds break the canonical order"""
    skip_without_fma()
    exe = compile_harness(tmp_path, "contact_shadows_vs_oracle", contract=True)
    differ = 0
    for case in cases:
        got = _run(exe, tmp_path, case)
        differ += int((got.view(np.uint32) != co.contact_shadows(case[1], case[2], case[3]).view(np.uint32)).sum())
    assert differ > 0
