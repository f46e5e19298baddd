"""The VSM shadow resolve's per-pixel source (csrc/oxc_vsm_resolve.cuh), compiled for the HOST through tests/host_shim/, against the
oracle (oracle/oxc_oracle_vsm_resolve.c) pixel for pixel, without a GPU: over 10^6 pixels of random depth (sky, NaN, Inf and
denormals included), random normals (hostile values included), random clipmaps with uneven page offsets (one not orthographic),
random tables with addresses beyond the atlas, and random atlases.  The GPU tier checks the same source as compiled by nvcc."""
import subprocess

import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.host_harness import compile_harness, skip_without_fma

@pytest.fixture(scope="module")
def vr():
    import pyoracle_vsm_resolve

    pyoracle_vsm_resolve.build()
    return pyoracle_vsm_resolve


def _cases():
    from tests.test_gpu_vsm_pages import clipmaps, vsm_context
    from tests.test_gpu_vsm_resolve import inverse_pv, random_inputs

    scene = synth.make_scene(3000, config_index=2, width=640, height=360, n_unique_meshes=8)
    out = []
    for seed, shape in ((31, "reference"), (32, "uneven")):
        rng = np.random.default_rng(seed)
        if shape == "reference":
            vsm = vsm_context(width=1280, height=720)
        else:
            vsm = vsm_context(size=24, page_size=64, physical=2048, width=640, height=360)
        cm = clipmaps(10, rng, center=(6.0, -2.0, -115.0))
        if shape == "uneven":
            cm["projection_view_mat"][3][3] = np.float32(1.0001)
            cm["projection_view_mat"][5][7] = np.float32(1e-4)
        cam, depth, normals, pt, atlas = random_inputs(rng, scene, vsm)
        out.append((shape, vsm, inverse_pv(cam), np.float32([1280, 720]) if shape == "reference" else cam["resolution"][0], cm, depth, normals, pt, atlas))
    return out


def _run(exe, tmp_path, case):
    shape, vsm, inv_pv, res, cm, depth, normals, pt, atlas = case
    src, dst = tmp_path / f"{shape}.in", tmp_path / f"{shape}.out"
    with open(src, "wb") as f:
        for a, dt in ((vsm, abi.VSM_CONTEXT_DT), (inv_pv, np.float32), (res, np.float32), (cm, abi.CLIPMAP_DT), (depth, np.float32),
                      (normals, np.float32), (pt, np.uint32), (atlas, np.float32)):
            f.write(np.ascontiguousarray(a, dtype=dt).tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout + r.stderr
    return np.fromfile(dst, dtype=np.float32).reshape(depth.shape), r.stdout


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_device_source_equals_the_oracle_on_the_host(vr, cases, tmp_path):
    exe = compile_harness(tmp_path, "vsm_resolve_vs_oracle")
    pixels = 0
    for case in cases:
        shape, vsm, inv_pv, res, cm, depth, normals, pt, atlas = case
        got, log = _run(exe, tmp_path, case)
        want, pcf = vr.vsm_resolve_shadows(vsm, inv_pv, res, cm, depth, normals, pt, atlas)
        np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32), err_msg=shape)
        assert pcf.sum() > 1000 and ((want > 0) & (want < 1)).sum() > 1000, (shape, log)
        pixels += depth.size
    assert pixels >= 1_000_000


def test_the_comparison_is_sensitive_to_contraction(vr, cases, tmp_path):
    """the same source built WITH fma contraction disagrees with the oracle: fused multiply-adds break the canonical order"""
    skip_without_fma()
    exe = compile_harness(tmp_path, "vsm_resolve_vs_oracle", contract=True)
    differ = 0
    for case in cases:
        shape, vsm, inv_pv, res, cm, depth, normals, pt, atlas = case
        got, _ = _run(exe, tmp_path, case)
        want, _ = vr.vsm_resolve_shadows(vsm, inv_pv, res, cm, depth, normals, pt, atlas)
        differ += int((got.view(np.uint32) != want.view(np.uint32)).sum())
    assert differ > 0
