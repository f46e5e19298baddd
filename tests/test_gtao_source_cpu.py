"""The GTAO's per-pixel source (csrc/oxc_gtao.cuh), compiled for the HOST through tests/host_shim/, against the oracle
(oracle/oxc_oracle_gtao.c) on every plane and every pixel, without a GPU: random frames with sky, NaN / Inf / denormal / negative depth,
non-finite normals, all four presets, random and hostile settings, and odd sizes down to 1 x 1.  The GPU tier checks the same source as
compiled by nvcc, with the prefilter's shared-memory tiling."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oxylus_b200 import abi
from tests.test_gpu_gtao import PLANES, assert_planes_equal, gtao_camera_for, random_frame, random_settings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


@pytest.fixture(scope="module")
def go():
    import pyoracle_gtao

    pyoracle_gtao.build()
    return pyoracle_gtao


def _build(tmp_path, extra):
    exe = str(tmp_path / ("gtao_vs_oracle" + ("_fma" if extra else "")))
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wno-unknown-pragmas"] + (extra or ["-ffp-contract=off"]) +
                          ["-I", os.path.join(ROOT, "tests", "host_shim"), "-I", os.path.join(ROOT, "oxylus_b200", "csrc"),
                           os.path.join(ROOT, "tests", "gtao_vs_oracle.cpp"), "-o", exe])
    return exe


def _cases():
    """(label, camera, settings, depth, normals)"""
    out = []
    sizes = [(1, 1), (3, 2), (17, 9), (33, 65), (160, 90), (211, 97), (64, 48), (120, 68)]
    for k, (w, h) in enumerate(sizes):
        rng = np.random.default_rng(300 + k)
        gcam, proj = gtao_camera_for(w, h, yaw=23.0 * k)
        depth, normals = random_frame(rng, w, h, proj, hostile=k % 2 == 0)
        if k < 4:
            settings = abi.gtao_settings(k, noise_index=k * 13)
        else:
            settings = random_settings(rng, hostile=k == 7)
        out.append((f"{w}x{h}", gcam, settings, depth, normals))
    return out


def _run(exe, tmp_path, case):
    label, gcam, settings, depth, normals = case
    h, w = depth.shape
    src, dst = tmp_path / f"{label}.in", tmp_path / f"{label}.out"
    with open(src, "wb") as f:
        f.write(bytes(gcam))
        f.write(bytes(settings))
        f.write(np.uint32([w, h]).tobytes())
        f.write(np.ascontiguousarray(depth, dtype=np.float32).tobytes())
        f.write(np.ascontiguousarray(normals, dtype=np.float32).tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = open(dst, "rb").read()
    _, total = abi.gtao_mip_layout(w, h)
    sizes = (total * 4, w * h * 4, w * h * 2, w * h * 4)
    dtypes = (np.float32, np.uint32, np.uint16, np.float32)
    got, off = {}, 0
    for k, n, dt in zip(PLANES, sizes, dtypes):
        got[k] = np.frombuffer(raw[off:off + n], dtype=dt).reshape(-1 if k == "mips" else (h, w))
        off += n
    return got, r.stdout


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_device_source_equals_the_oracle_on_the_host(go, cases, tmp_path):
    exe = _build(tmp_path, None)
    occluded = 0
    for case in cases:
        got, log = _run(exe, tmp_path, case)
        want = go.generate_ambient_occlusion(case[1], case[2], case[3], case[4])
        assert_planes_equal(got, want, case[0])
        occluded += int((want["ao"] < 0.95).sum())
    assert occluded > 1000


def test_the_comparison_is_sensitive_to_contraction(go, cases, tmp_path):
    """the same source built WITH fma contraction disagrees with the oracle: fused multiply-adds break the canonical order"""
    flags = subprocess.run(["grep", "-c", "fma", "/proc/cpuinfo"], capture_output=True, text=True).stdout.strip()
    if flags in ("", "0"):
        pytest.skip("host CPU has no FMA unit")
    exe = _build(tmp_path, ["-mfma", "-ffp-contract=fast"])
    differ = 0
    for case in cases[4:]:
        got, _ = _run(exe, tmp_path, case)
        want = go.generate_ambient_occlusion(case[1], case[2], case[3], case[4])
        differ += sum(int((np.asarray(got[k]).view(np.uint8) != np.asarray(want[k]).view(np.uint8)).sum()) for k in PLANES)
    assert differ > 0
