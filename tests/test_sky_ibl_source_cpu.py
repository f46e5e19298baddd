"""The sky IBL's per-texel source (csrc/oxc_sky_ibl.cuh), compiled for the HOST through tests/host_shim/ with the parameters of its
sky_ibl_make_params, against the oracle (oracle/oxc_oracle_sky_ibl.c) on every texel of the cube: the default record with cameras at 2 m,
10 km and 150 km and four suns, random records, odd LUT sizes, a history sequence, and hostile records, cameras, suns and cubes.  Also
canonical_atan2 and canonical_acos of oxc_exact.cuh against the oracle's on 2 M inputs.  The GPU tier checks the same source as
compiled by nvcc."""
import subprocess

import numpy as np
import pytest

from oxylus_b200 import abi
from tests.host_harness import compile_harness, skip_without_fma
from tests.test_gpu_atmosphere import HEIGHTS, SUNS, camera_for, hostile_atmospheres, random_atmosphere
from tests.test_gpu_sky_ibl import SMALL, hostile_cubes, luts


@pytest.fixture(scope="module")
def so():
    import pyoracle_sky_ibl

    pyoracle_sky_ibl.build()
    return pyoracle_sky_ibl


def _cases():
    """(label, record, camera, sun, intensity, ambient strength, frame index, cube or None)"""
    out = []
    default = abi.atmosphere(**SMALL)
    for hl, h in HEIGHTS.items():
        for sl in ("zenith", "horizon", "below", "45deg"):
            out.append((f"default-{hl}-{sl}", default, camera_for(h, yaw=11.0), SUNS[sl], 10.0, 0.15, 0, None))
    rng = np.random.default_rng(41)
    for k in range(3):
        a = random_atmosphere(rng, **SMALL)
        out.append((f"random{k}", a, camera_for(float(rng.uniform(-10, 20000))), tuple(rng.normal(size=3) * 3), float(rng.uniform(1, 20)),
                    float(rng.uniform(0, 1)), int(rng.integers(0, 2 ** 32)), None))
    odd = abi.atmosphere(transmittance_lut_size=(7, 3, 1), sky_view_lut_size=(2, 2, 1))
    out.append(("minimum-sky-view", odd, camera_for(0.2), SUNS["45deg"], 10.0, 0.15, 3, None))
    nan, inf = float("nan"), float("inf")
    cams = [camera_for(0.2), abi.pbr_camera(np.full(16, nan, np.float32), (nan, nan, nan)),
            abi.pbr_camera(np.eye(4, dtype=np.float32).reshape(16), (0.0, inf, 1e-40))]
    suns = [(nan, 1.0, 0.0), (0.0, 0.0, 0.0), (inf, 1e-40, -inf)]
    for k, a in enumerate(hostile_atmospheres(**SMALL)):
        out.append((f"hostile-record{k}", a, cams[k % 3], suns[k % 3], (10.0, nan, inf)[k % 3], 0.15, k, None))
    for k, cube in enumerate(hostile_cubes()):
        out.append((f"hostile-cube{k}", default, camera_for(1000.0), SUNS["45deg"], 10.0, (0.15, nan, -inf, 1e30)[k % 4],
                    (7, 0xFFFFFFFF, 1 << 24, 12345)[k % 4], cube))
    return out


def _run(exe, tmp_path, case, t, sv):
    label, a, cam, sun, intensity, strength, frame, cube = case
    cube = np.zeros((6, 32, 32, 4), np.float16) if cube is None else cube
    src, dst = tmp_path / f"{label}.in", tmp_path / f"{label}.out"
    with open(src, "wb") as f:
        f.write(bytes(a))
        f.write(bytes(cam))
        f.write(np.float32(list(sun) + [intensity, strength]).tobytes())
        f.write(np.uint32(frame).tobytes())
        f.write(np.ascontiguousarray(t, np.float16).tobytes())
        f.write(np.ascontiguousarray(sv, np.float16).tobytes())
        f.write(np.ascontiguousarray(cube, np.float16).tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    return np.fromfile(dst, dtype=np.float16).reshape(6, 32, 32, 4)


def _oracle(so, case, t, sv):
    _, a, cam, sun, intensity, strength, frame, cube = case
    return so.sky_ibl(a, cam, sun, intensity, strength, frame, t, sv, cube)


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_device_source_equals_the_oracle_on_the_host(so, cases, tmp_path):
    exe = compile_harness(tmp_path, "sky_ibl_vs_oracle")
    lit = 0
    for case in cases:
        t, sv = luts(case[1], case[2], case[3], case[4])
        got, want = _run(exe, tmp_path, case, t, sv), _oracle(so, case, t, sv)
        bad = np.argwhere(got.view(np.uint16) != want.view(np.uint16))
        assert bad.size == 0, f"{case[0]}: {len(bad)} channels differ, first at {bad[:3].tolist()}"
        lit += int((want[..., :3].astype(np.float32) > 0).sum())
    assert lit > 100000


def test_history_sequence_on_the_host(so, tmp_path):
    """five calls from a zeroed cube with frame_index 0..4: the first has no history, the next four lerp, all equal the oracle"""
    exe = compile_harness(tmp_path, "sky_ibl_vs_oracle")
    a = abi.atmosphere(**SMALL)
    cam = camera_for(0.2)
    t, sv = luts(a, cam, SUNS["45deg"], 10.0)
    got = want = None
    for frame in range(5):
        case = (f"seq{frame}", a, cam, SUNS["45deg"], 10.0, 0.15, frame, got)
        got = _run(exe, tmp_path, case, t, sv)
        want = _oracle(so, (case[0], a, cam, SUNS["45deg"], 10.0, 0.15, frame, want), t, sv)
        np.testing.assert_array_equal(got.view(np.uint16), want.view(np.uint16))
    assert (got[..., 3] == 1).all()


def test_functions_equal_the_oracle_on_the_host(so, tmp_path):
    """canonical_atan2 and canonical_acos compiled from oxc_exact.cuh give the oracle's bits on 2 M inputs and the special values"""
    exe = compile_harness(tmp_path, "sky_ibl_vs_oracle")
    rng = np.random.default_rng(5)
    n = 1_000_000
    y = np.concatenate([rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32), rng.normal(size=n).astype(np.float32)])
    x = np.concatenate([rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32),
                        rng.uniform(-1.0, 1.0, n).astype(np.float32)])
    special = np.float32([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 1.0000001, -1.0000001, 0.5, -0.5])
    yy, xx = np.meshgrid(special, special)
    y, x = np.concatenate([y, yy.ravel()]), np.concatenate([x, xx.ravel()])
    src, dst = tmp_path / "fn.in", tmp_path / "fn.out"
    with open(src, "wb") as f:
        f.write(np.uint64(y.size).tobytes())
        f.write(y.tobytes())
        f.write(x.tobytes())
    r = subprocess.run([exe, "--functions", str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    got = np.fromfile(dst, dtype=np.float32)
    np.testing.assert_array_equal(got[:y.size].view(np.uint32), so.atan2(y, x).view(np.uint32))
    np.testing.assert_array_equal(got[y.size:].view(np.uint32), so.acos(x).view(np.uint32))


def test_the_comparison_is_sensitive_to_contraction(so, cases, tmp_path):
    """the same source built WITH fma contraction disagrees with the oracle: fused multiply-adds break the canonical order"""
    skip_without_fma()
    exe = compile_harness(tmp_path, "sky_ibl_vs_oracle", contract=True)
    differ = 0
    for case in cases[:4]:
        t, sv = luts(case[1], case[2], case[3], case[4])
        differ += int((_run(exe, tmp_path, case, t, sv).view(np.uint16) != _oracle(so, case, t, sv).view(np.uint16)).sum())
    assert differ > 0
