"""FXAA's device source (csrc/oxc_fxaa.cuh), compiled for the HOST through tests/host_shim/ with the parameters of its builder, against
the oracle (oracle/oxc_oracle_fxaa.c) on every pixel and every tap count: hostile frames (NaN, +-inf, negatives, subnormals, 3e38), the
GPU module's frame kinds at small and odd extents; and the header's constants against the oracle's binary32 formation of the literals.
The header walks only the moving axis and the oracle carries both uv components, so the comparison also checks that the fixed component
stays bit-identical.  The GPU tier checks the same source as compiled by nvcc."""
import subprocess

import numpy as np
import pytest

from tests.host_harness import compile_harness, skip_without_fma
from tests.test_gpu_fxaa import small_frames
from tests.test_gpu_post import hostile_frame


@pytest.fixture(scope="module")
def so():
    import pyoracle_fxaa

    pyoracle_fxaa.build()
    return pyoracle_fxaa


def _cases():
    """(label, frame)"""
    rng = np.random.default_rng(29)
    out = []
    for w, h, seed in ((1, 1, 1), (1, 7, 2), (7, 1, 3), (2, 2, 4), (3, 3, 5), (37, 23, 6), (64, 36, 7)):
        out += [(f"{label}-{w}x{h}", f) for label, f in small_frames(w, h, seed)]
    for k, (w, h) in enumerate(((40, 26), (33, 17), (48, 30))):
        out.append((f"hostile{k}", hostile_frame(rng, w, h)))
    return out


def _run(exe, tmp_path, case):
    label, frame = case
    h, w = frame.shape[:2]
    src, dst = tmp_path / f"{label}.in", tmp_path / f"{label}.out"
    with open(src, "wb") as f:
        f.write(np.uint32([w, h]).tobytes())
        f.write(np.ascontiguousarray(frame, np.float32).tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = np.fromfile(dst, dtype=np.uint8)
    n = w * h * 16
    return raw[:16].view(np.float32), raw[16:16 + n].view(np.float32).reshape(h, w, 4), raw[16 + n:].reshape(h, w)


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_device_source_equals_the_oracle_on_the_host(so, cases, tmp_path):
    exe = compile_harness(tmp_path, "fxaa_vs_oracle")
    nonfinite, counts = 0, np.zeros(33, np.int64)
    for case in cases:
        table, got, taps = _run(exe, tmp_path, case)
        want, want_taps = so.fxaa(case[1], with_taps=True)
        bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
        assert bad.size == 0, f"{case[0]}: {len(bad)} values differ, first at {bad[:3].tolist()}"
        np.testing.assert_array_equal(taps, want_taps, err_msg=case[0])
        np.testing.assert_array_equal(table.view(np.uint32), so.constants().view(np.uint32))
        nonfinite += int((~np.isfinite(want)).sum())
        counts += np.bincount(taps.ravel(), minlength=33)
    assert nonfinite > 100  # the hostile cases do reach the NaN and inf paths
    assert counts[5] > 0 and counts[32] > 0 and all(counts[12:33] > 0)


def test_the_comparison_is_sensitive_to_contraction(so, cases, tmp_path):
    """the same source built WITH fma contraction disagrees with the oracle: fused multiply-adds break the canonical order"""
    skip_without_fma()
    exe = compile_harness(tmp_path, "fxaa_vs_oracle", contract=True)
    differ = 0
    for case in cases:
        _, got, _ = _run(exe, tmp_path, case)
        differ += int((got.view(np.uint32) != so.fxaa(case[1]).view(np.uint32)).sum())
    assert differ > 0
