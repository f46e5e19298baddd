"""The tonemap's device source (csrc/oxc_tonemap.cuh), compiled for the HOST through tests/host_shim/ with the parameters of its builder,
against the oracle (oracle/oxc_oracle_tonemap.c) on every pixel: hostile frames and bloom images (NaN, +-inf, negatives, subnormals,
3e38), hostile settings and records, every curve and flag subset at odd and tiny extents; and the header's hex constant table against
the oracle's binary32 formation of it.  The GPU tier checks the same source as compiled by nvcc."""
import subprocess

import numpy as np
import pytest

from oxylus_b200 import abi
from tests.host_harness import compile_harness, skip_without_fma
from tests.test_gpu_post import HOSTILE_RECORDS, hdr_frame, hostile_frame
from tests.test_gpu_tonemap import BL, CA, EA, FG, HOSTILE_SETTINGS, LENS, TB, TYPES, VG, bloom_image, hostile_settings


@pytest.fixture(scope="module")
def so():
    import pyoracle_tonemap

    pyoracle_tonemap.build()
    return pyoracle_tonemap


def _cases():
    """(label, frame, settings, record, bloom image)"""
    rng = np.random.default_rng(29)
    out = []
    for w, h in ((1, 1), (1, 7), (3, 2), (2, 2), (17, 9), (37, 22)):
        frame, bloom = hdr_frame(rng, w, h), bloom_image(rng, w, h)
        for t in TYPES:
            for flags in (0, EA | BL | LENS | TB, BL | VG | FG, CA | TB):
                flags &= ~BL if w < 2 or h < 2 else ~0
                out.append((f"hdr-{w}x{h}-{t}-{flags:#x}", frame, abi.tonemap_settings(flags, t, film_grain_seed=w), abi.Exposure(1.0, 1.5), bloom))
    for k in range(len(HOSTILE_SETTINGS)):
        w, h = (40, 26) if k % 2 else (33, 17)
        frame, bloom = hostile_frame(rng, w, h), hostile_frame(rng, w // 2, h // 2)
        for t in TYPES:
            flags = (EA | BL | LENS | TB) if k % 2 else (BL | VG | FG | EA)
            out.append((f"hostile{k}-{t}", frame, hostile_settings(k, flags, t), HOSTILE_RECORDS[k % len(HOSTILE_RECORDS)], bloom))
    return out


def _run(exe, tmp_path, case):
    label, frame, s, rec, bloom = case
    h, w = frame.shape[:2]
    src, dst = tmp_path / f"{label}.in", tmp_path / f"{label}.out"
    with open(src, "wb") as f:
        f.write(np.uint32([w, h]).tobytes())
        f.write(bytes(s))
        f.write(bytes(rec))
        f.write(np.ascontiguousarray(frame, np.float32).tobytes())
        f.write(np.ascontiguousarray(bloom, np.float32)[: h // 2, : w // 2].tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = np.fromfile(dst, dtype=np.float32)
    return raw[:33], raw[33:].reshape(h, w, 4)


def _oracle(so, case):
    _, frame, s, rec, bloom = case
    h, w = frame.shape[:2]
    return so.tonemap(frame, s, rec, bloom if s.scene_flags & BL else None)


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_device_source_equals_the_oracle_on_the_host(so, cases, tmp_path):
    exe = compile_harness(tmp_path, "tonemap_vs_oracle")
    nonfinite = 0
    for case in cases:
        table, got = _run(exe, tmp_path, case)
        want = _oracle(so, case)
        bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
        assert bad.size == 0, f"{case[0]}: {len(bad)} values differ, first at {bad[:3].tolist()}"
        np.testing.assert_array_equal(table.view(np.uint32), so.constants().view(np.uint32))
        nonfinite += int((~np.isfinite(want)).sum())
    assert nonfinite > 100  # the hostile cases do reach the NaN and inf paths


def test_the_comparison_is_sensitive_to_contraction(so, cases, tmp_path):
    """the same source built WITH fma contraction disagrees with the oracle: fused multiply-adds break the canonical order"""
    skip_without_fma()
    exe = compile_harness(tmp_path, "tonemap_vs_oracle", contract=True)
    differ = 0
    for case in cases[4:12]:
        _, got = _run(exe, tmp_path, case)
        differ += int((got.view(np.uint32) != _oracle(so, case).view(np.uint32)).sum())
    assert differ > 0
