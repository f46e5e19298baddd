"""Eye adaptation's and bloom's device sources (csrc/oxc_exposure.cuh, csrc/oxc_bloom.cuh), compiled for the HOST through
tests/host_shim/ with the parameters of their builders, against the oracle (oracle/oxc_oracle_post.c) on every bin, record and texel:
HDR, hostile and uniform frames at odd and tiny extents, NaN and Inf settings, delta times and records, bloom with HasEyeAdaptation on
and off, and the caller's last upsampled level.  The GPU tier checks the same sources as compiled by nvcc."""
import subprocess

import numpy as np
import pytest

from oxylus_b200 import abi
from tests.host_harness import compile_harness, skip_without_fma
from tests.test_gpu_post import HOSTILE_BLOOM, HOSTILE_EYE, HOSTILE_RECORDS, INF, NAN, hdr_frame, hostile_frame, uniform_frame


@pytest.fixture(scope="module")
def so():
    import pyoracle_post

    pyoracle_post.build()
    return pyoracle_post


def _cases():
    """(label, frame, eye settings, delta_time, record, bloom settings, upsampled content or None)"""
    rng = np.random.default_rng(23)
    out = []
    for w, h in ((1, 1), (2, 2), (3, 2), (2, 7), (67, 45), (96, 70), (161, 3)):
        out.append((f"hdr-{w}x{h}", hdr_frame(rng, w, h), abi.eye_adaptation_settings(), 0.016, abi.Exposure(1.0, 1.0),
                    abi.bloom_settings(scene_flags=abi.SCENE_HAS_EYE_ADAPTATION), None))
    for k, (es, bs) in enumerate(zip(HOSTILE_EYE, HOSTILE_BLOOM)):
        bs = abi.BloomSettings.from_buffer_copy(bs)
        bs.scene_flags = abi.SCENE_HAS_EYE_ADAPTATION if k % 2 else 0
        w, h = (37, 29) if k % 2 else (64, 33)
        n = abi.bloom_chain_texels(w, h)
        out.append((f"hostile{k}", hostile_frame(rng, w, h), es, (0.016, 0.0, INF, NAN, -1.0, 1e-40)[k], HOSTILE_RECORDS[k % len(HOSTILE_RECORDS)],
                    bs, rng.normal(size=(n, 4)).astype(np.float32)))
    out.append(("uniform", uniform_frame(40, 24), abi.eye_adaptation_settings(), 0.1, abi.Exposure(1.0, 1.0), abi.bloom_settings(), None))
    return out


def _run(exe, tmp_path, case):
    label, frame, es, dt, rec, bs, up = case
    h, w = frame.shape[:2]
    n = abi.bloom_chain_texels(w, h) if w >= 2 and h >= 2 else 0
    up = np.zeros((n, 4), np.float32) if up is None else up
    src, dst = tmp_path / f"{label}.in", tmp_path / f"{label}.out"
    with open(src, "wb") as f:
        f.write(np.uint32([w, h]).tobytes())
        f.write(bytes(es))
        f.write(np.float32(dt).tobytes())
        f.write(bytes(rec))
        f.write(bytes(bs))
        f.write(np.ascontiguousarray(frame, np.float32).tobytes())
        f.write(np.ascontiguousarray(up, np.float32).tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = np.fromfile(dst, dtype=np.uint32)
    return raw[:256], raw[256:258], raw[258:258 + n * 4].view(np.float32).reshape(n, 4), raw[258 + n * 4:].view(np.float32).reshape(n, 4)


def _oracle(so, case):
    _, frame, es, dt, rec, bs, up = case
    h, w = frame.shape[:2]
    rec, hist = so.eye_adaptation(frame, es, dt, rec)
    chains = so.bloom(frame, bs, rec, up) if w >= 2 and h >= 2 else (np.zeros((0, 4), np.float32),) * 2
    return hist, np.frombuffer(bytes(rec), np.uint32), chains[0], chains[1]


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_device_sources_equal_the_oracle_on_the_host(so, cases, tmp_path):
    exe = compile_harness(tmp_path, "post_vs_oracle")
    lit = 0
    for case in cases:
        got, want = _run(exe, tmp_path, case), _oracle(so, case)
        for name, g, wv in zip(("bins", "record", "downsampled", "upsampled"), got, want):
            bad = np.argwhere(g.view(np.uint32) != wv.view(np.uint32))
            assert bad.size == 0, f"{case[0]} {name}: {len(bad)} values differ, first at {bad[:3].tolist()}"
        lit += int((want[3][:, :3] > 0).sum())
    assert lit > 5000


def test_the_comparison_is_sensitive_to_contraction(so, cases, tmp_path):
    """the same sources built WITH fma contraction disagree with the oracle: fused multiply-adds break the canonical order"""
    skip_without_fma()
    exe = compile_harness(tmp_path, "post_vs_oracle", contract=True)
    differ = 0
    for case in cases[4:6]:
        got, want = _run(exe, tmp_path, case), _oracle(so, case)
        differ += sum(int((g.view(np.uint32) != wv.view(np.uint32)).sum()) for g, wv in zip(got, want))
    assert differ > 0
