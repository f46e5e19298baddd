"""The terrain draw's device source (csrc/oxc_terrain.cuh with the raster core), compiled for the HOST through tests/host_shim/ with the
parameters of its builder, against the oracle (oracle/oxc_oracle_terrain_draw.c) on every pixel of the vis buffer and every patch's
triangle count: flat, noisy and rough heightmaps, the three measurement cameras, a camera inside the terrain (the clip path), both
packings, tiny and clamped settings, an out-of-range instance count and bad patch indices.  The device finds each stitch step by
bisection, the oracle walks the strip, so the comparison also checks that the two give the same triangles.  The GPU tier checks the
same source as compiled by nvcc."""
import subprocess

import numpy as np
import pytest

from tests import helpers_terrain as ht
from tests.host_harness import compile_harness, skip_without_fma


@pytest.fixture(scope="module")
def so():
    import pyoracle_terrain_draw

    pyoracle_terrain_draw.build()
    return pyoracle_terrain_draw


def _cases():
    """(label, heightmap, settings, camera, width, height, prim_bits, instance_count, visible)"""
    out = []
    for k, (kind, pc, res) in enumerate((("flat", (4, 4), (32, 32)), ("noise", (8, 8), (64, 64)), ("rough", (3, 7), (20, 33)))):
        hm = ht.heightmap(res[0], res[1], 10 + k, kind)
        t = ht.terrain(pc, (128.0, 96.0), (0.0, 40.0))
        n = pc[0] * pc[1]
        vis = np.arange(n, dtype=np.uint32)
        for name, cam in ht.views(hm, t, 96, 54).items():
            out.append((f"{kind}-{name}", hm, ht.settings(t), cam, 96, 54, 8, n, vis))
        cam = ht.views(hm, t, 64, 40)["horizon"]
        out.append((f"{kind}-wide-ids", hm, ht.settings(t, 4.0), cam, 64, 40, 6, n, vis))
        out.append((f"{kind}-max1", hm, ht.settings(t, 1.0, 1.0), cam, 64, 40, 8, n, vis))
        out.append((f"{kind}-max3", hm, ht.settings(t, 1.0, 3.0), cam, 64, 40, 8, n, vis))
        bad = vis.copy()
        bad[::3] = n + 5
        out.append((f"{kind}-bad-index", hm, ht.settings(t, 2.0), cam, 64, 40, 8, n + 100, bad))
    hm = ht.heightmap(16, 16, 3, "noise")
    t = ht.terrain((2, 2), (8.0, 8.0), (0.0, 4.0))
    inside = ht.camera(48, 32, (0.0, 1.0, 0.0), (0.0, 1.0, -5.0), near=0.05)  # the terrain rises through the near plane
    out.append(("inside", hm, ht.settings(t, 1.0), inside, 48, 32, 8, 4, np.arange(4, dtype=np.uint32)))
    return out


def _run(exe, tmp_path, case):
    label, hm, st, cam, w, h, bits, count, visible = case
    src, dst = tmp_path / f"{label}.in", tmp_path / f"{label}.out"
    with open(src, "wb") as f:
        f.write(np.uint32([hm.shape[1], hm.shape[0]]).tobytes())
        f.write(np.ascontiguousarray(hm, np.uint16).tobytes())
        f.write(np.ascontiguousarray(st).tobytes())
        f.write(np.ascontiguousarray(cam).tobytes())
        f.write(np.uint32([w, h, bits, count, len(visible)]).tobytes())
        f.write(np.ascontiguousarray(visible, np.uint32).tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = np.fromfile(dst, dtype=np.uint8)
    return raw[: w * h * 8].view(np.uint64).reshape(h, w), raw[w * h * 8:].view(np.uint32)


def _oracle(so, case):
    label, hm, st, cam, w, h, bits, count, visible = case
    vis = np.full((h, w), 0xFFFFFFFF, np.uint64)
    so.draw_terrain(hm, st, visible, count, cam, vis, bits)
    return vis


@pytest.fixture(scope="module")
def cases():
    return _cases()


def test_device_source_equals_the_oracle_on_the_host(so, cases, tmp_path):
    exe = compile_harness(tmp_path, "terrain_draw_vs_oracle")
    written = 0
    for case in cases:
        got, tris = _run(exe, tmp_path, case)
        want = _oracle(so, case)
        bad = np.argwhere(got != want)
        assert bad.size == 0, f"{case[0]}: {len(bad)} pixels differ, first at {bad[:3].tolist()}"
        _, hm, st, cam, _, _, _, count, visible = case
        total = int(st["terrain"]["patch_count"][0].prod())
        for slot, idx in enumerate(visible):
            expect = so.patch(hm, st, cam, int(idx)).triangles if slot < min(count, total) and idx < total else 0
            assert tris[slot] == expect, f"{case[0]}: slot {slot}"
        written += int((want != 0xFFFFFFFF).sum())
    assert written > 10000


def test_the_comparison_is_sensitive_to_contraction(so, cases, tmp_path):
    """the same source built WITH fma contraction disagrees with the oracle: fused multiply-adds break the canonical order"""
    skip_without_fma()
    exe = compile_harness(tmp_path, "terrain_draw_vs_oracle", contract=True)
    differ = 0
    for case in cases:
        got, _ = _run(exe, tmp_path, case)
        differ += int((got != _oracle(so, case)).sum())
    assert differ > 0
