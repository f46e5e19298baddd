"""The G-buffer decode's material half (csrc/oxc_gbuffer.cuh: the device table oxc_set_materials builds, and gbuffer_shade), compiled
for the HOST through tests/host_shim/, against the oracle (oracle/oxc_oracle_gbuffer.c) on every pixel of a frame, without a GPU.  The
tables are the seeded random tables of tests/test_gpu_gbuffer.py: every image-flag subset, every format, filter, mipmap and address
mode, mip chains, odd sizes and negative uv transforms.  The per-pixel geometry records come from the oracle's own decode; the GPU
tier and the emulated library check the device's geometry half."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oxylus_b200 import abi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


@pytest.fixture(scope="module")
def gb():
    import pyoracle_gbuffer

    pyoracle_gbuffer.build()
    return pyoracle_gbuffer


def _build(tmp_path, extra):
    exe = str(tmp_path / ("gbuffer_vs_oracle" + ("_fma" if extra else "")))
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wno-unknown-pragmas"] + (extra or ["-ffp-contract=off"]) +
                          ["-I", os.path.join(ROOT, "tests", "host_shim"), "-I", os.path.join(ROOT, "oxylus_b200", "csrc"),
                           os.path.join(ROOT, "tests", "gbuffer_vs_oracle.cpp"), "-o", exe])
    return exe


@pytest.fixture(scope="module")
def frames(orc, gb):
    """two frames (640 x 360), each with its own random table and its per-pixel records; a few mesh instances name a material
    outside the table and one mesh's vertex_count is lowered below its indices, so every outcome of a decoded pixel occurs"""
    from tests.test_gpu_gbuffer import random_images, random_materials, random_samplers

    out = []
    for seed in (21, 22):
        rng = np.random.default_rng(seed)
        sc = synth.make_scene(200_000, config_index=2, width=640, height=360, n_unique_meshes=16)
        sc.mesh_instances["material_index"] = rng.integers(0, 48, sc.mesh_instance_count)
        sc.mesh_instances["material_index"][::17] = 48
        hs = orc.HostScene(sc)
        cam = sc.camera(0.0)
        ref = orc.cpu_frame(hs, cam, sc.width, sc.height, np.zeros((sc.max_meshlet_instance_count + 31) // 32, np.uint32), None,
                            min(16, os.cpu_count() or 1))
        v32, _ = orc.resolve(ref["vis64"])
        total = int(ref["visibility"]["total"][0])
        hs.meshes["vertex_count"][1] = 3  # the scene's mesh 1 now indexes past its vertices: status 2
        images = random_images(rng)
        samplers = random_samplers(rng)
        mats = random_materials(rng, 48, len(images), len(samplers))
        table = orc.MaterialTable(mats, images, samplers)
        rec, mat = gb.decode_pixels(hs, ref["meshlet_instances"], total, cam, v32)
        want, bad = gb.decode_gbuffer(hs, ref["meshlet_instances"], total, cam, v32, table, init=np.float32(0.0))
        out.append(dict(mats=mats, images=images, samplers=samplers, table=table, cam=cam, rec=rec, mat=mat, want=want, bad=bad))
    return out


def _run(exe, tmp_path, fr, name):
    src, dst = tmp_path / f"{name}.in", tmp_path / f"{name}.out"
    with open(src, "wb") as f:
        f.write(np.uint32(len(fr["mats"])).tobytes() + np.ascontiguousarray(fr["mats"], dtype=abi.MATERIAL_DT).tobytes())
        f.write(np.uint32(len(fr["images"])).tobytes())
        for i in range(len(fr["images"])):
            im = fr["table"].images[i]
            t = fr["table"].texels[i]
            f.write(np.array([im["width"], im["height"], im["format"], im["level_count"]], np.uint32).tobytes() + np.uint64(t.size).tobytes() + t.tobytes())
        f.write(np.uint32(len(fr["samplers"])).tobytes() + np.ascontiguousarray(fr["samplers"], dtype=abi.SAMPLER_DT).tobytes())
        f.write(np.ascontiguousarray(fr["cam"]["position"][0], dtype=np.float32).tobytes())
        f.write(np.uint64(fr["mat"].size).tobytes() + fr["rec"].tobytes() + fr["mat"].tobytes())
    r = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout + r.stderr
    got = np.fromfile(dst, dtype=np.float32).reshape(fr["mat"].shape + (4, 4))
    return {k: got[:, :, i] for i, k in enumerate(abi.GBUFFER_PLANES)}


def test_device_source_equals_the_oracle_on_the_host(frames, tmp_path):
    exe = _build(tmp_path, None)
    for n, fr in enumerate(frames):
        got = _run(exe, tmp_path, fr, f"frame{n}")
        written = fr["mat"] != -1
        for k in abi.GBUFFER_PLANES:
            g, w = got[k][written], fr["want"][k][written]
            nan_g, nan_w = np.isnan(g), np.isnan(w)
            np.testing.assert_array_equal(nan_g, nan_w, err_msg=k)
            np.testing.assert_array_equal(np.where(nan_g, 0, g).view(np.uint32), np.where(nan_w, 0, w).view(np.uint32), err_msg=k)
        assert (fr["mat"] >= 0).sum() > 50_000 and (fr["mat"] == -2).sum() > 100 and fr["bad"] > 100
        assert (got["albedo"][fr["mat"] == -2] == 0).all()


def test_the_comparison_is_sensitive_to_contraction(frames, tmp_path):
    """the same source built WITH fma contraction disagrees with the oracle: fused multiply-adds break the canonical order"""
    flags = subprocess.run(["grep", "-c", "fma", "/proc/cpuinfo"], capture_output=True, text=True).stdout.strip()
    if flags in ("", "0"):
        pytest.skip("host CPU has no FMA unit")
    exe = _build(tmp_path, ["-mfma", "-ffp-contract=fast"])
    differ = 0
    for n, fr in enumerate(frames):
        got = _run(exe, tmp_path, fr, f"fma{n}")
        written = fr["mat"] != -1
        for k in abi.GBUFFER_PLANES:
            differ += int((got[k][written].view(np.uint32) != fr["want"][k][written].view(np.uint32)).sum())
    assert differ > 0
