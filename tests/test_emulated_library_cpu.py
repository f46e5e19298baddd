"""The GPU parity suite in the CPU tier: the WHOLE library — C ABI, host mirror and every CUDA kernel, from the product's own
sources — is compiled by g++ against a SIMT emulator (tests/host_shim/simt/cuda_runtime.h: every CUDA thread of a block is a
fiber, warp collectives and block barriers rendezvous cooperatively, atomics are real) and tests/test_gpu_parity.py runs against
it in a subprocess (OXC_LIB_PATH selects the library capi loads).  Same tests, same oracle, same bit-exact bar; only the sizes
are bounded (the big scenes and the multi-GPU / NCCL test stay with the GPU tier).

What this shows: the kernels' logic and arithmetic as written — queues, compaction, scans, the raster's scheduling, the clip and
chunk queues, the host mirror's frame loop — reproduce the oracle under an independent execution model, without a GPU.  What it
does not show: anything about GPU scheduling, memory ordering or speed.  TEST INFRASTRUCTURE: the emulated library is built into
a temporary directory and nothing in oxylus_b200/ knows about it; the product has no CPU path (test_abi_cpu.py checks that)."""
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# bounded for the CPU tier: no 1 M / 10 M / 17 M scenes, no 150 k-meshlet 1080p scene, no NCCL; host_min links -loxcull by name
SELECT = ("not full_size and not config and not medium and not wide_id and not mgpu and not plain_c_host "
          "and not small_primitive_cull_parity")


@pytest.fixture(scope="module")
def emulated(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import build_emulated

    lib = build_emulated.build(str(tmp_path_factory.mktemp("emu")))
    # LD_LIBRARY_PATH: the library dlopens "libnccl.so.2" — the in-process stand-in built next to it (multi-rank test)
    return dict(os.environ, OXC_LIB_PATH=lib, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""),
                LD_LIBRARY_PATH=os.path.dirname(lib) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))


def test_gpu_parity_suite_on_the_simt_emulator(emulated):
    env = emulated
    res = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_parity.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                          "-k", SELECT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = res.stdout[-3000:] + res.stderr[-2000:]
    assert res.returncode == 0, tail
    m = re.search(r"(\d+) passed", res.stdout)
    assert m and int(m.group(1)) >= 35 and "failed" not in res.stdout and "skipped" not in res.stdout, tail


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_path_on_the_simt_emulator(emulated, world):
    """oxc_mgpu_* with `world` emulated ranks (threads of one process, each with its own context; tests/emulated_mgpu_check.py):
    sharding with the communication-free id base, the Hi-Z exchange through the peers' buffers and flags, the vis-buffer max-reduce
    and the survivor allgather reproduce a single context over the whole scene bit for bit — image, survivor set, counters, every
    Hi-Z level on every rank, each rank's mask slice, three frames.  (4 ranks never ran on hardware this round: 2 and 8 did.)"""
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "emulated_mgpu_check.py"), str(world)], cwd=ROOT, env=emulated, capture_output=True,
                         text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    verdict = json.loads(res.stdout.strip().splitlines()[-1])
    assert verdict["pass"] and verdict["world"] == world and all(r["peer_memory"] for r in verdict["ranks"])


def test_multi_gpu_path_with_alpha_discard_on_the_simt_emulator(emulated):
    """the same check with a material table on every rank (visbuffer_encode.slang:54-66): each shard splits its own survivors by
    material (global ids minus the rank's id base), the discarded fragments' holes travel through the Hi-Z exchange and the
    vis-buffer merge — 2 emulated ranks equal one context bit for bit, and the table does change the image"""
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "emulated_mgpu_check.py"), "2", "12000", "alpha"], cwd=ROOT, env=emulated,
                         capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    verdict = json.loads(res.stdout.strip().splitlines()[-1])
    assert verdict["pass"] and verdict["alpha"] and verdict["world"] == 2


def test_plain_c_host_on_the_simt_emulator(emulated, tmp_path):
    """examples/host_min.c (plain C11 against include/oxcull.h) linked with the emulated library: the quad frame and the
    alpha-tested frame (oxc_set_materials from C) print what the GPU test expects from the real library"""
    lib = emulated["OXC_LIB_PATH"]
    exe = str(tmp_path / "host_min_emu")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "host_min.c"),
                           "-L", os.path.dirname(lib), "-l:" + os.path.basename(lib), "-Wl,-rpath," + os.path.dirname(lib), "-lm", "-o", exe])
    res = subprocess.run([exe, "alpha"], capture_output=True, text=True, timeout=120, env=emulated)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "768 of 3072 pixels" in res.stdout and "alpha-tested: 384 of 768 quad pixels kept, 0 pixels differ" in res.stdout


def test_hostile_inputs_on_the_simt_emulator(emulated):
    """tests/emulated_torture_check.py: NaN / Inf / negative / denormal MeshletBounds fields, garbage cones, degenerate and extreme
    transforms — two-pass frames still equal the oracle bit for bit (survivors, mask, packed image)."""
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "emulated_torture_check.py"), "1"], cwd=ROOT, env=emulated, capture_output=True,
                         text=True, timeout=1200)
    assert res.returncode == 0 and res.stdout.strip().endswith("ok"), res.stdout[-2000:] + res.stderr[-2000:]


def test_gpu_variants_on_the_simt_emulator(emulated):
    """tests/test_gpu_variants.py: all nine k_cull_meshlets instantiations over three pyramid states, every flag subset and a second
    camera, the occlusion toggle across frames, the mesh-level flags and the automatic shard id base, mixed cameras through the
    raster and the triangle cull.  Its hostile frames are the torture script's, which test_hostile_inputs_on_the_simt_emulator runs."""
    res = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_variants.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                          "-k", "not hostile_frames"], cwd=ROOT, env=emulated, capture_output=True, text=True, timeout=900)
    m = re.search(r"(\d+) passed", res.stdout)
    assert res.returncode == 0 and m and int(m.group(1)) >= 18 and "skipped" not in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]


def test_gpu_culls_on_the_simt_emulator(emulated):
    """tests/test_gpu_culls.py: the shadow-clipmap cull at every pyramid shape, dirty mask, page offset and clipmap count, steered
    page edges, shards, the engine's pass order with and without a bound device camera (the Renderer case runs eagerly here: no
    graph capture), the multi-view cull at 1-16 views, the terrain cull at every grid but 512 x 512, flag subset and Hi-Z state.
    All 17 of those cases must pass."""
    res = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_culls.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                          "-k", "not 512x512"], cwd=ROOT, env=emulated, capture_output=True, text=True, timeout=900)
    m = re.search(r"(\d+) passed", res.stdout)
    assert res.returncode == 0 and m and int(m.group(1)) >= 17 and "skipped" not in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]


@pytest.mark.parametrize("order", ["default", "shuffle"])
def test_gpu_raster_on_the_simt_emulator(emulated, order):
    """tests/test_gpu_raster.py at the emulator's grid (2 SMs, one raster CTA each: 1024 survivors start a pass at 32-meshlet
    grabs): the stress scene's frames and variants against the oracle, the triangle classes and the meshlet-run checks of
    oxc_set_scene.  Once more with OXC_SIMT_ORDER=shuffle (the emulator resumes the threads of a block in a shuffled order)."""
    env = dict(emulated, OXC_TEST_RASTER_MIN_SURVIVORS="1024")
    if order == "shuffle":
        env["OXC_SIMT_ORDER"] = "shuffle"
    res = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_raster.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"],
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    m = re.search(r"(\d+) passed", res.stdout)
    assert res.returncode == 0 and m and int(m.group(1)) >= 9 and "skipped" not in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]


def test_gpu_parity_suite_with_hostile_scenes_on_the_simt_emulator(emulated):
    """the same suite once more with OXC_TEST_HOSTILE_SCENES set (tests/conftest.py): every synthetic scene the tests build gets
    the hostile record contents above, vertex positions included — hpb / multiview / plain culls, triangle cull, clip and chunk
    queues, decode, the host mirror: every parity assertion still holds"""
    env = dict(emulated, OXC_TEST_HOSTILE_SCENES="7", OXC_TEST_HOSTILE_MODE="all")
    res = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_parity.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                          "-k", SELECT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    m = re.search(r"(\d+) passed", res.stdout)
    assert res.returncode == 0 and m and int(m.group(1)) >= 35, res.stdout[-3000:] + res.stderr[-2000:]
