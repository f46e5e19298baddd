"""tests/test_gpu_gbuffer.py in the CPU tier: the whole library compiled by g++ against the SIMT emulator (tests/build_emulated.py,
tests/host_shim/simt/), loaded through OXC_LIB_PATH, the GPU module run against it in a subprocess, in the emulator's default and in a
shuffled thread order.  It runs k_decode_gbuffer's geometry half (decode_geometry), material half (gbuffer_shade), launch layout and
the C ABI's table building and argument checks against the oracle bit for bit: one random-table frame from both vis inputs, the
bad-vertex and bad-material cases, the refusals and the oracle-free checker quad.  It says nothing about GPU scheduling or speed; the
full-size frames, the CUDA-graph test (torch) and the renderer cases stay with the GPU tier."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ["test_random_tables_bit_exact[1]", "test_bad_material_and_refusals", "test_bad_vertex_index_writes_zeros",
         "test_checker_quad_at_texel_centres"]


@pytest.fixture(scope="module")
def emulated(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import build_emulated

    lib = build_emulated.build(str(tmp_path_factory.mktemp("emu_gbuffer")))
    return dict(os.environ, OXC_LIB_PATH=lib, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""),
                LD_LIBRARY_PATH=os.path.dirname(lib) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))


@pytest.mark.parametrize("order", ["default", "shuffle"])
def test_gpu_gbuffer_on_the_simt_emulator(emulated, order):
    env = dict(emulated)
    if order == "shuffle":
        env["OXC_SIMT_ORDER"] = "shuffle"
    ids = [os.path.join(ROOT, "tests", "test_gpu_gbuffer.py") + "::" + c for c in CASES]
    res = subprocess.run([sys.executable, "-m", "pytest"] + ids + ["-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"], cwd=ROOT, env=env,
                         capture_output=True, text=True, timeout=2400)
    m = re.search(r"(\d+) passed", res.stdout)
    assert res.returncode == 0 and m and int(m.group(1)) == len(CASES) and "skipped" not in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]
