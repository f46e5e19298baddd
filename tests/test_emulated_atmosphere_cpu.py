"""The atmosphere GPU module (tests/test_gpu_atmosphere.py) in the CPU tier: the whole library, from the product's own sources, compiled
by g++ against the SIMT emulator (tests/build_emulated.py, tests/host_shim/simt/) and loaded through OXC_LIB_PATH, as
tests/test_emulated_library_cpu.py does for the other passes.  It runs both atmosphere launches (the bake's row-major texels, the
per-frame launch's sky-view and aerial-perspective CTAs side by side), their parameters and their refusals at the odd and minimum sizes and
every camera height, once in the default fiber order and once shuffled; the reference sizes, the random and hostile records, the CUDA
graph and the renderer case stay on the GPU.  Each run reproduces the oracle bit for bit under an independent execution model; it says
nothing about GPU scheduling, memory ordering or speed."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SELECT = "odd or minimum or argument_refusals"
LEAST = 7  # test_sizes_and_heights at the odd and minimum sizes for three camera heights, and the refusals


@pytest.fixture(scope="module")
def emulated(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import build_emulated

    lib = build_emulated.build(str(tmp_path_factory.mktemp("emu")))
    return dict(os.environ, OXC_LIB_PATH=lib, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""),
                LD_LIBRARY_PATH=os.path.dirname(lib) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))


@pytest.mark.parametrize("order", ["default", "shuffle"])
def test_gpu_atmosphere_on_the_simt_emulator(emulated, order):
    env = dict(emulated)
    if order == "shuffle":
        env["OXC_SIMT_ORDER"] = "shuffle"  # the emulator resumes the threads of a block in a shuffled order
    res = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_atmosphere.py"), "-k", SELECT, "-m", "gpu", "-q",
                          "-x", "-p", "no:cacheprovider"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    m = re.search(r"(\d+) passed", res.stdout)
    passed = int(m.group(1)) if m else 0
    assert res.returncode == 0 and passed >= LEAST and "skipped" not in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]
