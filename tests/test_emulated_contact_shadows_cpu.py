"""tests/test_gpu_contact_shadows.py in the CPU tier: the whole library compiled by g++ against the SIMT emulator (tests/build_emulated.py,
tests/host_shim/simt/), loaded through OXC_LIB_PATH, the GPU module run against it in a subprocess, in the emulator's default and in a
shuffled thread order.  It shows the launch's layout (8 x 4 pixel tiles per warp, 32 x 8 per CTA), its parameter set-up and argument
checks reproduce the oracle bit for bit under an independent execution model; it says nothing about GPU scheduling or speed.  The
full-size cases, the CUDA-graph test (torch) and the renderer frames stay with the GPU tier."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emulated(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import build_emulated

    lib = build_emulated.build(str(tmp_path_factory.mktemp("emu_contact")))
    return dict(os.environ, OXC_LIB_PATH=lib, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""),
                LD_LIBRARY_PATH=os.path.dirname(lib) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))


@pytest.mark.parametrize("order", ["default", "shuffle"])
def test_gpu_contact_shadows_on_the_simt_emulator(emulated, order):
    """the small sizes, the step counts, random and hostile settings, the box on a plane and the argument checks, against the oracle"""
    env = dict(emulated)
    if order == "shuffle":
        env["OXC_SIMT_ORDER"] = "shuffle"
    res = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_contact_shadows.py"), "-m", "gpu", "-q", "-x",
                          "-p", "no:cacheprovider", "-k", "1x1 or 17x9 or test_steps or random_settings or box_on_plane or argument_refusals"],
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    m = re.search(r"(\d+) passed", res.stdout)
    assert res.returncode == 0 and m and int(m.group(1)) >= 14 and "skipped" not in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]
