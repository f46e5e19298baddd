"""FXAA's GPU module (tests/test_gpu_fxaa.py) in the CPU tier: the whole library, from the product's own sources, compiled by g++ against
the SIMT emulator (tests/build_emulated.py, tests/host_shim/simt/) and loaded through OXC_LIB_PATH, with the emulated build of
tests/test_emulated_library_cpu.py.  It runs k_fxaa's 8 x 4 pixel tiles per warp, the divergent walk and the per-call parameters on the
small cases (every frame kind with every tap count, the tiny extents, hostile frames) and the refusals, once in the default fiber order
and once shuffled; the full sizes, 1919 x 1079, the CUDA graph and the renderer chain stay on the GPU.  Each run reproduces the oracle bit for bit under an independent execution model;
it says nothing about GPU scheduling, memory ordering or speed."""
import os
import re
import subprocess
import sys

import pytest

from tests.test_emulated_library_cpu import ORDERS, ROOT, emulated  # noqa: F401 (emulated: the module-scoped fixture)

SELECT = "small or argument_refusals"
LEAST = 8  # every frame kind, the five tiny extents, hostile frames, the refusals


@pytest.mark.parametrize("order", ORDERS)
def test_gpu_fxaa_on_the_simt_emulator(emulated, order):  # noqa: F811
    env = dict(emulated)
    if order == "shuffle":
        env["OXC_SIMT_ORDER"] = "shuffle"  # the emulator resumes the threads of a block in a shuffled order
    res = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_fxaa.py"), "-k", SELECT, "-m", "gpu", "-q",
                          "-x", "-p", "no:cacheprovider"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    m = re.search(r"(\d+) passed", res.stdout)
    passed = int(m.group(1)) if m else 0
    assert res.returncode == 0 and passed >= LEAST and "skipped" not in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]
