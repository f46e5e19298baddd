"""The terrain draw's GPU module (tests/test_gpu_terrain_draw.py) in the CPU tier: the whole library, from the product's own sources,
compiled by g++ against the SIMT emulator (tests/build_emulated.py, tests/host_shim/simt/) and loaded through OXC_LIB_PATH, with the
emulated build of tests/test_emulated_library_cpu.py.  It runs k_draw_terrain's own scheduling — thread 0 setting the patch up in shared
memory and the barriers around its copy, the grid-stride patch slots, the device-side instance count, the chunk queue (big_push) and
k_raster_big — on the small cases (the 1 x 1 and 3 x 7 grids, a frame of meshlet words with depth ties in both packings, hostile
settings, counts and indices) and the refusals, once in the default fiber order and once shuffled; the full sizes, the 256 x 256 grid,
the CUDA graph and the renderer stay on the GPU.  Each run reproduces the oracle bit for bit under an independent execution model; it
says nothing about GPU scheduling, memory ordering or speed."""
import os
import re
import subprocess
import sys

import pytest

from tests.test_emulated_library_cpu import ORDERS, ROOT, emulated  # noqa: F401 (emulated: the module-scoped fixture)

SELECT = "1x1 or 3x7 or meshlet_frame or hostile or refusals"
LEAST = 5  # the two small grids, the meshlet frame, the hostile cases, the refusals


@pytest.mark.parametrize("order", ORDERS)
def test_gpu_terrain_draw_on_the_simt_emulator(emulated, order):  # noqa: F811
    env = dict(emulated)
    if order == "shuffle":
        env["OXC_SIMT_ORDER"] = "shuffle"  # the emulator resumes the threads of a block in a shuffled order
    res = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_terrain_draw.py"), "-k", SELECT, "-m", "gpu",
                          "-q", "-x", "-p", "no:cacheprovider"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    m = re.search(r"(\d+) passed", res.stdout)
    passed = int(m.group(1)) if m else 0
    assert res.returncode == 0 and passed >= LEAST and "skipped" not in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]
