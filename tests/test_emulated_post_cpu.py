"""The post-processing GPU module (tests/test_gpu_post.py) in the CPU tier: the whole library, from the product's own sources, compiled by g++
against the SIMT emulator (tests/build_emulated.py, tests/host_shim/simt/) and loaded through OXC_LIB_PATH, as
tests/test_emulated_sky_ibl_cpu.py does for the sky IBL cube.  It runs the histogram's warp-aggregated shared-memory atomics (__match_any_sync,
__popc, __ffs, atomicAdd), the average's shuffles and barrier, and the bloom's per-level launches and single-CTA tail with its barriers,
on the small cases (hostile frames and settings, the uniform frame, the adaptation sequence, the caller's last upsampled level) and the
refusals, once in the default fiber order and once shuffled; the reference sizes, the wrapping frame, the CUDA graph and the renderer
stay on the GPU.  Each run reproduces the oracle bit for bit under an independent execution model; it says nothing about GPU scheduling,
memory ordering or speed."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SELECT = "small or argument_refusals"
LEAST = 5  # the hostile frames, the uniform frame, the adaptation sequence, the last upsampled level, the refusals


@pytest.fixture(scope="module")
def emulated(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import build_emulated

    lib = build_emulated.build(str(tmp_path_factory.mktemp("emu")))
    return dict(os.environ, OXC_LIB_PATH=lib, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""),
                LD_LIBRARY_PATH=os.path.dirname(lib) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))


@pytest.mark.parametrize("order", ["default", "shuffle"])
def test_gpu_post_on_the_simt_emulator(emulated, order):
    env = dict(emulated)
    if order == "shuffle":
        env["OXC_SIMT_ORDER"] = "shuffle"  # the emulator resumes the threads of a block in a shuffled order
    res = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_post.py"), "-k", SELECT, "-m", "gpu", "-q",
                          "-x", "-p", "no:cacheprovider"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    m = re.search(r"(\d+) passed", res.stdout)
    passed = int(m.group(1)) if m else 0
    assert res.returncode == 0 and passed >= LEAST and "skipped" not in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]
