import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))  # test modules share mesh helpers (test_builder_cpu.torus / parse)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def orc():
    import pyoracle

    pyoracle.build()
    pyoracle.lib()
    return pyoracle


@pytest.fixture(scope="session")
def small_scene():
    from oxylus_b200 import synth

    return synth.make_scene(6000, config_index=2, width=640, height=360, n_unique_meshes=16)


# OXC_TEST_HOSTILE_SCENES=<seed>: every synthetic scene the tests build gets hostile MeshletBounds fields / cones / transforms
# (tests/emulated_torture_check.py: mutate).  Used by tests/test_emulated_library_cpu.py for a second pass of the GPU parity suite on the
# SIMT-emulated library; unset (the driver's GPU tier, every ordinary run) = no effect.
if os.environ.get("OXC_TEST_HOSTILE_SCENES"):
    import numpy as _np

    import emulated_torture_check as _etc
    from oxylus_b200 import synth as _synth

    _orig_make_scene = _synth.make_scene

    def _hostile_make_scene(*a, **k):
        return _etc.mutate(_orig_make_scene(*a, **k), _np.random.default_rng(int(os.environ["OXC_TEST_HOSTILE_SCENES"])), os.environ.get("OXC_TEST_HOSTILE_MODE", "all"))

    _synth.make_scene = _hostile_make_scene
