"""bench.py contract on CPU: the reference arm (`--impl reference`) runs without a GPU (it times the oracle port) and
prints ONE JSON line with the contract's keys; the product arm refuses to run without a CUDA device."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_json_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--meshlets", "20000", "--width", "640",
                          "--height", "360", "--steps", "1", "--warmup", "1"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.strip().splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["metric"] == "meshlet_instances_culled_per_s" and d["higher_is_better"] is True
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["value"] > 0 and d["vs_baseline"] is None and "workload" in d["config"]


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"], capture_output=True,
                         text=True, timeout=120, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""


def test_product_arm_needs_a_gpu():
    try:
        import torch

        if torch.cuda.is_available():
            return
    except Exception:
        pass
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "1"], capture_output=True, text=True,
                         timeout=300)
    assert out.returncode != 0 and "no CPU fallback" in (out.stderr + out.stdout)


def _bench_module():
    import importlib.util

    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _frame_like(h, w, rng):
    import numpy as np

    return {"vis_depth": rng.random((h, w), dtype=np.float32), "vis_id": rng.integers(0, 2**32, (h, w)).astype(np.float64),
            "survivor_ids": np.arange(300_000, dtype=np.float64), "counters": np.array([1e6, 2.6e5, 3.5e4, 1.2e7]),
            "visibility_mask": rng.integers(0, 2**32, 31250).astype(np.float64), "hiz": rng.random(1398101, dtype=np.float32)}


def test_dump_outputs_whole_when_small(tmp_path):
    import numpy as np

    bench = _bench_module()
    arrays = _frame_like(1080, 1920, np.random.default_rng(1))
    bench.dump_outputs(str(tmp_path), arrays)
    for name, a in arrays.items():
        got = np.load(tmp_path / f"{name}.npy")
        assert got.dtype == a.dtype and np.array_equal(got, a), name


def test_dump_outputs_4k_fits_64mb_with_a_fixed_sample(tmp_path):
    """A 3840x2160 frame is ~110 MB: large arrays keep the same seeded sample on every call, small ones stay whole."""
    import numpy as np

    bench = _bench_module()
    arrays = _frame_like(2160, 3840, np.random.default_rng(2))
    assert sum(a.nbytes for a in arrays.values()) > 64 << 20
    dirs = [tmp_path / "a", tmp_path / "b"]
    for d in dirs:
        bench.dump_outputs(str(d), arrays)
        assert sum(f.stat().st_size for f in d.iterdir()) <= 64 << 20
    for name, a in arrays.items():
        x, y = (np.load(d / f"{name}.npy") for d in dirs)
        assert x.dtype == a.dtype and np.array_equal(x, y), name
        if a.nbytes < 1 << 20:
            assert np.array_equal(x, a), name
        else:
            assert 0 < x.size < a.size and np.isin(x, a.ravel()).all(), name


def test_reference_arm_honours_steps_and_rejects_dump(tmp_path):
    args = [sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--meshlets", "20000", "--width", "640", "--height", "360"]
    out = subprocess.run(args + ["--steps", "6", "--warmup", "0"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    d = json.loads(out.stdout.strip().splitlines()[-1])
    assert d["steps"] == 6 and d["warmup"] == 0
    out = subprocess.run(args + ["--steps", "1", "--dump-outputs", str(tmp_path / "d")], capture_output=True, text=True, timeout=600)
    assert out.returncode != 0 and "--dump-outputs" in out.stderr and not (tmp_path / "d").exists()
