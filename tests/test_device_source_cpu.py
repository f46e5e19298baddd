"""The kernels' canonical arithmetic (csrc/oxc_exact.cuh), compiled for the HOST, against the CPU oracle — bit for bit, no GPU.

tests/device_vs_oracle.cpp includes the device headers through tests/host_shim/ (each __f*_rn intrinsic = one IEEE binary32
operation) and links oracle/liboxc_oracle.so: dequantize_half (all 65 536 inputs, both decoders), mat4 products, frustum
planes + test, project_aabb, test_occlusion, canonical log2, ceil(log2), the backface determinant; tests/raster_core_vs_oracle.cpp
does the same for the software raster's per-triangle core (csrc/oxc_raster_core.cuh).  The GPU tier checks the same source as
compiled by nvcc; this is the CPU-tier half of that statement."""
import subprocess

from tests.host_harness import compile_harness, skip_without_fma


def test_device_headers_equal_the_oracle_on_the_host(orc, tmp_path):
    exe = compile_harness(tmp_path, "device_vs_oracle", link_oracle=True)
    res = subprocess.run([exe, "300000"], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and res.stdout.strip().endswith("ok"), res.stdout + res.stderr


def test_the_comparison_is_sensitive_to_contraction(orc, tmp_path):
    """the same program built WITH fma contraction must disagree: one fused multiply-add anywhere breaks the canonical order"""
    skip_without_fma()
    exe = compile_harness(tmp_path, "device_vs_oracle", contract=True, link_oracle=True)
    res = subprocess.run([exe, "50000"], capture_output=True, text=True, timeout=600)
    assert res.returncode == 1 and "FAILED" in res.stdout


def test_raster_core_equals_the_oracle_on_the_host(orc, tmp_path):
    """csrc/oxc_raster_core.cuh (snapping, set-up, 32 / 64-bit stepped and direct edge functions, tie-break, depth, packed max,
    clipping) compiled for the host draws the same images as the oracle's raster specification, pixel for pixel: 300 000 random
    triangles from sub-pixel to screen-filling, shared edges, vertices behind the camera and outside the snap range"""
    exe = compile_harness(tmp_path, "raster_core_vs_oracle", link_oracle=True)
    res = subprocess.run([exe, "300000"], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and res.stdout.strip().endswith("ok"), res.stdout + res.stderr
    assert " 0 differ" in res.stdout and "(0 path disagreements)" in res.stdout and " 0 small-primitive disagreements" in res.stdout
