"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol include/oxcull.h
declares, the header is valid C, and — with no GPU — the product path FAILS LOUDLY (no CPU fallback)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oxylus_b200 import abi, capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "oxcull.h")


def _has_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ox[bcr]_[a-z0-9_]+)\s*\(", src)))


def test_header_is_valid_c_and_cxx():
    for lang, std in (("c", "-std=c11"), ("c++", "-std=c++17")):
        subprocess.check_call(["gcc", "-fsyntax-only", "-x", lang, std, "-Wall", "-Werror", HEADER])


def test_library_exports_every_declared_symbol():
    lib = capi.load()
    decl = declared_symbols()
    assert len(decl) >= 25
    assert sorted(capi.SYMBOLS) == decl, "capi.SYMBOLS and include/oxcull.h disagree"
    for s in decl:
        assert hasattr(lib, s), f"liboxcull.so does not export {s}"
    assert lib.oxc_version().decode().startswith("oxcull")


def test_struct_sizes_match_reference_layouts():
    # SceneGPU.hpp scalar-layout sizes (SURVEY §8)
    assert abi.MESHLET_BOUNDS_DT.itemsize == 16 and abi.MESH_DT.itemsize == 64 and abi.MESH_LOD_DT.itemsize == 64
    assert abi.CULL_CAMERA_DT.itemsize == 96 and abi.MESH_INSTANCE_DT.itemsize == 20 and abi.VISIBILITY_DT.itemsize == 12
    assert C.sizeof(abi.CreateInfo) == 32 and C.sizeof(abi.SceneDesc) == 64
    assert abi.MESH_DT.fields["bounds"][1] == 40 and abi.MESH_LOD_DT.fields["error"][1] == 60
    assert abi.MESHLET_BOUNDS_DT.fields["aabb_extent"][1] == 8 and abi.MESHLET_BOUNDS_DT.fields["cone_cutoff"][1] == 15
    # Material (SceneGPU.hpp:67-82, 56 B: flags at 20, albedo_image_index at 28, uv_size at 48) and the tables of oxc_set_materials
    assert abi.MATERIAL_DT.itemsize == 56 and abi.MATERIAL_DT.fields["flags"][1] == 20 and abi.MATERIAL_DT.fields["alpha_cutoff"][1] == 18
    assert abi.MATERIAL_DT.fields["albedo_image_index"][1] == 28 and abi.MATERIAL_DT.fields["uv_size"][1] == 48
    assert abi.ALPHA_IMAGE_DT.itemsize == 24 and abi.SAMPLER_DT.itemsize == 20 and C.sizeof(abi.MaterialTable) == 48


def test_hiz_extent_and_layout():
    # RendererInstance.cpp:573-577: bit_ceil((W+1)>>1)
    assert abi.hiz_extent(1920, 1080) == (1024, 1024)
    assert abi.hiz_extent(3840, 2160) == (2048, 2048)
    assert abi.hiz_extent(640, 360) == (512, 256)
    assert abi.hiz_extent(1, 1) == (1, 1)
    levels, offs, total = abi.hiz_layout(1024, 1024)
    assert levels == 11 and offs[1] == 1024 * 1024 and total == sum((1024 >> l) ** 2 for l in range(11))
    assert abi.hiz_layout(8192, 8192)[0] == 13  # min(mips, 13)


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_no_gpu_fails_loudly():
    lib = capi.load()
    info = abi.CreateInfo(4, 64, 64, 64, 0, 0)
    h = C.c_void_p()
    rc = lib.oxc_create(0, C.byref(info), C.byref(h))
    assert rc == capi.E_NO_DEVICE and not h.value
    assert b"no CPU fallback" in lib.oxc_last_error()
    with pytest.raises(capi.OxcError):
        capi.Context(0, 4, 64, 64, 64)
    r = C.c_void_p()
    assert lib.oxr_create(0, C.byref(info), 64, 64, C.byref(r)) != 0 and not r.value


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under oxylus_b200/ may reference oracle/."""
    pkg = os.path.join(ROOT, "oxylus_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".hpp", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                for needle in ("pyoracle", "oxc_oracle", "liboxc_oracle", "orc_"):
                    if needle == "orc_" and f.endswith(".py"):
                        continue
                    assert needle not in txt or "oracle/" in txt and needle not in re.sub(r"(#|//|/\*|\"\"\").*", "", txt), (f, needle)
    out = subprocess.run(["nm", "-D", "--undefined-only", capi.lib_path()], capture_output=True, text=True).stdout
    assert "orc_" not in out


def test_product_never_uses_the_test_emulator():
    """tests/host_shim/ (host stand-ins for the CUDA headers, the SIMT emulator) is test infrastructure: nothing under oxylus_b200/
    includes it, builds it or loads an emulated library, and the shipped liboxcull.so is the nvcc build (it holds sm_90a device
    code and none of the emulator's symbols).  The only trace in the product sources is the OXC_HOST_SOUNDNESS_HARNESS guard around
    inline PTX, which no product build defines."""
    pkg = os.path.join(ROOT, "oxylus_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".hpp", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                for needle in ("host_shim", "liboxcull_emu", "build_emulated", "simt::", "fake_nccl"):
                    assert needle not in txt, (f, needle)
    assert "OXC_HOST_SOUNDNESS_HARNESS" not in open(os.path.join(pkg, "build.py")).read()
    syms = subprocess.run(["nm", "-DC", capi.lib_path()], capture_output=True, text=True).stdout
    assert "simt::" not in syms
    if shutil.which("cuobjdump"):
        elf = subprocess.run(["cuobjdump", "-lelf", capi.lib_path()], capture_output=True, text=True).stdout
        assert "sm_90a" in elf, elf[:300]


def _build_host_min(tmp_path):
    exe = str(tmp_path / "host_min")
    libdir = os.path.dirname(capi.lib_path())
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "host_min.c"), "-L", libdir, "-loxcull", f"-Wl,-rpath,{libdir}", "-lm", "-o", exe])
    return exe


def test_plain_c_mesh_import_example(tmp_path):
    """examples/mesh_import.c: the builder side of the ABI (oxb_*: clusteriser + generated LOD chain) from plain C11 — pure host
    code, so it runs to completion without a GPU."""
    capi.load()
    exe = str(tmp_path / "mesh_import")
    libdir = os.path.dirname(capi.lib_path())
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "mesh_import.c"), "-L", libdir, "-loxcull", f"-Wl,-rpath,{libdir}", "-lm", "-o", exe])
    res = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and res.stdout.strip().endswith("ok"), res.stdout + res.stderr
    assert "lods 8" in res.stdout


def test_plain_c_host_compiles_links_and_fails_loudly_without_gpu(tmp_path):
    """examples/host_min.c: a C11 host using nothing but include/oxcull.h.  Without a CUDA device it must stop at oxc_create
    with the no-device error (exit code 3), never silently compute on the CPU."""
    capi.load()
    exe = _build_host_min(tmp_path)
    if _has_gpu():
        pytest.skip("GPU present: covered by the gpu-marked test")
    res = subprocess.run([exe], capture_output=True, text=True)
    assert res.returncode == 3 and "no CUDA device" in res.stderr
