"""Builds oxylus_b200/liboxcull.so (hand-written sm_90a kernels + C ABI + C++ host mirror) with nvcc.

In-tree build: the package loads the library from its own directory (the .so is git-ignored).
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# OXC_LIB_PATH: tuning sweeps load a variant built with OXC_NVCC_EXTRA overrides instead of the default library
LIB = os.environ.get("OXC_LIB_PATH") or os.path.join(HERE, "liboxcull.so")

SOURCES = [os.path.join(CSRC, "oxcull.cu"), os.path.join(CSRC, "host", "renderer_instance.cpp"),
           os.path.join(CSRC, "host", "mesh_builder.cpp"), os.path.join(CSRC, "host", "mesh_simplifier.cpp")]
DEPS = SOURCES + [
    os.path.join(CSRC, f)
    for f in ("oxc_types.cuh", "oxc_exact.cuh", "oxc_shader_math.cuh", "oxc_filtered.cuh", "oxc_raster_core.cuh", "kernels_cull.cuh", "kernels_decode.cuh", "kernels_hiz.cuh", "kernels_mgpu.cuh", "kernels_tri.cuh", "kernels_alpha.cuh", "kernels_vsm.cuh", "kernels_vsm_draw.cuh", "kernels_vsm_resolve.cuh", "kernels_gtao.cuh", "kernels_pbr.cuh", "kernels_contact_shadows.cuh", "kernels_atmosphere.cuh", "kernels_sky_ibl.cuh", "kernels_pbr_atmosphere.cuh", "kernels_exposure.cuh", "kernels_bloom.cuh", "kernels_tonemap.cuh", "kernels_fxaa.cuh", "kernels_terrain.cuh", "oxc_alpha.cuh", "oxc_gbuffer.cuh", "oxc_vsm_resolve.cuh", "oxc_gtao.cuh", "oxc_pbr.cuh", "oxc_contact_shadows.cuh", "oxc_atmosphere.cuh", "oxc_sky_ibl.cuh", "oxc_pbr_atmosphere.cuh", "oxc_exposure.cuh", "oxc_bloom.cuh", "oxc_tonemap.cuh", "oxc_fxaa.cuh", "oxc_terrain.cuh")
] + [os.path.join(CSRC, "host", "renderer_instance.hpp"), os.path.join(CSRC, "host", "mesh_simplifier.hpp"), os.path.join(os.path.dirname(HERE), "include", "oxcull.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--fmad=false",          # canonical arithmetic: no fma contraction (oracle/oxc_oracle.h)
    "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-ffp-contract=off", "-shared",
    "-Xptxas", "-v",
    "-ldl",  # NCCL is dlopen'ed by oxc_mgpu_init
]


def nvcc_path():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: liboxcull.so cannot be built (there is no CPU fallback)")


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    extra = os.environ.get("OXC_NVCC_EXTRA", "").split()  # tuning sweeps: -DOXC_... overrides of kernel constants
    cmd = [nvcc_path()] + NVCC_FLAGS + extra + ["-o", LIB] + SOURCES
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(HERE, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        sys.stderr.write(log)
        raise RuntimeError("nvcc failed building liboxcull.so")
    if verbose:
        print(log)
    return LIB


if __name__ == "__main__":
    build(force=True, verbose=True)
