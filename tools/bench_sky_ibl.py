"""Sky IBL cube timing on the H100: oxc_atmosphere_sky_ibl (one thread per texel and sample, 6 x 32 x 32 texels of 64 samples) against
the one-thread-per-texel form (tools/ubench/sky_ibl_serial.cu, compiled here into a temporary directory with the library's flags), both
over the reference's LUT sizes (transmittance 256 x 64, sky view 312 x 192) made on the device with the default record, the camera at
2 m and at 10 km and the sun at 45 degrees.  CUDA-event times per call over --launches launches after warm-up.  Both forms' cubes are
checked against the oracle (oracle/pyoracle_sky_ibl.py) in the same call, for a first call from a zeroed cube and a second with history.
Reads the card name and power limit in the same run.  Prints one JSON line and writes it to --out.

    python tools/bench_sky_ibl.py --launches 200 --out profiles/h100_sky_ibl/bench_sky_ibl.json
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from oxylus_b200 import abi, build, capi, synth  # noqa: E402

SUN = (0.0, 0.70710677, -0.70710677)  # 45 degrees above the horizon
STRENGTH = abi.SKY_IBL_SUN_AMBIENT_STRENGTH


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def camera_at(height):
    proj, view = synth.camera_matrices(1920, 1080, 0.0, eye=(0.0, height, 0.0))
    inv = np.linalg.inv(synth.mat_mul_cm(proj, view).reshape(4, 4).T.astype(np.float64)).T.astype(np.float32).reshape(16)
    return abi.pbr_camera(inv, (0.0, height, 0.0))


def timed(fn, launches, warmup):
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(torch.cuda.current_stream())
    for _ in range(launches):
        fn()
    e1.record(torch.cuda.current_stream())
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / launches


def serial_lib(tmp):
    """the one-thread-per-texel form, built with the library's nvcc flags into tmp"""
    so = os.path.join(tmp, "libsky_ibl_serial.so")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-ldl",)]
    res = subprocess.run([build.nvcc_path()] + flags + ["-o", so, os.path.join(ROOT, "tools", "ubench", "sky_ibl_serial.cu")],
                         capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed on sky_ibl_serial.cu:\n" + res.stderr)
    regs = [ln.strip() for ln in res.stderr.splitlines() if "registers" in ln or "spill" in ln]
    lib = C.CDLL(so)
    vp = C.c_void_p
    lib.sky_ibl_serial.argtypes = [C.POINTER(abi.Atmosphere), C.POINTER(abi.PbrCamera), vp, C.c_float, C.c_float, C.c_uint32, vp, vp, vp, vp]
    lib.sky_ibl_serial.restype = C.c_int
    return lib, regs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    capi.load()
    info = gpu_info()
    sc = synth.make_scene(200, config_index=2, width=64, height=64, n_unique_meshes=4)
    hw, hh = sc.hiz_extent()
    ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
    atm = abi.atmosphere()
    t_shape, sv_shape, ap_shape, cube_shape = (64, 256, 4), (192, 312, 4), (32, 32, 32, 4), abi.SKY_IBL_CUBE_SHAPE
    t, sv, apd, cube = (ctx.alloc(int(np.prod(s)) * 2) for s in (t_shape, sv_shape, ap_shape, cube_shape))
    sun = (C.c_float * 3)(*SUN)
    zero = np.zeros(cube_shape, np.float16)
    res = dict(gpu=info, launches=a.launches, cube=[6, 32, 32], samples=64, sizes=dict(transmittance=[256, 64], sky_view=[312, 192]))
    with tempfile.TemporaryDirectory() as tmp:
        serial, regs = serial_lib(tmp)
        res["serial_ptxas"] = regs
        ctx.atmosphere_transmittance(atm, t)
        runs = []
        for label, height in (("2m", 0.2), ("10km", 1000.0)):
            cam = camera_at(height)
            ctx.atmosphere_sky_luts(atm, cam, SUN, 10.0, t, sv, apd)

            def shipped(frame=7):
                ctx.atmosphere_sky_ibl(atm, cam, SUN, 10.0, STRENGTH, frame, t, sv, cube)

            def one_per_texel(frame=7):
                rc = serial.sky_ibl_serial(C.byref(atm), C.byref(cam), sun, 10.0, STRENGTH, frame, C.c_void_p(t), C.c_void_p(sv),
                                           C.c_void_p(cube), None)
                assert rc == 0, rc

            run = dict(camera=label)
            for name, fn in (("sample_parallel", shipped), ("texel_serial", one_per_texel), ("sample_parallel_again", shipped),
                             ("texel_serial_again", one_per_texel)):
                ctx.upload(cube, zero)
                run[f"us_{name}"] = round(timed(fn, a.launches, a.warmup), 2)
            if not a.no_oracle:
                import pyoracle_sky_ibl as so

                lut = ctx.download(t, np.float16, int(np.prod(t_shape))).reshape(t_shape)
                svh = ctx.download(sv, np.float16, int(np.prod(sv_shape))).reshape(sv_shape)
                want = so.sky_ibl(atm, cam, SUN, 10.0, STRENGTH, 0, lut, svh)
                want2 = so.sky_ibl(atm, cam, SUN, 10.0, STRENGTH, 1, lut, svh, want)
                for name, fn in (("sample_parallel", shipped), ("texel_serial", one_per_texel)):
                    ctx.upload(cube, zero)
                    fn(0)
                    got = ctx.download(cube, np.float16, zero.size).reshape(cube_shape)
                    fn(1)
                    got2 = ctx.download(cube, np.float16, zero.size).reshape(cube_shape)
                    run[f"oracle_equal_{name}"] = bool(np.array_equal(got.view(np.uint16), want.view(np.uint16)) and
                                                       np.array_equal(got2.view(np.uint16), want2.view(np.uint16)))
            runs.append(run)
            print(json.dumps(run), file=sys.stderr)
        res["runs"] = runs
    for p in (t, sv, apd, cube):
        ctx.free(p)
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
