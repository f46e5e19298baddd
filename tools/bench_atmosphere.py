"""Atmosphere LUT timing on the H100: the transmittance bake (oxc_atmosphere_transmittance, 256 x 64 texels of 1000 steps) and the
per-frame sky view and aerial perspective (oxc_atmosphere_sky_luts, 312 x 192 and 32 x 32 x 32 texels in one launch) at the reference's
sizes and default record, with the camera at 2 m and at 10 km and the sun at 45 degrees.  CUDA-event times per call over --launches
launches after warm-up.  The outputs are checked against the oracle (oracle/pyoracle_atmosphere.py) in the same call, and the per-frame
cost is reported against the measured end-to-end frame of DESIGN §6 (0.610 ms on an H100 SXM).  Reads the card name and power limit in
the same run.  Prints one JSON line and writes it to --out.

    python tools/bench_atmosphere.py --launches 200 --out profiles/h100_atmosphere/bench_atmosphere.json
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from oxylus_b200 import abi, capi, synth  # noqa: E402

SUN = (0.0, 0.70710677, -0.70710677)  # 45 degrees above the horizon
FRAME_MS = 0.610                      # DESIGN §6: the measured end-to-end frame, H100 SXM


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
    t_shape, sv_shape, ap_shape = (64, 256, 4), (192, 312, 4), (32, 32, 32, 4)
    t, sv, apd = (ctx.alloc(int(np.prod(s)) * 2) for s in (t_shape, sv_shape, ap_shape))
    us_bake = timed(lambda: ctx.atmosphere_transmittance(atm, t), a.launches, a.warmup)
    lut = ctx.download(t, np.float16, int(np.prod(t_shape))).reshape(t_shape)
    res = dict(gpu=info, launches=a.launches, sizes=dict(transmittance=[256, 64], sky_view=[312, 192], aerial_perspective=[32, 32, 32]),
               bake=dict(us_call=round(us_bake, 2), march_steps=256 * 64 * 1000))
    if not a.no_oracle:
        import pyoracle_atmosphere as ao

        res["bake"]["oracle_equal"] = bool(np.array_equal(lut.view(np.uint16), ao.transmittance(atm).view(np.uint16)))
    runs = []
    for label, height in (("2m", 0.2), ("10km", 1000.0)):
        cam = camera_at(height)
        us = timed(lambda: ctx.atmosphere_sky_luts(atm, cam, SUN, 10.0, t, sv, apd), a.launches, a.warmup)
        steps = 312 * 192 * 48 + 32 * 32 * sum(2 * (z + 1) for z in range(32))
        run = dict(camera=label, us_call=round(us, 2), march_steps=steps, frame_share=round(us / (FRAME_MS * 1000.0), 4))
        if not a.no_oracle:
            import pyoracle_atmosphere as ao

            got_sv = ctx.download(sv, np.float16, int(np.prod(sv_shape))).reshape(sv_shape)
            got_ap = ctx.download(apd, np.float16, int(np.prod(ap_shape))).reshape(ap_shape)
            want_sv, want_ap = ao.sky_luts(atm, cam, SUN, 10.0, lut)
            run["oracle_equal"] = bool(np.array_equal(got_sv.view(np.uint16), want_sv.view(np.uint16)) and
                                       np.array_equal(got_ap.view(np.uint16), want_ap.view(np.uint16)))
        runs.append(run)
        print(json.dumps(run), file=sys.stderr)
    res["sky_luts"] = runs
    res["frame_ms"] = FRAME_MS
    for p in (t, sv, apd):
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
