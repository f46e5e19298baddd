"""Atmospheric PBR apply timing on the H100: oxc_apply_pbr_atmosphere beside oxc_apply_pbr in the same run, on renderer frames of the
benchmark's synthetic scene (20,000 instances) over a ground plane (synth.with_ground_caster, 2 m under the camera, as
tools/bench_pbr.py), 1080p and 4K, 0, 16 and 256 lights (synth.make_lights), the sun at 45 degrees.  The sky tables are made on the
device by the library's own calls at the reference's extents: the transmittance bake, the per-frame sky-view and aerial-perspective
LUTs and two sky IBL updates.  Inputs are those of tools/bench_pbr.py.  CUDA-event times over --launches launches after --warmup, then
the kernel time from torch.profiler in a separate run.  At 1080p every output of both passes is checked against its oracle in the same
command.  The card's name, power limit and clocks are read in the same call.  Prints one JSON line and writes it to --out.

    python tools/bench_pbr_atmosphere.py --launches 200 --out profiles/h100_pbr_atmosphere/bench_pbr_atmosphere.json
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

LIGHT_COUNTS = (0, 16, 256)
SUN = (0.0, float(np.float32(np.sqrt(0.5))), float(np.float32(np.sqrt(0.5))))  # 45 degrees above the horizon


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def time_call(fn, launches, warmup, kernel):
    import torch
    from torch.profiler import ProfilerActivity, profile

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(torch.cuda.current_stream())
    for _ in range(launches):
        fn()
    e1.record(torch.cuda.current_stream())
    torch.cuda.synchronize()
    us_call = e0.elapsed_time(e1) * 1000.0 / launches
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(launches):
            fn()
        torch.cuda.synchronize()
    us_kernel = None
    for ev in prof.key_averages():
        if kernel + "(" in ev.key or kernel + "E" in ev.key:  # demangled or mangled; k_apply_pbr( is not k_apply_pbr_atmosphere(
            us_kernel = round(ev.device_time_total / max(ev.count, 1), 2)
    return round(us_call, 2), us_kernel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()

    capi.load()
    runs = []
    at = abi.atmosphere()
    for w, h in ((1920, 1080), (3840, 2160)):
        sc = synth.with_ground_caster(synth.make_scene(20000, config_index=2, width=w, height=h, n_unique_meshes=32), half_size=1200.0,
                                      center=(0.0, -2.0, -40.0))
        r = capi.Renderer(0, sc)
        cam = sc.camera(0.0)
        out = r.render(cam, want_indices=False)
        depth = out["depth"].copy()
        proj, view = synth.camera_matrices(w, h, 0.0)
        ao = r.generate_ambient_occlusion(cam, abi.gtao_camera(proj, view, 1000.0), abi.gtao_settings(3))
        r.close()
        hw, hh = sc.hiz_extent()
        ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
        ctx.set_scene(sc)
        px = w * h
        un_dev, v32_dev = ctx.alloc(px * 16), ctx.alloc(px * 4)
        ctx.upload(v32_dev, out["vis32"])
        ctx.cull_meshes(cam)
        ctx.decode_visbuffer(cam, w, h, {"uv_normal": un_dev}, vis32_dev=v32_dev)
        uvn = ctx.download(un_dev, np.float32, px * 4).reshape(h, w, 4)
        rng = np.random.default_rng(w)
        planes = dict(depth=depth, albedo=rng.random((h, w, 4), dtype=np.float32),
                      normal=np.ascontiguousarray(np.concatenate([uvn[..., 2:], uvn[..., 2:]], -1)),
                      emissive=(rng.random((h, w, 4), dtype=np.float32) * (rng.random((h, w, 1)) < 0.05)).astype(np.float32),
                      metallic_roughness_occlusion=rng.random((h, w, 4), dtype=np.float32), ambient_occlusion=ao,
                      shadow=np.where(rng.random((h, w)) < 0.4, 0.0, 1.0).astype(np.float32))
        inputs = {}
        for k, v in planes.items():
            inputs[k] = ctx.alloc(v.nbytes)
            ctx.upload(inputs[k], v)
        out_dev = ctx.alloc(px * 16)
        lights_all = synth.make_lights(np.random.default_rng(7), max(LIGHT_COUNTS))
        lights_dev = ctx.alloc(64 * max(LIGHT_COUNTS))
        ctx.upload(lights_dev, np.frombuffer(bytes(lights_all), np.uint8))
        pcam = synth.pbr_camera(cam)
        # the sky tables, made on the device at the reference's extents
        t, sv, apx = at.transmittance_lut_size, at.sky_view_lut_size, at.aerial_perspective_lut_size
        sky = dict(transmittance=ctx.alloc(t[0] * t[1] * 8), sky_view=ctx.alloc(sv[0] * sv[1] * 8),
                   aerial_perspective=ctx.alloc(apx[0] * apx[1] * apx[2] * 8), sky_cube=ctx.alloc(abi.SKY_IBL_CUBE_BYTES))
        ctx.upload(sky["sky_cube"], np.zeros(abi.SKY_IBL_CUBE_BYTES, np.uint8))
        ctx.atmosphere_transmittance(at, sky["transmittance"])
        ctx.atmosphere_sky_luts(at, pcam, SUN, 10.0, sky["transmittance"], sky["sky_view"], sky["aerial_perspective"])
        for f in range(2):
            ctx.atmosphere_sky_ibl(at, pcam, SUN, 10.0, abi.SKY_IBL_SUN_AMBIENT_STRENGTH, f, sky["transmittance"], sky["sky_view"], sky["sky_cube"])
        ctx.sync()
        host_sky = [ctx.download(sky["transmittance"], np.float16, t[0] * t[1] * 4).reshape(t[1], t[0], 4),
                    ctx.download(sky["sky_view"], np.float16, sv[0] * sv[1] * 4).reshape(sv[1], sv[0], 4),
                    ctx.download(sky["aerial_perspective"], np.float16, apx[0] * apx[1] * apx[2] * 4).reshape(apx[2], apx[1], apx[0], 4),
                    ctx.download(sky["sky_cube"], np.float16, 6 * 32 * 32 * 4).reshape(6, 32, 32, 4)]
        for n in LIGHT_COUNTS:
            base = abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_GTAO
            st = abi.pbr_settings(scene_flags=base, sun_direction=SUN, sun_intensity=10.0, light_count=n)
            sta = abi.pbr_settings(scene_flags=base | abi.SCENE_HAS_ATMOSPHERE, sun_direction=SUN, sun_intensity=10.0, light_count=n)
            calls = dict(apply_pbr=(lambda: ctx.apply_pbr(pcam, st, lights_dev, inputs, w, h, out_dev), "k_apply_pbr"),
                         apply_pbr_atmosphere=(lambda: ctx.apply_pbr_atmosphere(pcam, sta, at, lights_dev, inputs, sky, w, h, out_dev),
                                               "k_apply_pbr_atmosphere"))
            run = dict(width=w, height=h, lights=n, camera_y=round(float(pcam.position[1]), 3), depth_pixels=int((depth != 0).sum()))
            for name, (fn, kernel) in calls.items():
                us_call, us_kernel = time_call(fn, a.launches, a.warmup, kernel)
                run[name] = dict(us_call=us_call, us_kernel=us_kernel, pixels_per_s=round(px / (us_call * 1e-6)))
                if w == 1920 and not a.no_oracle:
                    fn()
                    ctx.sync()
                    got = ctx.download(out_dev, np.float32, px * 4).reshape(h, w, 4)
                    args = [planes[k] for k in ("depth", "albedo", "normal", "emissive", "metallic_roughness_occlusion", "ambient_occlusion",
                                                "shadow")] + [None]
                    if name == "apply_pbr":
                        import pyoracle_pbr

                        want = pyoracle_pbr.apply_pbr(pcam, st, lights_all, *args)
                    else:
                        import pyoracle_pbr_atmosphere

                        want = pyoracle_pbr_atmosphere.apply_pbr_atmosphere(pcam, sta, at, lights_all, *args, *host_sky)
                    run[name]["oracle_equal"] = bool(np.array_equal(got.view(np.uint32), want.view(np.uint32)))
            run["atmosphere_over_apply_pbr"] = round(run["apply_pbr_atmosphere"]["us_call"] / run["apply_pbr"]["us_call"], 3)
            runs.append(run)
            print(json.dumps(run), file=sys.stderr)
        for p in list(inputs.values()) + list(sky.values()) + [out_dev, lights_dev, un_dev, v32_dev]:
            ctx.free(p)
        ctx.close()
    res = dict(gpu=gpu_info(), launches=a.launches, sun=SUN, runs=runs)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
