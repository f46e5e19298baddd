"""PBR apply timing on the H100: oxc_apply_pbr alone on renderer frames of the benchmark's synthetic scene (20,000 instances) over a
ground plane (synth.with_ground_caster), 1080p and 4K, HasDirectionalLight | HasGTAO with 0, 16, 64 and 256 lights (synth.make_lights).
Inputs: the frame's depth; its decoded world normal (oxc_decode_visbuffer's uv_normal .zw) in both halves of the normal plane; the
renderer's GTAO; seeded albedo, emissive, metallic / roughness / occlusion and shadow planes.  CUDA-event times over --launches
launches after --warmup, then the kernel time from torch.profiler in a separate run.  At 1080p every light count's output is checked
against the oracle (oracle/pyoracle_pbr.py) in the same command.  The cost per light per pixel is the least-squares slope of the four
light counts.  Prints one JSON line and writes it to --out.

    python tools/bench_pbr.py --launches 200 --out profiles/h100_pbr/bench_pbr.json
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

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
LIGHT_COUNTS = (0, 16, 64, 256)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def algorithmic_bytes(w, h):
    """bytes the pass must move at least, from shapes: depth, ambient occlusion and shadow (4 B each) and four float4 planes (64 B) read,
    one float4 written; the lights (<= 16 KiB per CTA, from L2) are not counted"""
    px = w * h
    return dict(read=px * 76, written=px * 16, total=px * 92, floor_us=round(px * 92 / HBM_BYTES_PER_S * 1e6, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    capi.load()
    runs = []
    for w, h in ((1920, 1080), (3840, 2160)):
        sc = synth.with_ground_caster(synth.make_scene(20000, config_index=2, width=w, height=h, n_unique_meshes=32), half_size=1200.0,
                                      center=(0.0, -2.0, -40.0))  # 2 m under the camera, as tools/bench_gtao.py
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
        per_count = []
        for n in LIGHT_COUNTS:
            st = abi.pbr_settings(scene_flags=abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_GTAO, light_count=n)
            for _ in range(a.warmup):
                ctx.apply_pbr(pcam, st, lights_dev, inputs, w, h, out_dev)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(torch.cuda.current_stream())
            for _ in range(a.launches):
                ctx.apply_pbr(pcam, st, lights_dev, inputs, w, h, out_dev)
            e1.record(torch.cuda.current_stream())
            torch.cuda.synchronize()
            us_call = e0.elapsed_time(e1) * 1000.0 / a.launches
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.launches):
                    ctx.apply_pbr(pcam, st, lights_dev, inputs, w, h, out_dev)
                torch.cuda.synchronize()
            us_kernel = None
            for ev in prof.key_averages():
                if "k_apply_pbr" in ev.key:
                    us_kernel = round(ev.device_time_total / max(ev.count, 1), 2)
            run = dict(width=w, height=h, lights=n, us_call=round(us_call, 2), us_kernel=us_kernel, depth_pixels=int((depth != 0).sum()),
                       pixels_per_s=round(px / (us_call * 1e-6)), bytes=algorithmic_bytes(w, h))
            if w == 1920 and not a.no_oracle:
                import pyoracle_pbr

                got = ctx.download(out_dev, np.float32, px * 4).reshape(h, w, 4)
                want = pyoracle_pbr.apply_pbr(pcam, st, lights_all, planes["depth"], planes["albedo"], planes["normal"], planes["emissive"],
                                              planes["metallic_roughness_occlusion"], planes["ambient_occlusion"], planes["shadow"], None)
                run["oracle_equal"] = bool(np.array_equal(got.view(np.uint32), want.view(np.uint32)))
            per_count.append(run)
            runs.append(run)
            print(json.dumps(run), file=sys.stderr)
        # cost per light per pixel: least-squares slope of the call time over the light count
        x = np.float64([r_["lights"] for r_ in per_count])
        y = np.float64([r_["us_call"] for r_ in per_count])
        slope, icpt = np.polyfit(x, y, 1)
        runs.append(dict(width=w, height=h, fit_us_at_0_lights=round(icpt, 2), fit_us_per_light=round(slope, 3),
                         ns_per_light_per_mpixel=round(slope * 1e3 / (px / 1e6), 3)))
        print(json.dumps(runs[-1]), file=sys.stderr)
        for p in list(inputs.values()) + [out_dev, lights_dev, un_dev, v32_dev]:
            ctx.free(p)
        ctx.close()
    res = dict(gpu=gpu_info(), launches=a.launches, runs=runs)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
