"""GTAO timing on the H100: oxc_generate_ambient_occlusion on renderer frames of the benchmark's synthetic scene (20,000 instances)
over a ground plane (synth.with_ground_caster), so that about half the pixels hold depth; 1080p and 4K, each preset.  Per pass (the
prefilter, the sector pass, the denoise) and for the whole call: CUDA-event times over --launches launches after warm-up.  The 1080p
outputs are checked against the oracle (oracle/pyoracle_gtao.py) for each preset.  Prints one JSON line and writes it to --out.

    python tools/bench_gtao.py --launches 200 --out profiles/h100_gtao/bench_gtao.json
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


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def algorithmic_bytes(w, h, slices, samples):
    """bytes each pass must move at least, from shapes: the prefilter reads depth and writes the mips; the sector pass reads the
    centre mip-0 texel, the normal and 2 x slices x samples x 2 trilinear taps (8 texels each, counted as requested bytes, mostly from
    L2) and writes edges and binary16 occlusion; the denoise reads 9 occlusion and 5 edge texels (each fetched once from DRAM) and
    writes the final plane"""
    _, mips = abi.gtao_mip_layout(w, h)
    px = w * h
    return dict(prefilter_dram=px * 4 + mips * 4, main_dram=px * 4 + px * 16 + px * 4 + px * 2,
                main_taps_requested=px * slices * samples * 2 * 8 * 4, denoise_dram=px * 2 + px * 4 + px * 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    import torch

    capi.load()
    runs = []
    for w, h in ((1920, 1080), (3840, 2160)):
        sc = synth.with_ground_caster(synth.make_scene(20000, config_index=2, width=w, height=h, n_unique_meshes=32), half_size=1200.0,
                                      center=(0.0, -2.0, -40.0))  # 2 m under the camera, as tools/bench_vsm_resolve.py
        r = capi.Renderer(0, sc)
        cam = sc.camera(0.0)
        out = r.render(cam, want_indices=False)
        depth = out["depth"].copy()
        proj, view = synth.camera_matrices(w, h, 0.0)
        gcam = abi.gtao_camera(proj, view, 1000.0)
        ao_renderer = r.generate_ambient_occlusion(cam, gcam, abi.gtao_settings(3))
        r.close()
        # the frame's uv_normal plane on a context of its own, as oxr_generate_ambient_occlusion decodes it
        hw, hh = sc.hiz_extent()
        ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
        ctx.set_scene(sc)
        px = w * h
        normals_dev = ctx.alloc(px * 16)
        v32_dev = ctx.alloc(px * 4)
        ctx.upload(v32_dev, out["vis32"])
        ctx.cull_meshes(cam)
        ctx.decode_visbuffer(cam, w, h, {"uv_normal": normals_dev}, vis32_dev=v32_dev)
        normals = ctx.download(normals_dev, np.float32, px * 4).reshape(h, w, 4)
        depth_dev = ctx.alloc(px * 4)
        ctx.upload(depth_dev, depth)
        _, total = abi.gtao_mip_layout(w, h)
        t = abi.GtaoTargets(ctx.alloc(total * 4), ctx.alloc(px * 4), ctx.alloc(px * 2), ctx.alloc(px * 4))
        for preset in range(4):
            st = abi.gtao_settings(preset)
            for _ in range(a.warmup):
                ctx.generate_ambient_occlusion(gcam, st, depth_dev, normals_dev, w, h, t)
            torch.cuda.synchronize()
            # whole call
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(torch.cuda.current_stream())
            for _ in range(a.launches):
                ctx.generate_ambient_occlusion(gcam, st, depth_dev, normals_dev, w, h, t)
            e1.record(torch.cuda.current_stream())
            torch.cuda.synchronize()
            us_call = e0.elapsed_time(e1) * 1000.0 / a.launches
            # per pass from the profiler's kernel records
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.launches):
                    ctx.generate_ambient_occlusion(gcam, st, depth_dev, normals_dev, w, h, t)
                torch.cuda.synchronize()
            per = {}
            for ev in prof.key_averages():
                for k in ("k_gtao_prefilter", "k_gtao_main", "k_gtao_denoise"):
                    if k in ev.key:
                        per[k] = round(ev.device_time_total / max(ev.count, 1), 2)
            slices, samples = abi.GTAO_PRESETS[preset]
            run = dict(width=w, height=h, preset=preset, slices=slices, samples_per_side=samples, us_call=round(us_call, 2),
                       us_prefilter=per.get("k_gtao_prefilter"), us_main=per.get("k_gtao_main"), us_denoise=per.get("k_gtao_denoise"),
                       depth_pixels=int((depth != 0).sum()), pixels_per_s=round(px / (us_call * 1e-6)), bytes=algorithmic_bytes(w, h, slices, samples))
            if w == 1920 and not a.no_oracle:
                import pyoracle_gtao

                want = pyoracle_gtao.generate_ambient_occlusion(gcam, st, depth, normals)
                got = ctx.download(t.ambient_occlusion, np.float32, px).reshape(h, w)
                noisy = ctx.download(t.noisy_occlusion, np.uint16, px).reshape(h, w)
                run["oracle_equal"] = bool(np.array_equal(got.view(np.uint32), want["ao"].view(np.uint32)) and np.array_equal(noisy, want["noisy"]))
            if preset == 3:
                got = ctx.download(t.ambient_occlusion, np.float32, px).reshape(h, w)
                run["renderer_equal"] = bool(np.array_equal(got.view(np.uint32), ao_renderer.view(np.uint32)))
            runs.append(run)
            print(json.dumps(run), file=sys.stderr)
        for p in (normals_dev, v32_dev, depth_dev, t.depth_mips, t.edges, t.noisy_occlusion, t.ambient_occlusion):
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
