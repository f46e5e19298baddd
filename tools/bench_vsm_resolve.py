"""Times the VSM shadow resolve (oxc_vsm_resolve_shadows) at the reference's shape: 64 x 64 pages x 10 clipmaps, 128-px pages, an
8192^2 atlas, clipmaps built as the reference builds them (synth.make_vsm_clipmaps).  Renderer frames (oxr_render, oxr_vsm_update_pages, oxr_vsm_draw_shadows) run until the page loop is steady, then the
resolve alone is timed with CUDA events over many launches on the renderer's own depth, decoded normals, page table and atlas, at
1920 x 1080 and 3840 x 2160, once on the synthetic scene alone (a view that is mostly sky) and once with a ground plane under the
camera (the lower part of the image receivers).  The share of pixels that ran the PCF loop is counted by the oracle on the same frame.  Prints one JSON
line.  Not bench.py: the flagship workload does not include the shadow path.

    python tools/bench_vsm_resolve.py [--launches 200]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power, clock = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        return dict(card=name, power_limit=power, sm_clock=clock)
    except Exception as e:  # noqa: BLE001
        return dict(card="unknown", power_limit="unknown", error=str(e))


def run(width, height, launches, ground):
    import torch

    import pyoracle_vsm_resolve as vr
    from oxylus_b200 import abi, capi, synth
    from test_gpu_vsm_pages import LIGHT, vsm_context

    capi.load()
    sc = synth.make_scene(20000, config_index=2, width=width, height=height, n_unique_meshes=32)
    if ground:  # a tessellated plane 2 m below the camera: the lower half of the image becomes receivers, as in a game frame
        sc = synth.with_ground_caster(sc, half_size=1200.0, center=(0.0, -2.0, -40.0), grid=32)
    r = capi.Renderer(0, sc)
    vsm = vsm_context(width=width, height=height)
    vsm["directional_light_dir"][0] = -np.float32(LIGHT)  # towards the light, as the reference's
    cam = sc.camera(0.0)
    clip = synth.make_vsm_clipmaps(-np.float64(LIGHT), cam["position"][0])  # forward Z, page-snapped, Shadowmaps.cpp:9-60
    coarse = np.zeros(1, dtype=abi.CULL_CAMERA_DT)  # clipmap 9's view (Shadowmaps.cpp:433-463)
    coarse["projection_view"][0] = clip["projection_view_mat"][9]
    coarse["position"][0] = -np.float64(LIGHT) / np.linalg.norm(LIGHT)
    coarse["acceptable_lod_error"], coarse["mesh_instance_count"], coarse["resolution"][0] = 2.0, sc.mesh_instance_count, (8192, 8192)
    inv_pv = np.linalg.inv(cam["projection_view"][0].reshape(4, 4).T.astype(np.float64)).T.astype(np.float32).reshape(16)
    res = cam["resolution"][0]
    for _ in range(4):  # the same view until no page is dirty any more
        out = r.render(cam, want_indices=False)
        pg = r.vsm_update_pages(vsm, clip, inv_pv, res, hpb_levels=7)
        r.vsm_draw_shadows(coarse)
    shadow = r.vsm_resolve_shadows(cam)  # decodes the normals into the renderer's plane
    ctx = r.ctx
    px = width * height
    normals_dev = ctx.alloc(px * 16)
    depth_dev = ctx.alloc(px * 4)
    shadow_dev = ctx.alloc(px * 4)
    # the renderer's decode plane is private: decode again into our own plane from the frame's R32UI image
    vis32_dev = ctx.alloc(px * 4)
    ctx.upload(vis32_dev, out["vis32"])
    ctx.decode_visbuffer(cam, width, height, dict(uv_normal=normals_dev), vis32_dev=vis32_dev)
    ctx.upload(depth_dev, out["depth"])
    args = (vsm, inv_pv, res, clip, depth_dev, normals_dev, pg.page_tables, pg.physical_atlas, shadow_dev)
    for _ in range(10):
        ctx.vsm_resolve_shadows(*args)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(5):
        t0.record()
        for _ in range(launches):
            ctx.vsm_resolve_shadows(*args)
        t1.record()
        t1.synchronize()
        times.append(t0.elapsed_time(t1) * 1e3 / launches)
    got = ctx.download(shadow_dev, np.float32, px).reshape(height, width)
    assert np.array_equal(got.view(np.uint32), shadow.view(np.uint32))
    pt = ctx.download(pg.page_tables, np.uint32, 10 * 64 * 64).reshape(10, 64, 64)
    atlas = ctx.download(pg.physical_atlas, np.float32, 8192 * 8192).reshape(8192, 8192)
    normals = ctx.download(normals_dev, np.float32, px * 4).reshape(height, width, 4)
    want, pcf = vr.vsm_resolve_shadows(vsm, inv_pv, res, clip, out["depth"], normals, pt, atlas)
    for p in (normals_dev, depth_dev, shadow_dev, vis32_dev):
        ctx.free(p)
    r.close()
    us = float(np.median(times))
    return dict(scene="instances + ground plane" if ground else "instances only", width=width, height=height, us_per_resolve=round(us, 2), us_runs=[round(t, 2) for t in times],
                pixels_per_s=round(px / (us * 1e-6)), pcf_share=round(float(pcf.mean()), 4), non_sky_share=round(float((out["depth"] != 0).mean()), 4),
                oracle_equal=bool(np.array_equal(want.view(np.uint32), shadow.view(np.uint32))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    a = ap.parse_args()
    rows = [run(w, h, a.launches, ground) for ground in (False, True) for (w, h) in ((1920, 1080), (3840, 2160))]
    print(json.dumps(dict(bench="vsm_resolve", shape="64x64 pages x 10 clipmaps, 128-px pages, 8192^2 atlas", **card(), results=rows)))


if __name__ == "__main__":
    main()
