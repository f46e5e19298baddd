#!/usr/bin/env python
"""Extra measurements for the other BASELINE.json configs (not the driver's bench line):
  config 4: 16 views x 5M meshlet instances, one batched multi-view cull launch (bounds read once)
Prints one JSON line per measurement."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oxylus_b200 import abi, capi, synth  # noqa: E402


def multiview(n_meshlets=5_000_000, n_views=16, iters=20):
    sc = synth.make_scene(n_meshlets, config_index=4, width=1920, height=1080, placement="box")
    hw, hh = sc.hiz_extent()
    ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh, max_views=n_views,
                       stream=torch.cuda.current_stream().cuda_stream)
    ctx.set_scene(sc)
    cam = sc.camera()
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    total = int(ctx.visibility()["total"][0])
    dirs = synth.uniform(sc.seed, 90, 3 * n_views, -1.0, 1.0).reshape(n_views, 3)
    dirs[:, 1] = -np.abs(dirs[:, 1]) - 0.2
    views = np.concatenate([synth.make_ortho_view(dirs[v], (0.0, 0.0, -200.0), 60.0 * (1 + v % 4), 800.0, sc.mesh_instance_count)
                            for v in range(n_views)])
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(3):
        ctx.cull_meshlets_multiview(views, 1)
    torch.cuda.synchronize()
    ms = []
    for i in range(iters):
        flush.fill_(i)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ctx.cull_meshlets_multiview(views, 1)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    t = float(np.median(ms)) * 1e-3
    counts = ctx.view_counts()[:n_views]
    algo = total * 24 + total * 4 + n_views * sc.mesh_instance_count * 96
    peak = _peak()
    print(json.dumps({"workload": f"multi-view cull: {n_views} ortho views x {total} meshlet instances, directional cone + frustum per view",
                      "ms_per_launch_incl_plane_prepare": t * 1e3, "meshlet_view_tests_per_s": total * n_views / t,
                      "meshlets_per_s": total / t, "algorithmic_bytes": algo, "achieved_gbs": algo / t / 1e9, "frac_of_measured_hbm": algo / t / 1e9 / peak,
                      "visible_per_view": [int(c) for c in counts]}), flush=True)
    ctx.close()


def _peak():
    f = os.path.join(ROOT, "MEASURED_PEAKS.json")
    return json.load(open(f))["hbm_gbs"] if os.path.exists(f) else 3350.0  # H100 SXM data sheet (HBM3)


def _time(fn, iters, flush):
    ms = []
    for i in range(iters):
        flush.fill_(i)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)) * 1e-3


def decode(n_meshlets=1_000_000, iters=20):
    """vis-buffer decode (visbuffer_decode.slang geometry part) of the steady-state configs[1] frame at 1920x1080"""
    sc = synth.make_scene(n_meshlets, config_index=2, width=1920, height=1080)
    r = capi.Renderer(0, sc)
    r.set_external_depth(sc.occluder_depth)
    cam = sc.camera()
    for _ in range(4):
        got = r.render(cam, None)
    ctx = r.ctx
    ctx.stream = 0
    w, h = sc.width, sc.height
    v32 = torch.from_numpy(got["vis32"].view(np.int32)).cuda()
    planes = [torch.empty((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(5)]
    tg = dict(zip(("lambda_", "ddx", "ddy", "uv_normal", "uv_grad"), [p.data_ptr() for p in planes]))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for _ in range(3):
        ctx.decode_visbuffer(cam, w, h, tg, vis32_dev=v32.data_ptr())
    torch.cuda.synchronize()
    t = _time(lambda: ctx.decode_visbuffer(cam, w, h, tg, vis32_dev=v32.data_ptr()), iters, flush)
    t1 = _time(lambda: ctx.decode_visbuffer(cam, w, h, {"lambda_": tg["lambda_"]}, vis32_dev=v32.data_ptr()), iters, flush)
    covered = int((planes[0][:, :, 3] == 1.0).sum().item())
    algo = w * h * (4 + 80)
    print(json.dumps({"workload": f"vis-buffer decode {w}x{h}, {covered} covered pixels, 5 float4 planes out",
                      "ms_per_launch": t * 1e3, "pixels_per_s": w * h / t, "algorithmic_bytes": algo, "achieved_gbs": algo / t / 1e9,
                      "frac_of_measured_hbm": algo / t / 1e9 / _peak(), "ms_per_launch_lambda_plane_only": t1 * 1e3}), flush=True)
    r.close()


def hpb(size=128, layers=10, levels=8, iters=20):
    """hierarchical page bitmap build (rmvsm_downsample_hpb.slang, all levels, one launch)"""
    ctx = capi.Context(0, 4, 64, 64, 64, stream=0)
    rng = np.random.default_rng(3)
    pt = torch.from_numpy(rng.integers(0, 8, size=(layers, size, size)).astype(np.int32)).cuda()
    total = sum(layers * max(1, size >> l) ** 2 for l in range(levels))
    out = torch.empty(total, dtype=torch.uint8, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(3):
        ctx.build_hpb(pt.data_ptr(), size, layers, out.data_ptr(), levels)
    torch.cuda.synchronize()
    t = _time(lambda: ctx.build_hpb(pt.data_ptr(), size, layers, out.data_ptr(), levels), iters, flush)
    print(json.dumps({"workload": f"page bitmap build {layers} x {size}x{size}, {levels} levels, one launch", "us_per_build": t * 1e6}), flush=True)
    ctx.close()


if __name__ == "__main__":
    which = sys.argv[1:] or ["multiview"]
    for w_ in which:
        {"multiview": multiview, "decode": decode, "hpb": hpb}[w_]()
