#!/usr/bin/env python
"""Instrumentation run (variant library built with -DOXC_RASTER_STATS): per round of 32 triangles, how long is the longest
per-lane pixel loop, how many rounds run the triangle set-up, and how many meshlets draw anything?  Usage:  OXC_LIB_PATH=$PWD/oxylus_b200/liboxcull_stats.so python tools/raster_stats.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oxylus_b200 import abi, capi, pipeline, synth  # noqa: E402

scene = synth.make_scene(int(os.environ.get("N", 1_000_000)), config_index=2, width=1920, height=1080)
pipe = pipeline.VisibilityPipeline(scene, device=0)
cams = [scene.camera(0.0), scene.camera(2.0)]
for i in range(6):
    pipe.frame(cams[i % 2])
torch.cuda.synchronize()
n = 128
st0 = pipe.ctx.download(pipe.ctx.debug_stats_ptr(), np.uint64, n).copy()
frames = 4
for i in range(frames):
    pipe.frame(cams[i % 2])
torch.cuda.synchronize()
st = pipe.ctx.download(pipe.ctx.debug_stats_ptr(), np.uint64, n) - st0
for name, o in (("early", 0), ("late", 64)):
    h = st[o:o + 34].astype(np.float64)
    rounds = st[o + 43]
    print(f"--- {name}: rounds/frame {rounds / frames:.0f}  candidate px/round {st[o + 40] / max(1, rounds):.2f}  "
          f"mean max-lane px {st[o + 41] / max(1, rounds):.2f}  drawing lanes/round {st[o + 42] / max(1, rounds):.2f}  "
          f"deferred big tris/frame {st[o + 44] / frames:.0f}")
    print(f"   meshlets with a drawing triangle/frame {st[o + 46] / frames:.0f}  set-up rounds/frame {st[o + 47] / frames:.0f}")
    print("   histogram of max per-lane bbox area per round (0..32, 33+):")
    print("   " + " ".join(f"{int(x / frames)}" for x in h))
    cost_serial = float((h * np.arange(34)).sum())
    print(f"   sum of maxima = {cost_serial / frames:.0f} lane-pixel-iterations/frame on the critical path; balanced would be "
          f"{st[o + 40] / 32 / frames:.0f}")

# ---- per-warp timeline of the last frame's two raster launches (stats build only) ----
# the grid each launch used (statistics slot 45 of its half) x 8 warps per CTA; late records follow the early launch's
grids = pipe.ctx.download(pipe.ctx.debug_stats_ptr(), np.uint64, n)[[45, 64 + 45]].astype(np.int64)
assert grids[0] == grids[1] > 0, grids
nw = int(grids[0]) * 8
rec = pipe.ctx.download(pipe.ctx.debug_stats_ptr() + 128 * 8, np.uint64, 2 * nw * 6).reshape(2, nw, 6).astype(np.int64)
for name, r in (("early", rec[0]), ("late", rec[1])):
    r = r[r[:, 0] > 0]
    t0 = r[:, 0].min()
    dur = (r[:, 1] - r[:, 0]) / 1e3
    end = (r[:, 1] - t0) / 1e3
    print(f"--- {name} timeline: {len(r)} warps; kernel span {end.max():.1f} us; warp entry spread {(r[:, 0].max() - t0) / 1e3:.1f} us")
    print(f"   per-warp busy time us: mean {dur.mean():.1f} p50 {np.median(dur):.1f} p90 {np.percentile(dur, 90):.1f} max {dur.max():.1f}")
    print(f"   per-warp exit time us: p10 {np.percentile(end, 10):.1f} p50 {np.median(end):.1f} p90 {np.percentile(end, 90):.1f} p99 {np.percentile(end, 99):.1f}")
    print(f"   meshlets/warp mean {r[:, 4].mean():.1f} max {r[:, 4].max()}  grabs/warp mean {r[:, 5].mean():.1f}")
    print(f"   time in header chase {r[:, 2].sum() / max(1, r[:, 4].sum()) / 1e3:.2f} us/meshlet ({r[:, 2].sum() / max(1, r[:, 5].sum()) / 1e3:.2f} us/grab); "
          f"processing {r[:, 3].sum() / max(1, r[:, 4].sum()) / 1e3:.2f} us/meshlet")
    slow = np.argsort(-end)[:5]
    print("   slowest warps (exit us, meshlets, grabs, chase us, proc us):", [(round(float(end[i]), 1), int(r[i, 4]), int(r[i, 5]), round(r[i, 2] / 1e3, 1), round(r[i, 3] / 1e3, 1)) for i in slow])
