"""Terrain draw timing on the H100: oxc_draw_terrain on the reference's default terrain (1024 m, a 2048 x 2048 heightmap, 64 x 64
patches, target 16 px, max 64; tests/helpers_terrain.py builds a seeded one: smooth hills with 0.2 m of texel noise, and, with
--rough, 40 m of texel noise as a worst case) at 1080p and 4K from three cameras: 2 m above the ground
looking at the horizon, an aerial view, and a grazing view.  The patches come from oxc_cull_terrain (frustum test, as the late pass of a
frame with a cleared Hi-Z sees them).  CUDA-event times per call over --launches calls after --warmup, each call drawing into the same
vis buffer (the packed max leaves it unchanged, every atomic still runs).  Per view the oracle (oracle/pyoracle_terrain_draw.py) counts
the triangles and the pixels the terrain writes and checks the device's vis buffer bit for bit.  Reads the card name and power limit in
the same run.  Prints one JSON line and writes it to --out.

    python tools/bench_terrain.py --launches 50 --out profiles/h100_terrain/bench_terrain.json
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_post import gpu_info, timed  # noqa: E402
from oxylus_b200 import abi, capi  # noqa: E402
from tests import helpers_terrain as ht  # noqa: E402


def main():
    import pyoracle_terrain_draw as so

    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--rough", action="store_true", help="texel noise of 10 percent of the height range (40 m spikes 0.5 m apart) instead of 0.2 m")
    a = ap.parse_args()
    capi.load()
    hm = ht.heightmap(2048, 2048, 7, texel_noise=0.1 if a.rough else ht.DEFAULT_TEXEL_NOISE)
    t = ht.terrain()
    mm = ht.patch_minmax(hm, (64, 64))
    st = ht.settings(t)
    res = dict(gpu=gpu_info(), launches=a.launches, warmup=a.warmup, terrain="1024 m, 2048^2 R16, 64 x 64 patches, 16 px, max 64",
               texel_noise_m=400.0 * (0.1 if a.rough else ht.DEFAULT_TEXEL_NOISE),
               runs=[])
    ctx = capi.Context(0, 1, 1, 64, 64)
    ctx.clear_hiz()
    n = 4096
    hm_dev, mm_dev = ctx.alloc(hm.nbytes), ctx.alloc(mm.nbytes)
    ctx.upload(hm_dev, hm)
    ctx.upload(mm_dev, mm)
    vp, mp, cp = ctx.alloc(n * 4), ctx.alloc(128 * 4), ctx.alloc(16)
    for w, h in ((1920, 1080), (3840, 2160)):
        vis = ctx.alloc(w * h * 8)
        for name, cam in ht.views(hm, t, w, h).items():
            ctx.upload(mp, np.zeros(128, np.uint32))
            ctx.cull_terrain(t, mm_dev, cam, abi.CULL_TEST_FRUSTUM | abi.CULL_LATE_PASS, vp, mp, cp)
            count = int(ctx.download(cp, np.uint32, 4)[1])
            visible = ctx.download(vp, np.uint32, n)
            ctx.clear_visbuffer(vis, w, h)

            def call():
                ctx.draw_terrain(hm_dev, 2048, 2048, st, vp, cp, cam, w, h, vis)

            call()
            got = ctx.download(vis, np.uint64, w * h).reshape(h, w)
            want = np.full((h, w), 0xFFFFFFFF, np.uint64)
            tris = so.draw_terrain(hm, st, visible, count, cam, want)
            us = timed(call, a.launches, a.warmup)
            run = dict(extent=[w, h], view=name, patches=count, triangles=tris, pixels=int((want != 0xFFFFFFFF).sum()), us=round(us, 1),
                       oracle_equal=bool(np.array_equal(got, want)))
            res["runs"].append(run)
            print(json.dumps(run), file=sys.stderr)
        ctx.free(vis)
    for p in (hm_dev, mm_dev, vp, mp, cp):
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
