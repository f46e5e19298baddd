"""FXAA timing on the H100: oxc_fxaa on three frames at 1080p and 4K.  The lit frame is the benchmark scene's (tools/bench_post.py
lit_frame: 20,000 instances over a ground plane, oxc_apply_pbr with HasDirectionalLight | HasGTAO and 16 lights), the realistic case; a
flat frame, where every pixel exits early, is the floor; high-contrast noise, where nearly every pixel walks, is the ceiling.  CUDA-event
times per call over --launches calls after --warmup.  Per frame the oracle (oracle/pyoracle_fxaa.py) counts on the host the share of
edge pixels (those past the early exit) and the mean bilinear taps per pixel, and checks the device output bit for bit.  Bytes moved are
the algorithmic lower bound (16 B read and 16 B written per pixel) over the 3.35 TB/s data-sheet bandwidth.  Reads the card name and
power limit in the same run.  Prints one JSON line and writes it to --out.

    python tools/bench_fxaa.py --launches 200 --out profiles/h100_fxaa/bench_fxaa.json
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

from bench_post import HBM_BYTES_PER_S, gpu_info, lit_frame, timed  # noqa: E402
from oxylus_b200 import capi  # noqa: E402


def flat_frame(w, h):
    return np.broadcast_to(np.float32([0.8, 0.5, 0.3, 1.0]), (h, w, 4)).copy()


def noise_frame(w, h, seed=7):
    rng = np.random.default_rng(seed)
    f = np.where(rng.random((h, w, 1)) < 0.5, np.float32(0.0), rng.uniform(0.5, 8.0, (h, w, 1))).astype(np.float32)
    return np.concatenate([f * rng.uniform(0.5, 1.0, (h, w, 3)), rng.uniform(0, 1, (h, w, 1))], axis=2).astype(np.float32)


def main():
    import pyoracle_fxaa as so

    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    capi.load()
    res = dict(gpu=gpu_info(), launches=a.launches, warmup=a.warmup, hbm_bytes_per_s=HBM_BYTES_PER_S, runs=[])
    for w, h in ((1920, 1080), (3840, 2160)):
        ctx, lit = lit_frame(w, h)
        px = w * h
        out = ctx.alloc(px * 16)
        for name in ("lit", "flat", "noise"):
            if name == "lit":
                frame, host = lit, ctx.download(lit, np.float32, px * 4).reshape(h, w, 4)
            else:
                host = flat_frame(w, h) if name == "flat" else noise_frame(w, h)
                frame = ctx.alloc(px * 16)
                ctx.upload(frame, host)
            want, taps = so.fxaa(host, with_taps=True)

            def call():
                ctx.fxaa(frame, w, h, out)

            us = timed(call, a.launches, a.warmup)
            call()
            got = ctx.download(out, np.float32, px * 4).reshape(h, w, 4)
            nbytes = px * 32
            run = dict(extent=[w, h], frame=name, bytes=nbytes, us=round(us, 2), bound_us=round(nbytes / HBM_BYTES_PER_S * 1e6, 2),
                       bound_share=round(nbytes / HBM_BYTES_PER_S * 1e6 / us, 3), edge_share=round(float((taps > 5).mean()), 4),
                       mean_taps=round(float(taps.mean()), 2), oracle_equal=bool(np.array_equal(got.view(np.uint32), want.view(np.uint32))))
            res["runs"].append(run)
            print(json.dumps(run), file=sys.stderr)
            if name != "lit":
                ctx.free(frame)
        ctx.free(out)
        ctx.free(lit)
        ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
