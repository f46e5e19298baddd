"""Tonemap timing on the H100: oxc_tonemap on the benchmark scene's lit frame (tools/bench_post.py lit_frame: 20,000 instances over a
ground plane, oxc_apply_pbr with HasDirectionalLight | HasGTAO and 16 lights), with its HasEyeAdaptation and HasBloom inputs made on
the device (oxc_eye_adaptation's record and oxc_bloom's upsampled level 0 of the same frame), at 1080p and 4K.  Each curve runs with
the lens effects off and with all three on; CUDA-event times per call over --launches calls after --warmup.  Every output is checked
against the oracle (oracle/pyoracle_tonemap.py) in the same call unless --no-oracle.  Bytes moved are the algorithmic lower bound (16 B
read and 16 B written per pixel, plus the bloom image read once) over the 3.35 TB/s data-sheet bandwidth.  Reads the card name and
power limit in the same run.  Prints one JSON line and writes it to --out.

    python tools/bench_tonemap.py --launches 200 --out profiles/h100_tonemap/bench_tonemap.json
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
from oxylus_b200 import abi, capi  # noqa: E402

EA, BL = abi.SCENE_HAS_EYE_ADAPTATION, abi.SCENE_HAS_BLOOM
LENS = abi.SCENE_HAS_CHROMATIC_ABERRATION | abi.SCENE_HAS_VIGNETTE | abi.SCENE_HAS_FILM_GRAIN
TYPES = (("none", abi.TONEMAP_NONE), ("aces", abi.TONEMAP_ACES), ("agx", abi.TONEMAP_AGX), ("gt7", abi.TONEMAP_GT7))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    capi.load()
    res = dict(gpu=gpu_info(), launches=a.launches, warmup=a.warmup, hbm_bytes_per_s=HBM_BYTES_PER_S, runs=[])
    for w, h in ((1920, 1080), (3840, 2160)):
        ctx, lit = lit_frame(w, h)
        px, n = w * h, abi.bloom_chain_texels(w, h)
        rec, hist, down, up, out = ctx.alloc(8), ctx.alloc(1024), ctx.alloc(n * 16), ctx.alloc(n * 16), ctx.alloc(px * 16)
        ctx.upload(rec, np.frombuffer(bytes(abi.Exposure(1.0, 1.0)), np.uint8))
        ctx.eye_adaptation(lit, w, h, abi.eye_adaptation_settings(), 0.016, rec, hist)
        ctx.bloom(lit, w, h, abi.bloom_settings(scene_flags=EA), rec, down, up)
        ctx.sync()
        nbytes = px * 32 + (w // 2) * (h // 2) * 16
        host = record = image = None
        if not a.no_oracle:
            import pyoracle_tonemap as so

            host = ctx.download(lit, np.float32, px * 4).reshape(h, w, 4)
            record = abi.Exposure.from_buffer_copy(ctx.download(rec, np.uint8, 8).tobytes())
            image = ctx.download(up, np.float32, (w // 2) * (h // 2) * 4).reshape(h // 2, w // 2, 4)
        for name, t in TYPES:
            for lens in (0, LENS):
                s = abi.tonemap_settings(EA | BL | lens, t, film_grain_seed=3)

                def call():
                    ctx.tonemap(lit, w, h, s, rec, up, out)

                us = timed(call, a.launches, a.warmup)
                run = dict(extent=[w, h], curve=name, lens=bool(lens), bytes=nbytes, us=round(us, 2),
                           bound_us=round(nbytes / HBM_BYTES_PER_S * 1e6, 2), bound_share=round(nbytes / HBM_BYTES_PER_S * 1e6 / us, 3))
                if not a.no_oracle:
                    call()
                    got = ctx.download(out, np.float32, px * 4).reshape(h, w, 4)
                    run["oracle_equal"] = bool(np.array_equal(got.view(np.uint32), so.tonemap(host, s, record, image).view(np.uint32)))
                res["runs"].append(run)
                print(json.dumps(run), file=sys.stderr)
        for p in (lit, rec, hist, down, up, out):
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
