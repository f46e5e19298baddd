"""Contact-shadow timing on the H100: oxc_contact_shadows on renderer frames of the benchmark's synthetic scene (20,000 instances) over a
ground plane (synth.with_ground_caster), so that about half the pixels hold depth; 1080p and 4K, steps 8 (the reference's default), 16
and 64, with a low sun behind the casters and the reference's thickness (0.1) over a 0.5 m ray, so that rays on the ground run to the
step count.  CUDA-event times per call over --launches launches after warm-up.  The 1080p outputs are checked against the oracle
(oracle/pyoracle_contact_shadows.py) and oxr_contact_shadows' output.  Reads the card name and power limit in the same run.  Prints
one JSON line and writes it to --out.

    python tools/bench_contact_shadows.py --launches 200 --out profiles/h100_contact_shadows/bench_contact_shadows.json
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

SUN = (0.2, 0.3, -1.0)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def contact_camera(w, h):
    proj, view = synth.camera_matrices(w, h, 0.0)
    inv = np.linalg.inv(synth.mat_mul_cm(proj, view).reshape(4, 4).T.astype(np.float64)).T.astype(np.float32).reshape(16)
    return abi.contact_shadow_camera(inv, view, proj, 0.1)


def algorithmic_bytes(w, h, steps_run):
    """the centre depth read and the output written once per pixel from DRAM; each march step's bilinear tap of 4 texels counted as
    requested bytes (neighbouring rays share lines, mostly served by L1 / L2)"""
    px = w * h
    return dict(dram=px * 4 + px * 4, taps_requested=int(steps_run) * 4 * 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    import torch

    capi.load()
    info = gpu_info()
    runs = []
    for w, h in ((1920, 1080), (3840, 2160)):
        sc = synth.with_ground_caster(synth.make_scene(20000, config_index=2, width=w, height=h, n_unique_meshes=32), half_size=1200.0,
                                      center=(0.0, -2.0, -40.0))
        r = capi.Renderer(0, sc)
        cam = sc.camera(0.0)
        depth = r.render(cam, want_indices=False)["depth"].copy()
        ccam = contact_camera(w, h)
        renderer_out = r.contact_shadows(ccam, abi.contact_shadow_settings(SUN, 8, 0.1, 0.5))
        r.close()
        hw, hh = sc.hiz_extent()
        ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
        px = w * h
        depth_dev, out_dev = ctx.alloc(px * 4), ctx.alloc(px * 4)
        ctx.upload(depth_dev, depth)
        for steps in (8, 16, 64):
            st = abi.contact_shadow_settings(SUN, steps, 0.1, 0.5)
            for _ in range(a.warmup):
                ctx.contact_shadows(ccam, st, depth_dev, w, h, out_dev)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(torch.cuda.current_stream())
            for _ in range(a.launches):
                ctx.contact_shadows(ccam, st, depth_dev, w, h, out_dev)
            e1.record(torch.cuda.current_stream())
            torch.cuda.synchronize()
            us_call = e0.elapsed_time(e1) * 1000.0 / a.launches
            got = ctx.download(out_dev, np.float32, px).reshape(h, w)
            run = dict(width=w, height=h, steps=steps, us_call=round(us_call, 2), depth_pixels=int((depth != 0).sum()),
                       contact_pixels=int((got < 1).sum()), pixels_per_s=round(px / (us_call * 1e-6)))
            if w == 1920 and not a.no_oracle:
                import pyoracle_contact_shadows as co

                lib, counts = co.lib(), np.zeros(3, np.int32)
                want = co.contact_shadows(ccam, st, depth)
                run["oracle_equal"] = bool(np.array_equal(got.view(np.uint32), want.view(np.uint32)))
                # march steps the oracle takes (the hit step ends a ray early), for the requested tap bytes
                steps_run = 0
                sub = np.ascontiguousarray(depth, dtype=np.float32)
                for y in range(0, h, 8):
                    for x in range(0, w, 8):
                        lib.orc_cs_pixel(co.C.byref(ccam), co.C.byref(st), co._p(sub), w, h, x, y, co._p(counts))
                        steps_run += counts[0] if counts[1] < 0 else counts[1] + 1
                run["mean_steps"] = round(steps_run / (((h + 7) // 8) * ((w + 7) // 8)), 2)
                run["bytes"] = algorithmic_bytes(w, h, run["mean_steps"] * px)
                if steps == 8:
                    run["renderer_equal"] = bool(np.array_equal(got.view(np.uint32), renderer_out.view(np.uint32)))
            runs.append(run)
            print(json.dumps(run), file=sys.stderr)
        ctx.free(depth_dev)
        ctx.free(out_dev)
        ctx.close()
    res = dict(gpu=info, launches=a.launches, runs=runs)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
