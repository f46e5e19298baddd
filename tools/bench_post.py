"""Eye adaptation and bloom timing on the H100: oxc_eye_adaptation and oxc_bloom on a lit frame made on the device from the benchmark's
synthetic scene (20,000 instances over a ground plane, as tools/bench_pbr.py: the renderer's depth, decoded normals and GTAO, seeded
material planes, oxc_apply_pbr with HasDirectionalLight | HasGTAO and 16 lights) and on a uniform frame (every pixel in one bin, the
histogram's adversarial case), at 1080p and 4K.  CUDA-event times per call over --launches calls after --warmup.  Bloom runs in two
forms, alternated in the same call: the library's (per-level launches for the large levels, one single-CTA kernel for every level from
the first one of at most 1024 texels down and back up) and every level as its own launch (tools/ubench/bloom_per_level.cu, compiled
here into a temporary directory with the library's flags).  The histogram, the record and both chains of both forms are checked against
the oracle (oracle/pyoracle_post.py) in the same call.  Bytes moved are the algorithmic lower bound (each pass reads its source level
once and writes its destination once) over the 3.35 TB/s data-sheet bandwidth.  Reads the card name and power limit in the same run.
Prints one JSON line and writes it to --out.

    python tools/bench_post.py --launches 200 --out profiles/h100_post/bench_post.json
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from oxylus_b200 import abi, build, capi, synth  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn, launches, warmup):
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(torch.cuda.current_stream())
    for _ in range(launches):
        fn()
    e1.record(torch.cuda.current_stream())
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / launches


def per_level_lib(tmp):
    so = os.path.join(tmp, "libbloom_per_level.so")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-ldl",)]
    res = subprocess.run([build.nvcc_path()] + flags + ["-o", so, os.path.join(ROOT, "tools", "ubench", "bloom_per_level.cu")],
                         capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed on bloom_per_level.cu:\n" + res.stderr)
    lib = C.CDLL(so)
    vp = C.c_void_p
    lib.bloom_per_level.argtypes = [vp, C.c_uint32, C.c_uint32, C.POINTER(abi.BloomSettings), vp, C.POINTER(abi.BloomTargets), vp]
    lib.bloom_per_level.restype = C.c_int
    return lib


def lit_frame(w, h):
    """the benchmark scene's lit frame, made on the device; returns (context, device pointer)"""
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
                  emissive=(rng.random((h, w, 4), dtype=np.float32) * 20.0 * (rng.random((h, w, 1)) < 0.02)).astype(np.float32),
                  metallic_roughness_occlusion=rng.random((h, w, 4), dtype=np.float32), ambient_occlusion=ao,
                  shadow=np.where(rng.random((h, w)) < 0.4, 0.0, 1.0).astype(np.float32))
    inputs = {}
    for k, v in planes.items():
        inputs[k] = ctx.alloc(v.nbytes)
        ctx.upload(inputs[k], v)
    lights = synth.make_lights(np.random.default_rng(7), 16)
    lights_dev = ctx.alloc(64 * 16)
    ctx.upload(lights_dev, np.frombuffer(bytes(lights), np.uint8))
    frame = ctx.alloc(px * 16)
    ctx.apply_pbr(synth.pbr_camera(cam), abi.pbr_settings(scene_flags=abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_GTAO, light_count=16),
                  lights_dev, inputs, w, h, frame)
    ctx.sync()
    for p in list(inputs.values()) + [un_dev, v32_dev, lights_dev]:
        ctx.free(p)
    return ctx, frame


def bloom_bytes(w, h):
    """each pass reads its source once and writes its destination once (16 B per texel); the upsample also reads the downsampled level"""
    lv = abi.bloom_levels(w, h)
    t = [lw * lh for lw, lh, _ in lv]
    b = w * h * 16 + t[0] * 16
    b += sum((t[i - 1] + t[i]) * 16 for i in range(1, len(t)))
    b += sum((t[i] + 2 * t[i - 1]) * 16 for i in range(1, len(t)))
    return b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    capi.load()
    res = dict(gpu=gpu_info(), launches=a.launches, hbm_bytes_per_s=HBM_BYTES_PER_S, runs=[])
    es = abi.eye_adaptation_settings()
    bs = abi.bloom_settings(scene_flags=abi.SCENE_HAS_EYE_ADAPTATION)
    with tempfile.TemporaryDirectory() as tmp:
        per_level = per_level_lib(tmp)
        for w, h in ((1920, 1080), (3840, 2160)):
            ctx, lit = lit_frame(w, h)
            px, n = w * h, abi.bloom_chain_texels(w, h)
            uni = ctx.alloc(px * 16)
            ctx.upload(uni, np.broadcast_to(np.float32([2.0, 2.0, 2.0, 1.0]), (h, w, 4)).copy())
            rec, hist, down, up = ctx.alloc(8), ctx.alloc(1024), ctx.alloc(n * 16), ctx.alloc(n * 16)
            targets = abi.BloomTargets(int(down), int(up))
            one = np.frombuffer(bytes(abi.Exposure(1.0, 1.0)), np.uint8)
            for label, frame in (("lit", lit), ("uniform", uni)):
                run = dict(extent=[w, h], frame=label, levels=len(abi.bloom_levels(w, h)), eye_bytes=px * 16 + 1024,
                           bloom_bytes=bloom_bytes(w, h))
                ctx.upload(rec, one)

                def eye():
                    ctx.eye_adaptation(frame, w, h, es, 0.016, rec, hist)

                def fused():
                    ctx.bloom(frame, w, h, bs, rec, down, up)

                def levels():
                    rc = per_level.bloom_per_level(C.c_void_p(frame), w, h, C.byref(bs), C.c_void_p(rec), C.byref(targets), None)
                    assert rc == 0, rc

                run["us_eye_adaptation"] = round(timed(eye, a.launches, a.warmup), 2)
                for k in range(2):
                    for name, fn in (("bloom_fused_tail", fused), ("bloom_per_level", levels)):
                        run[f"us_{name}_{k}"] = round(timed(fn, a.launches, a.warmup), 2)
                run["eye_bound_share"] = round(run["eye_bytes"] / HBM_BYTES_PER_S * 1e6 / run["us_eye_adaptation"], 3)
                best = min(run["us_bloom_fused_tail_0"], run["us_bloom_fused_tail_1"])
                run["bloom_fused_bound_share"] = round(run["bloom_bytes"] / HBM_BYTES_PER_S * 1e6 / best, 3)
                if not a.no_oracle:
                    import pyoracle_post as so

                    host = ctx.download(frame, np.float32, px * 4).reshape(h, w, 4)
                    ctx.upload(rec, one)
                    eye()
                    want_rec, want_hist = so.eye_adaptation(host, es, 0.016, abi.Exposure(1.0, 1.0))
                    got_rec = ctx.download(rec, np.uint32, 2)
                    run["oracle_equal_eye"] = bool(np.array_equal(ctx.download(hist, np.uint32, 256), want_hist) and
                                                   np.array_equal(got_rec, np.frombuffer(bytes(want_rec), np.uint32)))
                    want = so.bloom(host, bs, want_rec)
                    for name, fn in (("fused_tail", fused), ("per_level", levels)):
                        ctx.upload(down, np.zeros(n * 4, np.float32))
                        ctx.upload(up, np.zeros(n * 4, np.float32))
                        fn()
                        got = ctx.download(down, np.float32, n * 4).reshape(n, 4), ctx.download(up, np.float32, n * 4).reshape(n, 4)
                        run[f"oracle_equal_bloom_{name}"] = bool(all(np.array_equal(g.view(np.uint32), wv.view(np.uint32))
                                                                     for g, wv in zip(got, want)))
                res["runs"].append(run)
                print(json.dumps(run), file=sys.stderr)
            for p in (lit, uni, rec, hist, down, up):
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
