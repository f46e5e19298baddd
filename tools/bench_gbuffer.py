"""Times oxc_decode_gbuffer (and oxc_decode_visbuffer next to it) on the benchmark's scene (BASELINE.json configs[1], 1 M meshlet
instances) at 1920 x 1080 and 3840 x 2160, with 64
materials of five seeded RGBA8 1024^2 images each (full mip chains), every material with all five images.  CUDA events over
--launches launches after a warm-up; one JSON line with the card's name and power limit.

    python tools/bench_gbuffer.py [--launches 200] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from oxylus_b200 import abi, capi, synth  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def mip_chain(l0):
    levels = [l0]
    while levels[-1].shape[0] > 1:
        a = levels[-1].astype(np.uint16)
        levels.append(((a[0::2, 0::2] + a[1::2, 0::2] + a[0::2, 1::2] + a[1::2, 1::2] + 2) // 4).astype(np.uint8))
    return levels


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    import pyoracle as orc
    import pyoracle_gbuffer as gb

    capi.load()
    rng = np.random.default_rng(1)
    n_mat, side = 64, 1024
    result = dict(gpu=gpu_info(), launches=a.launches, materials=n_mat, image_side=side, hbm_bytes_per_s=HBM_BYTES_PER_S, runs=[])
    for w, h in ((1920, 1080), (3840, 2160)):
        sc = synth.make_scene(1_000_000, config_index=2, width=w, height=h)
        sc.mesh_instances["material_index"] = rng.integers(0, n_mat, sc.mesh_instance_count)
        hw, hh = sc.hiz_extent()
        ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
        ctx.set_scene(sc)
        images, host_images, ptrs, texel_bytes = [], [], [], 0
        for i in range(n_mat * 5):
            lv = mip_chain(rng.integers(0, 256, (side, side, 4), dtype=np.uint8))
            t = np.concatenate([l.reshape(-1) for l in lv])
            d = ctx.alloc(t.size)
            ctx.upload(d, t)
            ptrs.append(d)
            texel_bytes += t.size
            fmt = abi.IMAGE_RGBA8_SRGB if i % 5 in (0, 2) else abi.IMAGE_RGBA8_UNORM
            images.append((d, side, side, fmt, len(lv)))
            host_images.append((lv, fmt))
        m = np.zeros(n_mat, dtype=abi.MATERIAL_DT)
        for i in range(n_mat):
            m[i]["flags"] = 31
            m[i]["albedo_color"] = [15360] * 4
            m[i]["emissive_color"] = [15360] * 3
            m[i]["metallic_factor"] = m[i]["roughness_factor"] = 15360
            m[i]["uv_size"] = [15360, 15360]
            m[i]["albedo_image_index"], m[i]["normal_image_index"], m[i]["emissive_image_index"] = 5 * i, 5 * i + 1, 5 * i + 2
            m[i]["metallic_roughness_image_index"], m[i]["occlusion_image_index"] = 5 * i + 3, 5 * i + 4
        ctx.set_materials(m, images)
        cam = sc.camera(0.0)
        vis_dev = ctx.alloc(w * h * 8)
        from test_gpu_parity import _frame_gpu

        _frame_gpu(capi, ctx, sc, cam, None, vis_dev)
        planes = {k: ctx.alloc(w * h * 16) for k in abi.GBUFFER_PLANES}
        un = ctx.alloc(w * h * 16)
        ctx.sync()

        def timed(fn):
            for _ in range(10):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.launches):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) * 1e3 / a.launches

        us_g = timed(lambda: ctx.decode_gbuffer(cam, w, h, planes, vis64_dev=vis_dev))
        us_d = timed(lambda: ctx.decode_visbuffer(cam, w, h, {"uv_normal": un}, vis64_dev=vis_dev))
        v32 = (ctx.download(vis_dev, np.uint64, w * h) & np.uint64(0xFFFFFFFF)).astype(np.uint32).reshape(h, w)
        decoded = int((v32 != 0xFFFFFFFF).sum())
        written = w * h * 16 * 4
        # texel bytes the decode requests: the oracle's fetch count over the same frame and table (one 4-byte word per fetch on the
        # device), and the distinct 32-byte sectors would be fewer; bytes that reached DRAM are not measured (no profiler here)
        hs = orc.HostScene(sc)
        mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
        gb.texel_fetches(reset=True)
        gb.decode_gbuffer(hs, mi, int(vis["total"][0]), cam, v32, orc.MaterialTable(m, host_images))
        texel_bytes_requested = 4 * gb.texel_fetches(reset=True)
        result["runs"].append(dict(width=w, height=h, us_decode_gbuffer=round(us_g, 2), pixels_per_s=round(w * h / (us_g * 1e-6), 1),
                                   decoded_pixels=decoded, bytes_written=written, texel_bytes_resident=texel_bytes,
                                   texel_bytes_requested=texel_bytes_requested,
                                   requested_share_of_hbm_peak=round((written + texel_bytes_requested) / (us_g * 1e-6) / HBM_BYTES_PER_S, 4),
                                   write_share_of_hbm_peak=round(written / (us_g * 1e-6) / HBM_BYTES_PER_S, 4),
                                   us_decode_visbuffer_uv_normal=round(us_d, 2)))
        for p in ptrs + list(planes.values()) + [vis_dev, un]:
            ctx.free(p)
        ctx.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
