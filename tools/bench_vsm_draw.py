"""Times the VSM shadow raster (oxc_vsm_draw_pages, the last step of Passes/Shadowmaps.cpp:433-754) on the GPU.

Same frames as tools/bench_vsm.py (reference sizes: 128-px pages, 64 x 64 pages x 10 clipmaps, 4096 physical pages, 8192^2 atlas,
1080p depth of a ground plane): the steady, dirty-instances and sun-moved pairs A / B replayed alternately from CUDA graphs.  Each
graph holds the page update, then the shadow cull of the coarse camera (oxc_cull_meshes + oxc_cull_meshlets_hpb_dirty_dev on the
device flags) and the draw.  The casters are the instances of the synthetic scene plus the ground itself: a tessellated plane at
y = 0 (synth.with_ground_caster, 2400 m square, 1024 meshlets, 65536 triangles) that is also what the camera's depth image sees,
so every dirty page lies on a caster and is filled.
The draw's own time is the difference between graphs with and without it (CUDA events over many replays).  Reported per kind: dirty
pages, (meshlet, clipmap) pairs that reached triangle work, work items, texels of the frame's dirty pages holding a depth below the
clear value, and ns of draw time per such texel.  Prints one JSON line with the card's name and power limit; --out also writes it.  Needs a CUDA
device (no fallback)."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_vsm import LIGHT, clipmaps, ground_depth, gpu_info  # noqa: E402
from oxylus_b200 import abi, capi, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_vsm_draw.py needs a CUDA device")
    W, H = 1920, 1080
    sc = synth.with_ground_caster(synth.make_scene(4000, config_index=2, width=640, height=360, n_unique_meshes=8, seed=3),
                                  half_size=1200.0, center=(0.0, 0.0, -40.0), grid=32)
    hw, hh = sc.hiz_extent()
    stream = torch.cuda.Stream()
    ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh, max_views=10, stream=stream.cuda_stream)
    ctx.set_scene(sc)
    vsm = np.zeros(1, dtype=abi.VSM_CONTEXT_DT)
    vsm["page_size"], vsm["page_table_size"], vsm["physical_page_table_size"], vsm["clipmap_count"] = 128, 64, 8192, 10
    vsm["depth_extent"][0] = (W, H)
    vsm["first_clipmap_width"], vsm["clipmap_selection_bias"], vsm["virtual_extent"], vsm["z_length"] = 10.0, 0.25, 8192.0, 2000.0
    P, E = 4096, 10 * 64 * 64
    res = np.float32([W, H])
    dev = lambda n: torch.zeros(n, dtype=torch.uint8, device="cuda")  # noqa: E731
    buf = dict(pt=dev(E * 4), occ=dev(P * 4), req=dev(E * 12), al=dev(40), fl=dev(P * 4), coords=dev(E * 8), flags=dev(40),
               hpb=dev(sum(10 * max(1, 64 >> l) ** 2 for l in range(7))), atlas=dev(8192 * 8192 * 4))
    ptr = {k: v.data_ptr() for k, v in buf.items()}
    coarse = synth.make_ortho_view(LIGHT, (0.0, 0.0, -40.0), 10.0 * 2 ** 9, 2000.0, sc.mesh_instance_count)
    coarse["position"][0] = -np.asarray(LIGHT) / np.linalg.norm(LIGHT)
    frames = {}
    for name, eye, off in (("A", (0.0, 20.0, 0.0), 0), ("B", (0.0, 20.0, -4.0), 1)):
        inv, depth = ground_depth(W, H, eye)
        frames[name] = dict(inv=inv, depth=torch.from_numpy(depth).cuda(), cm=clipmaps(off))
    dirty = torch.arange(5, dtype=torch.int32, device="cuda")
    prev_np = sc.transforms.copy()
    prev_np["world"][:, 12] += np.float32(2.0)
    prev = torch.from_numpy(prev_np.view(np.uint8).reshape(-1).copy()).cuda()

    def enqueue(fr, kind, draw):
        sun = kind == "sun"
        ctx.vsm_begin_frame(vsm, sun, ptr["pt"], ptr["occ"], P, ptr["al"])
        if kind == "dirty":
            ctx.vsm_invalidate_pages(vsm, fr["cm"], dirty.data_ptr(), 5, prev.data_ptr(), ptr["pt"])
        ctx.mark_visible_pages(fr["inv"], res, fr["cm"], vsm, fr["depth"].data_ptr(), ptr["pt"], ptr["occ"], ptr["al"], ptr["req"], E)
        ctx.vsm_allocate_pages(vsm, ptr["pt"], ptr["occ"], P, ptr["req"], E, ptr["al"], ptr["fl"], ptr["coords"], ptr["flags"])
        ctx.build_hpb(ptr["pt"], 64, 10, ptr["hpb"], 7)
        ctx.vsm_clear_dirty_pages(vsm, ptr["al"], ptr["coords"], ptr["atlas"])
        ctx.cull_meshes(coarse, abi.CULL_TEST_ALL)
        ctx.cull_meshlets_hpb_dirty_dev(coarse, fr["cm"], ptr["flags"], ptr["hpb"], 64, 7)
        if draw:
            ctx.vsm_draw_pages(vsm, coarse, fr["cm"], ptr["flags"], ptr["pt"], ptr["atlas"])

    def graph(fr, kind, draw):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream, capture_error_mode="thread_local"):
            enqueue(fr, kind, draw)
        return g

    def time_pair(ga, gb):
        for _ in range(a.warmup):
            ga.replay(); gb.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record(stream)
            for _ in range(a.replays):
                ga.replay(); gb.replay()
            e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1000.0 / (2 * a.replays)

    enqueue(frames["A"], "sun", True)  # the first draw allocates the context's scratch: outside any capture
    torch.cuda.synchronize()
    result = dict(metric="vsm_shadow_draw_us", sizes="64x64 pages x 10 clipmaps, 4096 physical pages, 8192^2 atlas, 1080p depth, synthetic casters + tessellated ground caster",
                  replays=a.replays, frames={})
    for kind in ("steady", "dirty", "sun"):
        base = time_pair(graph(frames["A"], kind, False), graph(frames["B"], kind, False))
        ga, gb = graph(frames["A"], kind, True), graph(frames["B"], kind, True)
        full = time_pair(ga, gb)
        ga.replay()  # frame A after B: the state a steady replay sees
        torch.cuda.synchronize()
        st = ctx.vsm_draw_stats()
        al = buf["al"][:8].view(torch.int32).cpu().numpy()
        nd = int(al[1])
        coords = buf["coords"][: nd * 8].view(torch.int32).view(-1, 2).long()
        pages = buf["atlas"].view(torch.int32).view(64, 128, 64, 128)[coords[:, 1], :, coords[:, 0], :]  # this frame's dirty pages
        texels = int((pages != 0x3F800000).sum().item())  # written below the clear value
        draw_us = full - base
        result["frames"][kind] = dict(update_and_cull_us=round(base, 2), draw_us=round(draw_us, 2), dirty_pages=nd,
                                      pairs_reaching_triangle_work=st["pairs"], work_items=st["items"], texels_with_depth=texels,
                                      share_of_dirty_texels=round(texels / max(1, nd * 128 * 128), 4),
                                      ns_per_texel=round(draw_us * 1000.0 / texels, 3) if texels else None)
        del ga, gb
    result.update(gpu_info())
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
