"""Times the VSM page bookkeeping (oxc_vsm_*, Passes/Shadowmaps.cpp:100-430 up to the shadow raster) on the GPU.

Reference sizes (RendererInstance.hpp:262-267): 128-px pages, 64 x 64 pages x 10 clipmaps, 4096 physical pages, 8192^2 R32F atlas.
The depth is a 1920 x 1080 reverse-Z image of a ground plane seen from 20 m up.  Each kind of frame is a pair of frames A / B
replayed alternately from CUDA graphs, so every replay starts from the state the other one left:
  steady   B's camera is 4 m further along and the finest clipmap's page offset has scrolled by one page: a few pages change
  dirty    as steady, plus 5 dirty mesh instances whose previous and current boxes are invalidated (and reallocated) every frame
  sun      sun_moved on every frame: the table is cleared, every visible page is reallocated and its 64 KiB cleared
Per-stage times are differences of graphs holding the first k stages, timed with CUDA events over many replays; the clear kernel
is also timed alone on the sun frame's dirty list, and its bytes / time is compared with the H100 SXM data-sheet 3.35 TB/s.
Prints one JSON line; --out also writes it to a file.  Needs a CUDA device (no fallback)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oxylus_b200 import abi, capi, synth  # noqa: E402

STAGES = ("begin_frame", "invalidate", "mark_visible", "allocate", "build_hpb", "clear_dirty")
LIGHT = (0.3, -1.0, 0.2)


def ground_depth(w, h, eye):
    """camera at `eye` looking down the -z axis and 25 degrees down; depth of the plane y = 0 (0 = sky)"""
    pv = synth.mat_mul_cm(synth.perspective_reverse_z(60.0, w / h, 0.1, 1000.0),
                          synth.look_at(eye, (eye[0], 0.0, eye[2] - 43.0), (0.0, 1.0, 0.0)))
    m = pv.reshape(4, 4).T.astype(np.float64)
    inv = np.linalg.inv(m)
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    u, v = (xs + 0.5) / w, (ys + 0.5) / h

    def unproj(z):
        ndc = np.stack([u * 2 - 1, v * 2 - 1, np.full_like(u, z), np.ones_like(u)], axis=-1)
        p = ndc @ inv.T
        return p[..., :3] / p[..., 3:4]

    p0, p1 = unproj(1.0), unproj(1e-4)
    t = p0[..., 1] / (p0[..., 1] - p1[..., 1])
    world = p0 + t[..., None] * (p1 - p0)
    clip = np.concatenate([world, np.ones_like(world[..., :1])], axis=-1) @ m.T
    depth = np.where((t > 0) & (t < 1), clip[..., 2] / clip[..., 3], 0.0).astype(np.float32)
    depth[(depth <= 0) | ~np.isfinite(depth)] = 0.0
    return inv.T.astype(np.float32).reshape(16), depth


def clipmaps(offset0):
    cm = np.zeros(10, dtype=abi.CLIPMAP_DT)
    for k in range(10):
        v = synth.make_ortho_view(LIGHT, (0.0, 0.0, -40.0), 10.0 * (2 ** k), 2000.0, 1)
        cm["projection_view_mat"][k] = v["projection_view"][0]
        cm["page_offset"][k] = (offset0 + 3 * k, -2 * k) if k == 0 else (3 * k, -2 * k)
    return cm


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # the card's name still comes from the runtime
        import torch

        return dict(gpu=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})", max_sm_clock="unknown")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_vsm.py needs a CUDA device")
    W, H = 1920, 1080
    sc = synth.make_scene(4000, config_index=2, width=640, height=360, n_unique_meshes=8, seed=3)
    hw, hh = sc.hiz_extent()
    stream = torch.cuda.Stream()
    ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh, stream=stream.cuda_stream)
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
    frames = {}
    for name, eye, off in (("A", (0.0, 20.0, 0.0), 0), ("B", (0.0, 20.0, -4.0), 1)):
        inv, depth = ground_depth(W, H, eye)
        frames[name] = dict(inv=inv, depth=torch.from_numpy(depth).cuda(), cm=clipmaps(off))
    dirty = torch.arange(5, dtype=torch.int32, device="cuda")
    prev = torch.from_numpy(sc.transforms.view(np.uint8).copy()).cuda()
    prev_np = sc.transforms.copy()
    prev_np["world"][:, 12] += np.float32(2.0)  # every instance moved 2 m in x since the previous frame
    prev.copy_(torch.from_numpy(prev_np.view(np.uint8).reshape(-1)))

    def enqueue(fr, kind, n_stages):
        sun = kind == "sun"
        calls = [
            lambda: ctx.vsm_begin_frame(vsm, sun, ptr["pt"], ptr["occ"], P, ptr["al"]),
            lambda: ctx.vsm_invalidate_pages(vsm, fr["cm"], dirty.data_ptr(), 5, prev.data_ptr(), ptr["pt"]) if kind == "dirty" else None,
            lambda: ctx.mark_visible_pages(fr["inv"], res, fr["cm"], vsm, fr["depth"].data_ptr(), ptr["pt"], ptr["occ"], ptr["al"], ptr["req"], E),
            lambda: ctx.vsm_allocate_pages(vsm, ptr["pt"], ptr["occ"], P, ptr["req"], E, ptr["al"], ptr["fl"], ptr["coords"], ptr["flags"]),
            lambda: ctx.build_hpb(ptr["pt"], 64, 10, ptr["hpb"], 7),
            lambda: ctx.vsm_clear_dirty_pages(vsm, ptr["al"], ptr["coords"], ptr["atlas"]),
        ]
        for c in calls[:n_stages]:
            c()

    def graph(fr, kind, n):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream, capture_error_mode="thread_local"):
            enqueue(fr, kind, n)
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

    def counters():
        torch.cuda.synchronize()
        c = buf["al"][:16].view(torch.int32).cpu().numpy()
        return dict(requests=int(c[0]), dirty_pages=int(c[1]), free_pages=int(c[2]))

    result = dict(metric="vsm_page_bookkeeping_us", sizes="64x64 pages x 10 clipmaps, 4096 physical pages, 8192^2 atlas, 1080p depth",
                  replays=a.replays, frames={})
    for kind in ("steady", "dirty", "sun"):
        cum = []
        for n in range(1, len(STAGES) + 1):
            ga, gb = graph(frames["A"], kind, n), graph(frames["B"], kind, n)
            cum.append(time_pair(ga, gb))
            del ga, gb
        ga, gb = graph(frames["A"], kind, len(STAGES)), graph(frames["B"], kind, len(STAGES))
        ga.replay(); gb.replay()
        seen = counters()
        stages = {s: round(cum[i] - (cum[i - 1] if i else 0.0), 2) for i, s in enumerate(STAGES)}
        result["frames"][kind] = dict(total_us=round(cum[-1], 2), stages_us=stages, **seen)
        if kind == "sun":
            gc = torch.cuda.CUDAGraph()  # the clear alone, on the sun frame's dirty list
            with torch.cuda.graph(gc, stream=stream, capture_error_mode="thread_local"):
                ctx.vsm_clear_dirty_pages(vsm, ptr["al"], ptr["coords"], ptr["atlas"])
            t = time_pair(gc, gc)
            nbytes = seen["dirty_pages"] * 128 * 128 * 4
            result["clear"] = dict(dirty_pages=seen["dirty_pages"], bytes=nbytes, us=round(t, 2), tb_per_s=round(nbytes / (t * 1e-6) / 1e12, 3),
                                   share_of_3_35_tb_per_s=round(nbytes / (t * 1e-6) / 3.35e12, 3))
    result.update(gpu_info())
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
