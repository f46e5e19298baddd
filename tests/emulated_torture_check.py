#!/usr/bin/env python
"""Hostile-but-representable inputs through the whole two-pass frame: MeshletBounds fields set to NaN, +-Inf, negative extents,
+-0, the largest half, denormal-flushed values, garbage cone bytes; vertex positions with the same special values; transforms scaled by 1e-12 / 1e6, mirrored, with a zero
column, at the camera, far away.  No mesh builder produces such records, but the reference's shaders — and therefore the oracle —
are defined for them, and "bit-identical to the canonical evaluation for every input" has to hold for them too (this is the
scenario that found the cone filter turning a NaN radius into 0 and the frustum filter assuming h >= 0).
Runs against whichever library capi loads: tests/test_emulated_library_cpu.py runs main() on the SIMT-emulated library, and
tests/test_gpu_variants.py::test_hostile_frames runs every case of cases() on the GPU, where rcp.approx.ftz / rsqrt.approx.ftz
give the hardware's flush-to-zero results that the emulator's IEEE stand-ins do not.  (tests/conftest.py imports mutate() under
this module's name.)

    python tests/emulated_torture_check.py [seeds]"""
import copy
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import pyoracle as orc  # noqa: E402
from oxylus_b200 import abi, capi, synth  # noqa: E402

SPECIALS = np.array([0x0000, 0x8000, 0x0001, 0x03FF, 0x0400, 0x7BFF, 0xFBFF, 0x7C00, 0xFC00, 0x7E00, 0x3C00, 0xBC00], dtype=np.uint16)


def mutate(base, rng, mode):
    sc = copy.deepcopy(base)
    for m in sc.meshes:
        lods = np.frombuffer(sc.blob, dtype=abi.MESH_LOD_DT, count=int(m["lod_count"]), offset=int(m["lods"]))
        for d in lods:
            n = int(d["meshlet_bounds_count"])
            b = np.ndarray((n, 8), dtype=np.uint16, buffer=sc.blob.data, offset=int(d["meshlet_bounds"]))  # c.xyz | cone xy | e.xyz | cone z, cutoff
            hit = rng.random(n) < 0.15
            if mode in ("bounds", "all"):
                for c in (0, 1, 2, 4, 5, 6):
                    sel = hit & (rng.random(n) < 0.5)
                    b[sel, c] = SPECIALS[rng.integers(0, len(SPECIALS), int(sel.sum()))]
            if mode in ("cones", "all"):
                sel = rng.random(n) < 0.3
                b[sel, 3] = rng.integers(0, 65536, int(sel.sum())).astype(np.uint16)
                b[sel, 7] = rng.integers(0, 65536, int(sel.sum())).astype(np.uint16)
    if mode in ("vertices", "all"):  # vertex positions: u16 x 4 per vertex (scene.slang:478-484)
        for m in sc.meshes:
            n = int(m["vertex_count"])
            v = np.ndarray((n, 4), dtype=np.uint16, buffer=sc.blob.data, offset=int(m["vertex_positions"]))
            for c in range(3):
                sel = rng.random(n) < 0.02
                v[sel, c] = SPECIALS[rng.integers(0, len(SPECIALS), int(sel.sum()))]
    if mode in ("transforms", "all"):
        t = sc.transforms["world"]
        for i in np.nonzero(rng.random(len(t)) < 0.2)[0]:
            kind = int(rng.integers(0, 6))
            if kind == 0:
                t[i, :12] *= np.float32(1e-12)
            elif kind == 1:
                t[i, :12] *= np.float32(1e6)
            elif kind == 2:
                t[i, 0:3] *= np.float32(-1)
            elif kind == 3:
                t[i, 0:3] = 0
            elif kind == 4:
                t[i, 12:15] = (0, 0, 0)
            else:
                t[i, 12:15] *= np.float32(1e4)
    if mode in ("texcoords", "all"):  # u16 x 2 halves per vertex (scene.slang:491-497): NaN / Inf / huge / denormal uv reach the alpha
        for m in sc.meshes:           # test's interpolation, texel addressing and wrap modes (drawn last: earlier draws unchanged)
            if int(m["texture_coords"]) == 0:
                continue
            n = int(m["vertex_count"])
            v = np.ndarray((n, 2), dtype=np.uint16, buffer=sc.blob.data, offset=int(m["texture_coords"]))
            for c in range(2):
                sel = rng.random(n) < 0.03
                v[sel, c] = SPECIALS[rng.integers(0, len(SPECIALS), int(sel.sum()))]
    return sc


def hostile_cameras(sc):
    """cameras a host could hand over by mistake: degenerate near planes, a far-away eye, badly scaled or NaN matrix entries,
    LOD thresholds of 0 / Inf"""
    out = []
    for k in range(10):
        cam = sc.camera(5.0 * k).copy()
        if k == 1: cam["near_clip"] = 1e-30
        if k == 2: cam["near_clip"] = 50.0
        if k == 3: cam["position"][0] = [1e6, 0, 0]
        if k == 4: cam["projection_view"][0] *= np.float32(1e-6)
        if k == 5: cam["projection_view"][0] *= np.float32(1e6)
        if k == 6: cam["acceptable_lod_error"] = 0.0
        if k == 7: cam["acceptable_lod_error"] = np.inf
        if k == 8: cam["projection_view"][0][5] = np.nan
        if k == 9: cam["near_clip"] = np.nan
        out.append(cam)
    return out


def alpha_table():
    """four materials over mip-mapped / single-level images with every filter, mipmap and address mode between them (oracle table)"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_oracle_alpha import checker, material

    rng = np.random.default_rng(77)
    images = [(orc.mip_chain(checker(32, 4)), abi.IMAGE_RGBA8_UNORM), (orc.mip_chain(rng.integers(0, 256, (16, 8), dtype=np.uint8)), abi.IMAGE_R8_UNORM),
              (rng.integers(0, 256, (4, 4), dtype=np.uint8), abi.IMAGE_R8_UNORM)]
    mats = np.array([material(), material(image=0, cutoff=0.5), material(image=1, cutoff=0.4, albedo_a=0.9, sampler=1), material(image=2, cutoff=0.5, sampler=2)],
                    dtype=abi.MATERIAL_DT)
    smp = np.array([abi.sampler(), abi.sampler(mip=abi.MIPMAP_NEAREST, u=abi.ADDRESS_MIRRORED_REPEAT, v=abi.ADDRESS_CLAMP_TO_EDGE),
                    abi.sampler(mag=abi.FILTER_NEAREST, min=abi.FILTER_LINEAR)], dtype=abi.SAMPLER_DT)
    return orc.MaterialTable(mats, images, smp), mats, smp


def frames_equal(sc, frames=2, cams=None, occluder_depth=None, alpha=False):
    if alpha:  # every fourth mesh instance opaque, the others alpha tested (visbuffer_encode.slang:54-66)
        sc = copy.deepcopy(sc)
        sc.mesh_instances["material_index"] = np.arange(sc.mesh_instance_count) % 4
    hs = orc.HostScene(sc)
    w, h = sc.width, sc.height
    hw, hh = sc.hiz_extent()
    ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
    ctx.set_scene(sc)
    tab = None
    if alpha:
        tab, mats, smp = alpha_table()
        dev, _ = tab.device_images(ctx)
        ctx.set_materials(mats, dev, smp)
    vis, occ = ctx.alloc(w * h * 8), ctx.alloc(w * h * 4)
    depth = sc.occluder_depth if occluder_depth is None else occluder_depth
    ctx.upload(occ, depth)
    mask = np.zeros((sc.max_meshlet_instance_count + 31) // 32, dtype=np.uint32)
    ok = True
    for cam in (cams if cams is not None else [sc.camera(3.0 * f) for f in range(frames)]):
        ref = orc.frame(hs, cam, w, h, mask, depth, materials=tab)
        ctx.clear_visbuffer_with_depth(vis, occ, w, h)
        ctx.clear_hiz()
        ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
        ctx.cull_meshlets(cam, abi.CULL_TEST_ALL, True)
        ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, w, h, vis)
        ctx.build_hiz_packed(vis, w, h)
        ctx.cull_meshlets(cam, abi.CULL_TEST_ALL | abi.CULL_LATE_PASS, True)
        ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL | abi.CULL_LATE_PASS, w, h, vis)
        v = ctx.visibility()
        e, l = int(v["early"][0]), int(v["late"][0])
        same = (e, l) == (ref["early"], ref["late"])
        same = same and np.array_equal(np.sort(ctx.visible_indices(e + l)), np.sort(ref["visible"][: ref["early"] + ref["late"]]))
        same = same and np.array_equal(ctx.download(vis, np.uint64, w * h).reshape(h, w), ref["vis64"]) and np.array_equal(ctx.mask(), mask)
        same = same and np.array_equal(np.concatenate([x.ravel() for x in ctx.hiz_levels()]).view(np.uint32), ref["hiz"].data.view(np.uint32))
        ok = ok and bool(same)
    ctx.close()
    return ok


def base_scene():
    return synth.make_scene(8000, config_index=2, width=320, height=180, n_unique_meshes=24, max_lods=2, ragged=True)


def hostile_depth(base):
    """the scene's occluder depth with 1 % of its pixels NaN, +-Inf, out of [0, 1], denormal or -0"""
    depth = base.occluder_depth.copy()
    rng = np.random.default_rng(3)
    sel = rng.random(depth.shape) < 0.01
    depth[sel] = rng.choice(np.array([np.nan, np.inf, -np.inf, -1.0, 2.0, 1e-45, -0.0], dtype=np.float32), int(sel.sum()))
    return depth


def cases(seeds=2):
    """(label, mutation mode or None, seed, hostile cameras, material table, hostile external depth) of every check main() runs.
    With a material table the same hostility reaches the alpha test's interpolation, level selection and texel addressing."""
    out = [(f"{mode} seed {seed}", mode, seed, False, False, False) for seed in range(seeds)
           for mode in ("bounds", "cones", "vertices", "transforms", "all")]
    out.append(("cameras", None, 0, True, False, False))
    out += [(f"all + alpha seed {seed}", "all", seed, False, True, False) for seed in range(seeds)]
    out += [("cameras + alpha", None, 0, True, True, False), ("external depth", None, 0, False, False, True)]
    return out


def run_case(base, case):
    _, mode, seed, cams, alpha, depth = case
    sc = base if mode is None else mutate(base, np.random.default_rng(seed * 10 + 1), mode)
    return frames_equal(sc, cams=hostile_cameras(base) if cams else None, occluder_depth=hostile_depth(base) if depth else None, alpha=alpha)


def main():
    seeds = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    base = base_scene()
    bad = [case[0] for case in cases(seeds) if not run_case(base, case)]
    print(f"{seeds * 5} hostile scenes x 2 frames, 10 hostile cameras, {seeds} hostile scenes + 10 hostile cameras with a material table, hostile external depth: "
          f"{'ok' if not bad else 'MISMATCH ' + repr(bad)}")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
