"""ctypes wrapper of the CPU oracle (oracle/liboxc_oracle.so).  TEST INFRASTRUCTURE ONLY.

Importers allowed by the project rules: tests/, __graft_entry__.smoke(), bench.py's cpu_baseline and
--impl reference legs.  The product package (oxylus_b200/) never imports this module.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(_HERE))
from oxylus_b200 import abi  # noqa: E402  (ABI struct definitions only)

_LIB = None


CFLAGS = ["-O2", "-std=c11", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-function", "-pthread"]


def build_so(name, units, deps, force=False):
    """compiles the C files `units` into oracle/<name> when it is missing or older than one of `deps` (every oracle file it is made
    from) or include/oxcull.h.  The library is written under a per-process name and renamed into place, so concurrent test
    processes never load a half-written one."""
    so = os.path.join(_HERE, name)
    srcs = [os.path.join(_HERE, f) for f in deps] + [os.path.join(os.path.dirname(_HERE), "include", "oxcull.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        tmp = so + f".{os.getpid()}.tmp"
        subprocess.check_call([os.environ.get("CC", "gcc")] + CFLAGS + ["-shared", "-o", tmp] + [os.path.join(_HERE, u) for u in units] +
                              ["-lm", "-lpthread"])
        os.replace(tmp, so)
    return so


def build(force=False):
    return build_so("liboxc_oracle.so", ["oxc_oracle.c"], ["oxc_oracle.c", "oxc_oracle.h", "oxc_oracle_math.inc"], force)


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liboxc_oracle.so")
        if not os.path.exists(so):
            build()
        _LIB = C.CDLL(so)
        _LIB.orc_dequantize_half.restype = C.c_float
        _LIB.orc_dequantize_half.argtypes = [C.c_uint16]
        _LIB.orc_ceil_log2_u32.restype = C.c_uint32
        _LIB.orc_ceil_log2_u32.argtypes = [C.c_uint32]
        _LIB.orc_hiz_total_texels.restype = C.c_uint32
        _LIB.orc_hiz_level_count.restype = C.c_uint32
        _LIB.orc_cpu_baseline_cull.restype = C.c_uint64
        _LIB.orc_cpu_frame.restype = C.c_uint64
    return _LIB


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None else C.c_void_p(0)


class HostScene:
    """Host copies of a synth.Scene (mesh_instances is mutable: cull_meshes writes lod_index)."""

    def __init__(self, scene):
        self.meshes = np.ascontiguousarray(scene.meshes)
        self.mesh_instances = np.ascontiguousarray(scene.mesh_instances).copy()
        self.transforms = np.ascontiguousarray(scene.transforms)
        self.blob = np.ascontiguousarray(scene.blob)
        self.desc = abi.SceneDesc()
        self.desc.meshes = self.meshes.ctypes.data
        self.desc.mesh_count = len(self.meshes)
        self.desc.mesh_instances = self.mesh_instances.ctypes.data
        self.desc.mesh_instance_count = len(self.mesh_instances)
        self.desc.transforms = self.transforms.ctypes.data
        self.desc.transform_count = len(self.transforms)
        self.desc.blob = self.blob.ctypes.data
        self.desc.blob_size = self.blob.size
        self.max_meshlets = scene.max_meshlet_instance_count

    @property
    def ref(self):
        return C.byref(self.desc)


class Hiz:
    def __init__(self, w, h):
        self.w, self.h = w, h
        self.levels, self.offsets, self.total = abi.hiz_layout(w, h)
        self.data = np.zeros(self.total, dtype=np.float32)
        self.c = abi.OrcHiz()
        lib().orc_hiz_layout(C.c_uint32(w), C.c_uint32(h), C.byref(self.c))
        assert self.c.levels == self.levels and list(self.c.level_offset)[: self.levels] == self.offsets
        self.c.data = self.data.ctypes.data

    def level(self, l):
        mw, mh = max(1, self.w >> l), max(1, self.h >> l)
        return self.data[self.offsets[l] : self.offsets[l] + mw * mh].reshape(mh, mw)

    @property
    def ref(self):
        return C.byref(self.c)


def dequantize_half(h):
    return float(lib().orc_dequantize_half(C.c_uint16(int(h))))


def cull_meshes(hs: HostScene, cam, flags, first=0, count=0xFFFFFFFF):
    mi = np.zeros(max(1, hs.max_meshlets), dtype=abi.MESHLET_INSTANCE_DT)
    vis = np.zeros(1, dtype=abi.VISIBILITY_DT)
    cmd = np.zeros(1, dtype=abi.DISPATCH_CMD_DT)
    lib().orc_cull_meshes(hs.ref, _p(cam), C.c_uint32(flags), C.c_uint32(first), C.c_uint32(count), _p(mi), _p(vis), _p(cmd))
    return mi, vis, cmd


def cull_meshlets_hiz(hs, mi, vis, cam, flags, hiz: Hiz, mask, visible=None):
    if visible is None:
        visible = np.zeros(max(1, hs.max_meshlets), dtype=np.uint32)
    cmd = np.zeros(1, dtype=abi.DISPATCH_CMD_DT)
    lib().orc_cull_meshlets_hiz(hs.ref, _p(mi), _p(cam), C.c_uint32(flags), hiz.ref, _p(vis), _p(visible), _p(mask), _p(cmd))
    return visible, cmd


def cull_meshlets_flags(hs, mi, vis, cam, flags, hiz: Hiz, mask, f64=False):
    out = np.zeros(max(1, int(vis["total"][0])), dtype=np.uint8)
    fn = lib().orc_cull_meshlets_hiz_f64 if f64 else lib().orc_cull_meshlets_hiz_f32_flags
    fn(hs.ref, _p(mi), _p(cam), C.c_uint32(flags), hiz.ref, _p(vis), _p(mask), _p(out))
    return out[: int(vis["total"][0])]


def cull_meshlets(hs, mi, vis, cam):
    visible = np.zeros(max(1, hs.max_meshlets), dtype=np.uint32)
    cmd = np.zeros(1, dtype=abi.DISPATCH_CMD_DT)
    lib().orc_cull_meshlets(hs.ref, _p(mi), _p(cam), _p(vis), _p(visible), _p(cmd))
    return visible, cmd


def cull_meshlets_multiview(hs, mi, total, views, directional):
    bits = np.zeros(max(1, total), dtype=np.uint32)
    counts = np.zeros(abi.MAX_VIEWS, dtype=np.uint32)
    lib().orc_cull_meshlets_multiview(hs.ref, _p(mi), C.c_uint32(total), _p(views), C.c_uint32(len(views)),
                                      C.c_int(int(directional)), _p(bits), _p(counts))
    return bits[:total], counts


def build_hiz(depth, hiz: Hiz):
    depth = np.ascontiguousarray(depth, dtype=np.float32)
    h, w = depth.shape
    lib().orc_build_hiz(_p(depth), C.c_uint32(w), C.c_uint32(h), hiz.ref)
    return hiz


def cull_triangles(hs, mi, visible, first, count, cam, id_base=0):
    out = np.zeros(max(1, count) * 64 * 3, dtype=np.uint32)
    cmd = np.zeros(1, dtype=abi.DRAW_CMD_DT)
    lib().orc_cull_triangles(hs.ref, _p(mi), _p(visible), C.c_uint32(first), C.c_uint32(count), _p(cam),
                             C.c_uint32(id_base), _p(out), _p(cmd))
    return out[: int(cmd["index_count"][0])], cmd


def cull_triangles_small_primitive(hs, mi, visible, first, count, cam, w, h, id_base=0):
    """(index buffer, draw cmd, number of triangles the opt-in small-primitive cull removed)"""
    out = np.zeros(max(1, count) * 64 * 3, dtype=np.uint32)
    cmd = np.zeros(1, dtype=abi.DRAW_CMD_DT)
    fn = lib().orc_cull_triangles_small_primitive
    fn.restype = C.c_uint64
    culled = fn(hs.ref, _p(mi), _p(visible), C.c_uint32(first), C.c_uint32(count), _p(cam), C.c_uint32(id_base), C.c_uint32(w), C.c_uint32(h),
                _p(out), _p(cmd))
    return out[: int(cmd["index_count"][0])], cmd, int(culled)


def clear_visbuffer(w, h):
    vis = np.zeros((h, w), dtype=np.uint64)
    lib().orc_clear_visbuffer(_p(vis), C.c_uint32(w), C.c_uint32(h))
    return vis


def raster(hs, mi, visible, first, count, cam, vis, id_base=0):
    h, w = vis.shape
    ntri = C.c_uint64(0)
    lib().orc_raster_visbuffer(hs.ref, _p(mi), _p(visible), C.c_uint32(first), C.c_uint32(count), _p(cam),
                               C.c_uint32(id_base), C.c_uint32(w), C.c_uint32(h), _p(vis), C.byref(ntri))
    return int(ntri.value)


def raster_clip(hs, mi, visible, first, count, cam, vis, id_base=0):
    """specification-only variant with near / side-plane clipping; returns (triangles passing the cull, triangles clipped)"""
    h, w = vis.shape
    ntri, nclip = C.c_uint64(0), C.c_uint64(0)
    lib().orc_raster_visbuffer_clip(hs.ref, _p(mi), _p(visible), C.c_uint32(first), C.c_uint32(count), _p(cam),
                                    C.c_uint32(id_base), C.c_uint32(w), C.c_uint32(h), _p(vis), C.byref(ntri), C.byref(nclip))
    return int(ntri.value), int(nclip.value)


def mip_chain(level0):
    """2x2 box-filtered mip chain (rounded to nearest) of a uint8 image [h, w] or [h, w, 4] down to 1x1: list of levels"""
    levels = [np.ascontiguousarray(level0, dtype=np.uint8)]
    while levels[-1].shape[0] > 1 or levels[-1].shape[1] > 1:
        a = levels[-1].astype(np.uint32)
        h, w = a.shape[0], a.shape[1]
        ys = (np.arange(max(1, h // 2)) * 2)
        xs = (np.arange(max(1, w // 2)) * 2)
        y1, x1 = np.minimum(ys + 1, h - 1), np.minimum(xs + 1, w - 1)
        s = a[ys][:, xs] + a[ys][:, x1] + a[y1][:, xs] + a[y1][:, x1]
        levels.append(((s + 2) // 4).astype(np.uint8))
    return levels


class MaterialTable:
    """host-side OxcMaterialTable for the oracle: images = list of (texels, format) with texels a uint8 array [h, w, 4] / [h, w]
    (single level) or a LIST of such arrays (levels 0.., packed one after the other as the ABI wants them)"""

    def __init__(self, materials, images=(), samplers=None):
        self.materials = np.ascontiguousarray(materials, dtype=abi.MATERIAL_DT)
        self.texels, self.level0, self.levels = [], [], []
        for t, _ in images:
            lv = t if isinstance(t, (list, tuple)) else [t]
            self.level0.append(np.ascontiguousarray(lv[0], dtype=np.uint8))
            self.levels.append(len(lv))
            self.texels.append(np.ascontiguousarray(np.concatenate([np.ascontiguousarray(l, dtype=np.uint8).reshape(-1) for l in lv])))
        self.images = np.zeros(len(images), dtype=abi.ALPHA_IMAGE_DT)
        for i, (_, fmt) in enumerate(images):
            self.images[i] = (self.texels[i].ctypes.data, self.level0[i].shape[1], self.level0[i].shape[0], fmt, self.levels[i] if self.levels[i] > 1 else 0)
        self.samplers = None if samplers is None else np.ascontiguousarray(samplers, dtype=abi.SAMPLER_DT)
        self.ref = abi.MaterialTable()
        self.ref.materials, self.ref.material_count = self.materials.ctypes.data, len(self.materials)
        self.ref.images, self.ref.image_count = (self.images.ctypes.data if len(self.images) else None), len(self.images)
        if self.samplers is not None:
            self.ref.samplers, self.ref.sampler_count = self.samplers.ctypes.data, len(self.samplers)

    def device_images(self, ctx):
        """uploads every image (all levels) through `ctx`; returns (the `images` argument of set_materials, the device pointers)"""
        out, ptrs = [], []
        for i, t in enumerate(self.texels):
            d = ctx.alloc(t.size)
            ctx.upload(d, t)
            ptrs.append(d)
            out.append((d, int(self.images["width"][i]), int(self.images["height"][i]), int(self.images["format"][i]), int(self.images["level_count"][i])))
        return out, ptrs


def raster_alpha(hs, mi, visible, first, count, cam, vis, table: MaterialTable, id_base=0):
    """clipped raster with the alpha-tested discard of visbuffer_encode.slang:54-66; returns (triangles passing the cull,
    triangles of alpha-tested materials among them)"""
    h, w = vis.shape
    ntri, nalpha = C.c_uint64(0), C.c_uint64(0)
    lib().orc_raster_visbuffer_alpha(hs.ref, _p(mi), _p(visible), C.c_uint32(first), C.c_uint32(count), _p(cam), C.c_uint32(id_base),
                                     C.c_uint32(w), C.c_uint32(h), _p(vis), C.byref(table.ref), C.byref(ntri), C.byref(nalpha))
    return int(ntri.value), int(nalpha.value)


def raster_overdraw(hs, mi, visible, first, count, cam, overdraw, table=None):
    """RENDER_OVERDRAW of the encode pass: overdraw[h, w] (uint32) += 1 per shaded fragment of the pass's survivors"""
    h, w = overdraw.shape
    lib().orc_raster_overdraw(hs.ref, _p(mi), _p(visible), C.c_uint32(first), C.c_uint32(count), _p(cam), C.c_uint32(w), C.c_uint32(h),
                              _p(overdraw), C.byref(table.ref) if table is not None else None)


def alpha_sample(texels, fmt, u, v, sampler=None, level=0):
    """one level of an image (texels: one array, or the list of its levels) through the sampler's min filter / address modes"""
    lv = texels if isinstance(texels, (list, tuple)) else [texels]
    t = np.ascontiguousarray(np.concatenate([np.ascontiguousarray(l, dtype=np.uint8).reshape(-1) for l in lv]))
    img = np.zeros(1, dtype=abi.ALPHA_IMAGE_DT)
    img[0] = (t.ctypes.data, lv[0].shape[1], lv[0].shape[0], fmt, len(lv))
    smp = None if sampler is None else np.array([sampler], dtype=abi.SAMPLER_DT)
    lib().orc_alpha_sample.restype = C.c_float
    return float(lib().orc_alpha_sample(_p(img), _p(smp), C.c_uint32(level), C.c_float(u), C.c_float(v)))


def raster_triangle_alpha(table: MaterialTable, material_index, clip, uv, data, vis):
    """one clip-space triangle of `material_index` through the raster + alpha specification; returns 1 if it was clipped"""
    c = np.ascontiguousarray(clip, dtype=np.float32).reshape(3, 4)
    t = np.ascontiguousarray(uv, dtype=np.float32).reshape(3, 2)
    h, w = vis.shape
    return int(lib().orc_raster_triangle_alpha(C.byref(table.ref), C.c_uint32(material_index), _p(c), _p(t), C.c_uint32(data), C.c_uint32(w),
                                               C.c_uint32(h), _p(vis)))


def resolve(vis):
    h, w = vis.shape
    v32 = np.zeros((h, w), dtype=np.uint32)
    d = np.zeros((h, w), dtype=np.float32)
    lib().orc_resolve_visbuffer(_p(vis), C.c_uint32(w), C.c_uint32(h), _p(v32), _p(d))
    return v32, d


def merge_occluder_depth(vis, occluder_depth):
    """depth written by passes outside the path: vis = max(vis, depth<<32 | ~0)"""
    if occluder_depth is None:
        return vis
    packed = (occluder_depth.astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(0xFFFFFFFF)
    np.maximum(vis, packed, out=vis)
    return vis


def frame(hs, cam, width, height, mask, occluder_depth=None, first=0, count=0xFFFFFFFF, id_base_fn=None,
          between_passes=None, after_frame=None, materials=None):
    """Serial two-pass frame exactly as RendererInstance::render sequences it (RendererInstance.cpp:842-884).
    Returns dict with every intermediate the GPU parity tests compare.

    Multi-rank simulation (tests/test_dist_cpu.py): first/count = this rank's mesh-instance shard,
    id_base_fn(total) -> global id base (exchange of emitted counts), between_passes(img) / after_frame(img)
    = the vis-buffer max-reduce hooks.  `visible` holds LOCAL meshlet-instance indices; add id_base for global ids."""
    hw, hh = abi.hiz_extent(width, height)
    hiz = Hiz(hw, hh)  # cleared to 0 every frame (RendererInstance.cpp:579-588)
    mi, vis, cmd = cull_meshes(hs, cam, abi.CULL_TEST_ALL, first, count)
    id_base = int(id_base_fn(int(vis["total"][0]))) if id_base_fn else 0
    img = clear_visbuffer(width, height)
    merge_occluder_depth(img, occluder_depth)
    visible, tcmd_e = cull_meshlets_hiz(hs, mi, vis, cam, abi.CULL_TEST_ALL, hiz, mask)
    e = int(vis["early"][0])
    mask_after_early = mask.copy()
    def _raster(first_, count_):
        if materials is not None:  # visbuffer_encode.slang:54-66
            return raster_alpha(hs, mi, visible, first_, count_, cam, img, materials, id_base)[0]
        return raster_clip(hs, mi, visible, first_, count_, cam, img, id_base)[0]  # the product's raster clips what the plain spec drops

    ntri_e = _raster(0, e)
    if between_passes:
        between_passes(img)
    _, depth = resolve(img)
    build_hiz(depth, hiz)
    visible, tcmd_l = cull_meshlets_hiz(hs, mi, vis, cam, abi.CULL_TEST_ALL | abi.CULL_LATE_PASS, hiz, mask, visible)
    l = int(vis["late"][0])
    ntri_l = _raster(e, l)
    if after_frame:
        after_frame(img)
    return dict(meshlet_instances=mi, visibility=vis, visible=visible, early=e, late=l, hiz=hiz, vis64=img,
                mask_after_early=mask_after_early, ntri_early=ntri_e, ntri_late=ntri_l, cull_meshlets_cmd=cmd, id_base=id_base)


def cull_meshlets_hpb(hs, mi, vis, cam, clipmaps, dirty_flags, hpb, hpb_size, hpb_levels):
    visible = np.zeros(max(1, hs.max_meshlets), dtype=np.uint32)
    cmd = np.zeros(1, dtype=abi.DISPATCH_CMD_DT)
    cm = np.ascontiguousarray(clipmaps)
    df = np.ascontiguousarray(dirty_flags, dtype=np.uint32)
    hp = np.ascontiguousarray(hpb, dtype=np.uint8)
    lib().orc_cull_meshlets_hpb(hs.ref, _p(mi), _p(cam), _p(cm), _p(df), C.c_uint32(len(cm)), _p(hp), C.c_uint32(hpb_size),
                                C.c_uint32(hpb_levels), _p(vis), _p(visible), _p(cmd))
    return visible[: int(cmd["x"][0])], cmd


def cull_terrain(terrain, patch_minmax, cam, flags, hiz: Hiz, mask):
    n = int(terrain["patch_count"][0][0]) * int(terrain["patch_count"][0][1])
    visible = np.zeros(max(1, n), dtype=np.uint32)
    cmd = np.zeros(1, dtype=abi.DRAW_INDIRECT_DT)
    pm = np.ascontiguousarray(patch_minmax, dtype=np.float32)
    lib().orc_cull_terrain(_p(terrain), _p(pm), _p(cam), C.c_uint32(flags), hiz.ref, _p(visible), _p(mask), _p(cmd))
    return visible[: int(cmd["instance_count"][0])], cmd


def hpb_layout(size, layers, levels):
    """(offsets[levels], total bytes) of the pyramid: level l is layers x s_l x s_l bytes, s_l = max(1, size >> l)."""
    offs, off = [], 0
    for l in range(levels):
        offs.append(off)
        s = max(1, size >> l)
        off += layers * s * s
    return offs, off


def build_hpb(page_table, levels):
    """page_table: (layers, size, size) u32 -> flat pyramid bytes."""
    pt = np.ascontiguousarray(page_table, dtype=np.uint32)
    layers, size, _ = pt.shape
    _, total = hpb_layout(size, layers, levels)
    out = np.zeros(total, dtype=np.uint8)
    lib().orc_build_hpb(_p(pt), C.c_uint32(size), C.c_uint32(layers), _p(out), C.c_uint32(levels))
    return out


def log2_canonical(x):
    fn = lib().orc_log2_canonical
    fn.restype = C.c_float
    return float(fn(C.c_float(x)))


def mark_visible_pages(inv_pv, resolution, clipmaps, vsm, depth, page_tables, occupancy, request_capacity):
    """rmvsm_mark_visible_pages.slang: updates page_tables / occupancy in place; returns the allocation requests [n, 3]."""
    count = np.zeros(1, dtype=np.uint32)
    req = np.zeros((max(1, request_capacity), 3), dtype=np.int32)
    lib().orc_mark_visible_pages(_p(np.ascontiguousarray(inv_pv, dtype=np.float32)), _p(np.ascontiguousarray(resolution, dtype=np.float32)),
                                 _p(np.ascontiguousarray(clipmaps)), _p(np.ascontiguousarray(vsm)), _p(np.ascontiguousarray(depth, dtype=np.float32)),
                                 _p(page_tables), _p(occupancy), _p(count), _p(req), C.c_uint32(request_capacity))
    return req[: min(int(count[0]), request_capacity)], int(count[0])


def decode_visbuffer(hs, mi, total, cam, vis32):
    """Five (H, W, 4) f32 planes: lambda(+status), ddx, ddy, uv_normal, uv_grad."""
    v = np.ascontiguousarray(vis32, dtype=np.uint32)
    h, w = v.shape
    planes = [np.zeros((h, w, 4), dtype=np.float32) for _ in range(5)]
    lib().orc_decode_visbuffer(hs.ref, _p(mi), C.c_uint32(total), _p(cam), _p(v), C.c_uint32(w), C.c_uint32(h),
                               *[_p(x) for x in planes])
    return dict(zip(("lambda_", "ddx", "ddy", "uv_normal", "uv_grad"), planes))


def cpu_baseline_cull(hs, mi, total, cam, mode, n_threads):
    out = np.zeros(max(1, total), dtype=np.uint32)
    n = lib().orc_cpu_baseline_cull(hs.ref, _p(mi), C.c_uint32(total), _p(cam), C.c_int(mode), C.c_int(n_threads), _p(out))
    return out[: int(n)]


def cpu_frame(hs, cam, width, height, mask, occluder_depth, n_threads):
    hw, hh = abi.hiz_extent(width, height)
    mi = np.zeros(max(1, hs.max_meshlets), dtype=abi.MESHLET_INSTANCE_DT)
    visible = np.zeros(max(1, hs.max_meshlets), dtype=np.uint32)
    img = np.zeros((height, width), dtype=np.uint64)
    vc = np.zeros(1, dtype=abi.VISIBILITY_DT)
    tri = C.c_uint64(0)
    occ = np.ascontiguousarray(occluder_depth, dtype=np.float32) if occluder_depth is not None else None
    lib().orc_cpu_frame(hs.ref, _p(cam), C.c_uint32(width), C.c_uint32(height), C.c_uint32(hw), C.c_uint32(hh),
                        _p(mask), _p(occ), C.c_int(n_threads), _p(mi), _p(visible), _p(img), _p(vc), C.byref(tri))
    return dict(meshlet_instances=mi, visible=visible, vis64=img, visibility=vc, triangles=int(tri.value))
