"""ctypes binding of liboxcull.so (include/oxcull.h).  Fails loudly when the CUDA library is missing or no
GPU is present: there is no CPU fallback in the product path.
"""
import ctypes as C
import os

import numpy as np

from . import abi, build as _build

_LIB = None

OK = 0
E_NO_DEVICE = -3

# every symbol include/oxcull.h declares (tests check the .so exports all of them)
SYMBOLS = [
    "oxc_last_error", "oxc_kernel_launch_count", "oxc_version", "oxc_create", "oxc_destroy", "oxc_set_scene",
    "oxc_update_transforms", "oxc_reset_visibility_mask", "oxc_clear_hiz", "oxc_set_shard", "oxc_set_shard_auto", "oxc_cull_meshes",
    "oxc_cull_meshlets", "oxc_build_hiz", "oxc_build_hiz_packed", "oxc_build_hiz_mip0_packed", "oxc_build_hiz_from_mip0", "oxc_cull_triangles", "oxc_cull_triangles_small_primitive", "oxc_clear_visbuffer",
    "oxc_raster_visbuffer", "oxc_raster_visbuffer_clip_pass", "oxc_set_materials", "oxc_raster_overdraw", "oxc_clear_overdraw", "oxc_resolve_visbuffer", "oxc_merge_depth", "oxc_clear_visbuffer_with_depth", "oxc_cull_meshlets_multiview", "oxc_cull_meshlets_hpb", "oxc_cull_terrain", "oxc_draw_terrain",
    "oxc_decode_visbuffer", "oxc_decode_gbuffer", "oxc_build_hpb", "oxc_mark_visible_pages",
    "oxc_vsm_begin_frame", "oxc_vsm_invalidate_pages", "oxc_vsm_allocate_pages", "oxc_vsm_clear_dirty_pages", "oxc_cull_meshlets_hpb_dirty_dev",
    "oxc_vsm_draw_pages", "oxc_vsm_draw_stats", "oxc_vsm_resolve_shadows", "oxc_generate_ambient_occlusion", "oxc_apply_pbr",
    "oxc_contact_shadows", "oxc_atmosphere_transmittance", "oxc_atmosphere_sky_luts", "oxc_atmosphere_sky_ibl", "oxc_apply_pbr_atmosphere", "oxr_apply_pbr_atmosphere",
    "oxc_eye_adaptation", "oxc_bloom", "oxc_bloom_level_count", "oxc_bloom_chain_texels", "oxr_eye_adaptation", "oxr_bloom",
    "oxc_tonemap", "oxr_tonemap", "oxc_fxaa", "oxr_fxaa",
    "oxc_get_outputs", "oxc_check_status", "oxc_mark_hiz_dirty", "oxc_bind_camera_buffer", "oxc_load_camera", "oxc_debug_stats_ptr",
    "oxc_mgpu_get_unique_id", "oxc_mgpu_init", "oxc_mgpu_init_with_comm", "oxc_mgpu_shutdown", "oxc_mgpu_info", "oxc_mgpu_exchange_hiz",
    "oxc_mgpu_exchange_frame", "oxc_mgpu_stage_survivors", "oxc_mgpu_set_survivor_capacity", "oxc_copy", "oxc_sync", "oxc_device_alloc", "oxc_device_free", "oxc_debug_dequantize_half",
    "oxb_last_error", "oxb_build_mesh", "oxb_mesh_blob_size", "oxb_mesh_lod0_meshlet_count", "oxb_mesh_emit", "oxb_mesh_free", "oxb_simplify",
    "oxr_create", "oxr_destroy", "oxr_context", "oxr_update", "oxr_update_transforms", "oxr_set_external_depth", "oxr_set_terrain", "oxr_set_materials", "oxr_overdraw", "oxr_render", "oxr_submit", "oxr_wait",
    "oxr_vsm_update_pages", "oxr_vsm_pages", "oxr_vsm_draw_shadows", "oxr_vsm_resolve_shadows", "oxr_decode_gbuffer",
    "oxr_generate_ambient_occlusion", "oxr_apply_pbr", "oxr_contact_shadows", "oxr_apply_pbr_with_contact_shadows",
    "oxr_atmosphere_luts", "oxr_atmosphere_sky_ibl",
]


class OxcError(RuntimeError):
    pass


def lib_path():
    return _build.LIB


def load(build_if_missing=True):
    """Load liboxcull.so; raises if it cannot be built/loaded (never falls back to a CPU path)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(_build.LIB):
        if not build_if_missing:
            raise OxcError("liboxcull.so missing: run `python -m oxylus_b200.build` (needs nvcc); no CPU fallback exists")
        _build.build()
    lib = C.CDLL(_build.LIB)
    lib.oxc_last_error.restype = C.c_char_p
    lib.oxc_version.restype = C.c_char_p
    lib.oxc_kernel_launch_count.restype = C.c_uint64
    lib.oxr_context.restype = C.c_void_p
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    lib.oxc_create.argtypes = [i32, C.POINTER(abi.CreateInfo), C.POINTER(vp)]
    lib.oxc_destroy.argtypes = [vp]
    lib.oxc_destroy.restype = None
    lib.oxc_set_scene.argtypes = [vp, C.POINTER(abi.SceneDesc), vp]
    lib.oxc_update_transforms.argtypes = [vp, vp, u32, u32, vp]
    lib.oxc_reset_visibility_mask.argtypes = [vp, vp]
    lib.oxc_clear_hiz.argtypes = [vp, vp]
    lib.oxc_set_shard.argtypes = [vp, u32, u32, vp]
    lib.oxc_set_shard_auto.argtypes = [vp, u32, u32]
    lib.oxc_cull_meshes.argtypes = [vp, vp, u32, vp]
    lib.oxc_cull_meshlets.argtypes = [vp, vp, u32, i32, vp]
    lib.oxc_build_hiz.argtypes = [vp, vp, u32, u32, vp]
    lib.oxc_build_hiz_packed.argtypes = [vp, vp, u32, u32, vp]
    lib.oxc_build_hiz_mip0_packed.argtypes = [vp, vp, u32, u32, vp]
    lib.oxc_build_hiz_from_mip0.argtypes = [vp, vp]
    lib.oxc_cull_triangles.argtypes = [vp, vp, u32, vp]
    lib.oxc_cull_triangles_small_primitive.argtypes = [vp, vp, u32, u32, u32, vp]
    lib.oxc_clear_visbuffer.argtypes = [vp, vp, u32, u32, vp]
    lib.oxc_raster_visbuffer.argtypes = [vp, vp, u32, u32, u32, vp, i32, vp]
    lib.oxc_raster_visbuffer_clip_pass.argtypes = [vp, vp, u32, u32, u32, vp, vp]
    lib.oxc_set_materials.argtypes = [vp, C.POINTER(abi.MaterialTable), vp]
    lib.oxc_raster_overdraw.argtypes = [vp, vp, u32, u32, u32, vp, i32, vp]
    lib.oxc_clear_overdraw.argtypes = [vp, vp, u32, u32, vp]
    lib.oxc_resolve_visbuffer.argtypes = [vp, vp, u32, u32, vp, vp, vp]
    lib.oxc_merge_depth.argtypes = [vp, vp, vp, u32, u32, vp]
    lib.oxc_clear_visbuffer_with_depth.argtypes = [vp, vp, vp, u32, u32, vp]
    lib.oxc_cull_meshlets_multiview.argtypes = [vp, vp, u32, i32, vp]
    lib.oxc_cull_meshlets_hpb.argtypes = [vp, vp, vp, vp, u32, vp, u32, u32, vp]
    lib.oxc_cull_terrain.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp, vp]
    lib.oxc_draw_terrain.argtypes = [vp, vp, u32, u32, vp, vp, vp, vp, u32, u32, vp, vp]
    lib.oxc_decode_visbuffer.argtypes = [vp, vp, vp, vp, u32, u32, C.POINTER(abi.DecodeTargets), vp]
    lib.oxc_decode_gbuffer.argtypes = [vp, vp, vp, vp, u32, u32, C.POINTER(abi.GBufferTargets), vp]
    lib.oxc_build_hpb.argtypes = [vp, vp, u32, u32, vp, u32, vp]
    lib.oxc_mark_visible_pages.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, u32, vp]
    lib.oxc_vsm_begin_frame.argtypes = [vp, vp, i32, vp, vp, u32, vp, vp]
    lib.oxc_vsm_invalidate_pages.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp]
    lib.oxc_vsm_allocate_pages.argtypes = [vp, vp, vp, vp, u32, vp, u32, vp, vp, vp, vp, vp]
    lib.oxc_vsm_clear_dirty_pages.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.oxc_cull_meshlets_hpb_dirty_dev.argtypes = [vp, vp, vp, vp, u32, vp, u32, u32, vp]
    lib.oxc_vsm_draw_pages.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    lib.oxc_vsm_draw_stats.argtypes = [vp, vp, vp]
    lib.oxc_vsm_resolve_shadows.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.oxc_generate_ambient_occlusion.argtypes = [vp, C.POINTER(abi.GtaoCamera), C.POINTER(abi.GtaoSettings), vp, vp, u32, u32,
                                                   C.POINTER(abi.GtaoTargets), vp]
    lib.oxc_get_outputs.argtypes = [vp, C.POINTER(abi.Outputs)]
    lib.oxc_check_status.argtypes = [vp, vp, C.POINTER(C.c_uint32)]
    lib.oxc_mark_hiz_dirty.argtypes = [vp]
    lib.oxc_bind_camera_buffer.argtypes = [vp, vp]
    lib.oxc_load_camera.argtypes = [vp, vp, vp, vp]
    lib.oxc_mgpu_get_unique_id.argtypes = [vp]
    lib.oxc_mgpu_init.argtypes = [vp, u32, u32, vp, u32]
    lib.oxc_mgpu_init_with_comm.argtypes = [vp, vp, u32]
    lib.oxc_mgpu_shutdown.argtypes = [vp]
    lib.oxc_mgpu_info.argtypes = [vp, C.POINTER(abi.MgpuInfo)]
    lib.oxc_mgpu_exchange_hiz.argtypes = [vp, vp, u32, u32, vp]
    lib.oxc_mgpu_exchange_frame.argtypes = [vp, vp, u32, u32, i32, u32, vp]
    lib.oxc_mgpu_stage_survivors.argtypes = [vp, i32, vp]
    lib.oxc_mgpu_set_survivor_capacity.argtypes = [vp, u32]
    lib.oxc_debug_stats_ptr.argtypes = [vp]
    lib.oxc_debug_stats_ptr.restype = vp
    lib.oxc_copy.argtypes = [vp, vp, vp, u64, i32, vp]
    lib.oxc_sync.argtypes = [vp, vp]
    lib.oxc_device_alloc.argtypes = [vp, u64, C.POINTER(vp)]
    lib.oxc_device_free.argtypes = [vp, vp]
    lib.oxc_debug_dequantize_half.argtypes = [vp, vp, vp, vp]
    lib.oxb_last_error.restype = C.c_char_p
    lib.oxb_build_mesh.argtypes = [C.POINTER(abi.MeshInput), C.POINTER(vp)]
    lib.oxb_mesh_blob_size.argtypes = [vp]
    lib.oxb_mesh_blob_size.restype = u64
    lib.oxb_mesh_lod0_meshlet_count.argtypes = [vp]
    lib.oxb_mesh_lod0_meshlet_count.restype = u32
    lib.oxb_mesh_emit.argtypes = [vp, u64, vp, vp]
    lib.oxb_mesh_free.argtypes = [vp]
    lib.oxb_mesh_free.restype = None
    lib.oxb_simplify.argtypes = [vp, vp, u64, vp, vp, u32, u64, C.c_float, vp]
    lib.oxb_simplify.restype = C.c_int64
    lib.oxr_create.argtypes = [i32, C.POINTER(abi.CreateInfo), u32, u32, C.POINTER(vp)]
    lib.oxr_destroy.argtypes = [vp]
    lib.oxr_destroy.restype = None
    lib.oxr_context.argtypes = [vp]
    lib.oxr_update.argtypes = [vp, C.POINTER(abi.SceneDesc)]
    lib.oxr_update_transforms.argtypes = [vp, vp, u32, u32]
    lib.oxr_set_external_depth.argtypes = [vp, vp]
    lib.oxr_set_materials.argtypes = [vp, C.POINTER(abi.MaterialTable)]
    lib.oxr_set_terrain.argtypes = [vp, vp, u32, u32, vp, vp]
    lib.oxr_overdraw.argtypes = [vp, vp, vp]
    lib.oxr_submit.argtypes = [vp, vp, vp, vp, vp, u32, C.POINTER(C.c_int)]
    lib.oxr_wait.argtypes = [vp, i32, C.POINTER(abi.FrameResult)]
    lib.oxr_render.argtypes = [vp, vp, vp, vp, vp, vp, u32, C.POINTER(abi.FrameResult)]
    lib.oxr_vsm_update_pages.argtypes = [vp, C.POINTER(abi.VsmPageContext)]
    lib.oxr_vsm_pages.argtypes = [vp, C.POINTER(abi.VsmPages)]
    lib.oxr_vsm_draw_shadows.argtypes = [vp, vp]
    lib.oxr_vsm_resolve_shadows.argtypes = [vp, vp, vp]
    lib.oxr_decode_gbuffer.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.oxr_generate_ambient_occlusion.argtypes = [vp, vp, C.POINTER(abi.GtaoCamera), C.POINTER(abi.GtaoSettings), vp]
    lib.oxc_apply_pbr.argtypes = [vp, C.POINTER(abi.PbrCamera), C.POINTER(abi.PbrSettings), vp, C.POINTER(abi.PbrInputs), u32, u32, vp, vp]
    lib.oxr_apply_pbr.argtypes = [vp, vp, C.POINTER(abi.PbrCamera), C.POINTER(abi.PbrSettings), vp, C.c_int, vp, vp, vp]
    lib.oxc_contact_shadows.argtypes = [vp, C.POINTER(abi.ContactShadowCamera), C.POINTER(abi.ContactShadowSettings), vp, u32, u32, vp, vp]
    lib.oxr_contact_shadows.argtypes = [vp, C.POINTER(abi.ContactShadowCamera), C.POINTER(abi.ContactShadowSettings), vp]
    lib.oxr_apply_pbr_with_contact_shadows.argtypes = [vp, vp, C.POINTER(abi.PbrCamera), C.POINTER(abi.PbrSettings), vp, C.c_int, vp, vp,
                                                       vp, vp, vp]
    lib.oxc_atmosphere_transmittance.argtypes = [vp, C.POINTER(abi.Atmosphere), vp, vp]
    lib.oxc_atmosphere_sky_luts.argtypes = [vp, C.POINTER(abi.Atmosphere), C.POINTER(abi.PbrCamera), vp, C.c_float, vp, vp, vp, vp]
    lib.oxr_atmosphere_luts.argtypes = [vp, C.POINTER(abi.Atmosphere), C.POINTER(abi.PbrCamera), vp, C.c_float, vp, vp, vp]
    lib.oxc_atmosphere_sky_ibl.argtypes = [vp, C.POINTER(abi.Atmosphere), C.POINTER(abi.PbrCamera), vp, C.c_float, C.c_float, u32, vp, vp, vp,
                                           vp]
    lib.oxr_atmosphere_sky_ibl.argtypes = [vp, C.POINTER(abi.Atmosphere), C.POINTER(abi.PbrCamera), vp, C.c_float, vp]
    lib.oxr_apply_pbr_atmosphere.argtypes = [vp, vp, C.POINTER(abi.PbrCamera), C.POINTER(abi.PbrSettings), C.POINTER(abi.Atmosphere), vp,
                                             C.c_int, vp, vp, vp, vp, vp]
    lib.oxc_apply_pbr_atmosphere.argtypes = [vp, C.POINTER(abi.PbrCamera), C.POINTER(abi.PbrSettings), C.POINTER(abi.Atmosphere), vp,
                                             C.POINTER(abi.PbrInputs), C.POINTER(abi.PbrSky), u32, u32, vp, vp]
    lib.oxc_eye_adaptation.argtypes = [vp, vp, u32, u32, C.POINTER(abi.EyeAdaptationSettings), C.c_float, vp, vp, vp]
    lib.oxc_bloom.argtypes = [vp, vp, u32, u32, C.POINTER(abi.BloomSettings), vp, C.POINTER(abi.BloomTargets), vp]
    lib.oxr_eye_adaptation.argtypes = [vp, C.POINTER(abi.EyeAdaptationSettings), C.c_float, C.POINTER(abi.Exposure)]
    lib.oxr_bloom.argtypes = [vp, C.POINTER(abi.BloomSettings), vp]
    lib.oxc_tonemap.argtypes = [vp, vp, u32, u32, C.POINTER(abi.TonemapSettings), vp, vp, vp, vp]
    lib.oxr_tonemap.argtypes = [vp, C.POINTER(abi.TonemapSettings), vp]
    lib.oxc_fxaa.argtypes = [vp, vp, u32, u32, vp, vp]
    lib.oxr_fxaa.argtypes = [vp, vp]
    lib.oxc_bloom_level_count.restype, lib.oxc_bloom_level_count.argtypes = u32, [u32, u32]
    lib.oxc_bloom_chain_texels.restype, lib.oxc_bloom_chain_texels.argtypes = C.c_uint64, [u32, u32]
    _LIB = lib
    return lib


def _check(rc, what):
    if rc != OK:
        raise OxcError(f"{what} failed ({rc}): {load().oxc_last_error().decode()}")


def kernel_launch_count():
    return int(load().oxc_kernel_launch_count())


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return C.c_void_p(a.ctypes.data)
    return C.c_void_p(int(a))


def simplify(indices, positions, normals, target_index_count, target_error=3.4028234663852886e38):
    """oxb_simplify: -> (new indices u32 array, result_error np.float32).  Host-only: works without a GPU."""
    lib = load()
    idx = np.ascontiguousarray(indices, dtype=np.uint32).reshape(-1)
    pos = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
    nrm = None if normals is None else np.ascontiguousarray(normals, dtype=np.float32).reshape(-1, 3)
    dst = np.zeros(max(idx.size, 1), dtype=np.uint32)
    err = np.zeros(1, dtype=np.float32)
    n = lib.oxb_simplify(_ptr(dst), _ptr(idx), idx.size, _ptr(pos), _ptr(nrm), len(pos), int(target_index_count), float(target_error), _ptr(err))
    if n < 0:
        raise OxcError(f"oxb_simplify failed ({n}): {lib.oxb_last_error().decode()}")
    return dst[:n].copy(), err[0]


class BuiltMesh:
    """OxbMesh wrapper: one mesh run through the host-side builder (oxb_build_mesh).  lods = [(indices, error), ...],
    LOD 0 first.  Host-only: works without a GPU."""

    def __init__(self, positions, lods, normals=None, texcoords=None, spatial=False, auto_lods=False):
        self.lib = load()
        pos = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
        nrm = None if normals is None else np.ascontiguousarray(normals, dtype=np.float32).reshape(-1, 3)
        tc = None if texcoords is None else np.ascontiguousarray(texcoords, dtype=np.float32).reshape(-1, 2)
        idx = [np.ascontiguousarray(i, dtype=np.uint32).reshape(-1) for i, _ in lods]
        mi = abi.MeshInput()
        mi.positions, mi.normals, mi.texcoords = _ptr(pos), _ptr(nrm), _ptr(tc)
        mi.vertex_count, mi.lod_count = len(pos), len(lods)
        mi.cluster_mode = 1 if spatial else 0
        mi.auto_lods = 1 if auto_lods else 0
        for l, (a, (_, err)) in enumerate(zip(idx, lods)):
            mi.lod_indices[l] = a.ctypes.data
            mi.lod_index_counts[l] = a.size
            mi.lod_errors[l] = float(err)
        h = C.c_void_p()
        rc = self.lib.oxb_build_mesh(C.byref(mi), C.byref(h))
        if rc != OK:
            raise OxcError(f"oxb_build_mesh failed ({rc}): {self.lib.oxb_last_error().decode()}")
        self.h = h
        self.blob_size = int(self.lib.oxb_mesh_blob_size(h))
        self.lod0_meshlet_count = int(self.lib.oxb_mesh_lod0_meshlet_count(h))

    def emit(self, base_offset, dst: np.ndarray):
        """copies the blob into dst (uint8 view at scene_blob[base_offset:]) and returns the rebased MESH_DT record"""
        assert dst.dtype == np.uint8 and dst.size >= self.blob_size
        rec = np.zeros(1, dtype=abi.MESH_DT)
        rc = self.lib.oxb_mesh_emit(self.h, base_offset, _ptr(dst), _ptr(rec))
        if rc != OK:
            raise OxcError(f"oxb_mesh_emit failed ({rc}): {self.lib.oxb_last_error().decode()}")
        return rec

    def close(self):
        if getattr(self, "h", None):
            self.lib.oxb_mesh_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def assemble_scene(built, mesh_of_instance, transforms, width, height, transform_index=None, seed=0):
    """Scene tables from builder output (the shape Scene::runtime_update hands over, Scene.cpp:1226-1290): one blob of
    all meshes, mesh instances with LOD-0 prefix sums as visibility offsets (Scene.cpp:1255-1260)."""
    from . import synth

    bases, off = [], 0
    for b in built:
        bases.append(off)
        off += b.blob_size
    blob = np.zeros(max(16, off), dtype=np.uint8)
    meshes = np.zeros(len(built), dtype=abi.MESH_DT)
    for i, b in enumerate(built):
        meshes[i] = b.emit(bases[i], blob[bases[i]:])[0]
    mesh_of_instance = np.asarray(mesh_of_instance, dtype=np.uint32)
    inst = np.zeros(len(mesh_of_instance), dtype=abi.MESH_INSTANCE_DT)
    inst["mesh_index"] = mesh_of_instance
    inst["transform_index"] = np.arange(len(inst)) if transform_index is None else transform_index
    lod0 = np.array([b.lod0_meshlet_count for b in built], dtype=np.int64)[mesh_of_instance]
    inst["meshlet_instance_visibility_offset"] = np.concatenate([[0], np.cumsum(lod0)[:-1]]) if len(inst) else []
    xf = np.zeros(len(transforms), dtype=abi.TRANSFORM_DT)
    xf["world"] = np.asarray(transforms, dtype=np.float32).reshape(len(transforms), 16)
    return synth.Scene(meshes, inst, xf, blob, int(lod0.sum()), width, height, seed)


def material_table(materials, images=None, samplers=None):
    """(abi.MaterialTable or None, the arrays it points to) from an abi.MATERIAL_DT array, a list of (device pointer, width,
    height, format[, level_count]) and an optional abi.SAMPLER_DT array"""
    if materials is None or len(materials) == 0:
        return None, ()
    mats = np.ascontiguousarray(materials, dtype=abi.MATERIAL_DT)
    imgs = np.zeros(len(images or []), dtype=abi.ALPHA_IMAGE_DT)
    for i, im in enumerate(images or []):  # (device pointer, width, height, format[, level_count])
        imgs[i] = (int(im[0]), im[1], im[2], im[3], im[4] if len(im) > 4 else 0)
    smp = None if samplers is None else np.ascontiguousarray(samplers, dtype=abi.SAMPLER_DT)
    t = abi.MaterialTable()
    t.materials, t.material_count = mats.ctypes.data, len(mats)
    t.images, t.image_count = (imgs.ctypes.data if len(imgs) else None), len(imgs)
    t.samplers, t.sampler_count = (None if smp is None else smp.ctypes.data), (0 if smp is None else len(smp))
    return t, (mats, imgs, smp)


class Context:
    """OxcContext wrapper.  `stream` is a raw cudaStream_t handle (int; 0 = default stream)."""

    def __init__(self, device, max_mesh_instances, max_meshlet_instances, hiz_w, hiz_h, alloc_reordered_indices=False,
                 max_views=0, stream=0, max_mask_bits=0, wide_ids=False):
        self.lib = load()
        info = abi.CreateInfo(max_mesh_instances, max_meshlet_instances, hiz_w, hiz_h, int(alloc_reordered_indices), max_views,
                              max_mask_bits, int(wide_ids))
        h = C.c_void_p()
        _check(self.lib.oxc_create(device, C.byref(info), C.byref(h)), "oxc_create")
        self.h = h
        self.stream = stream
        self.max_meshlet_instances = max_meshlet_instances
        self.max_mesh_instances = max_mesh_instances
        self._keep = None
        self.out = abi.Outputs()
        _check(self.lib.oxc_get_outputs(self.h, C.byref(self.out)), "oxc_get_outputs")
        self._owned = True

    @classmethod
    def from_handle(cls, handle, stream=0):
        self = cls.__new__(cls)
        self.lib = load()
        self.h = C.c_void_p(handle)
        self.stream = stream
        self._keep = None
        self.out = abi.Outputs()
        _check(self.lib.oxc_get_outputs(self.h, C.byref(self.out)), "oxc_get_outputs")
        self._owned = False
        return self

    def close(self):
        if getattr(self, "h", None) and self._owned:
            self.lib.oxc_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- scene ----
    def set_scene(self, scene):
        from . import synth

        desc, keep = synth.scene_desc(scene)
        self._keep = keep
        _check(self.lib.oxc_set_scene(self.h, C.byref(desc), self.stream), "oxc_set_scene")
        self.sync()

    def update_transforms(self, transforms, first=0):
        t = np.ascontiguousarray(transforms)
        _check(self.lib.oxc_update_transforms(self.h, _ptr(t), first, len(t), self.stream), "oxc_update_transforms")
        self.sync()

    def reset_visibility_mask(self):
        _check(self.lib.oxc_reset_visibility_mask(self.h, self.stream), "oxc_reset_visibility_mask")

    def clear_hiz(self):
        _check(self.lib.oxc_clear_hiz(self.h, self.stream), "oxc_clear_hiz")

    def set_shard(self, first, count, id_base_dev=None):
        _check(self.lib.oxc_set_shard(self.h, first, count, _ptr(id_base_dev)), "oxc_set_shard")

    def set_shard_auto(self, first, count):
        _check(self.lib.oxc_set_shard_auto(self.h, first, count), "oxc_set_shard_auto")

    # ---- passes ----
    def cull_meshes(self, cam, flags=abi.CULL_TEST_ALL):
        _check(self.lib.oxc_cull_meshes(self.h, _ptr(cam), flags, self.stream), "oxc_cull_meshes")

    def cull_meshlets(self, cam, flags, use_hiz=True):
        _check(self.lib.oxc_cull_meshlets(self.h, _ptr(cam), flags, int(use_hiz), self.stream), "oxc_cull_meshlets")

    def build_hiz(self, depth_dev, w, h):
        _check(self.lib.oxc_build_hiz(self.h, _ptr(depth_dev), w, h, self.stream), "oxc_build_hiz")

    def build_hiz_packed(self, vis_dev, w, h):
        _check(self.lib.oxc_build_hiz_packed(self.h, _ptr(vis_dev), w, h, self.stream), "oxc_build_hiz_packed")

    def build_hiz_mip0_packed(self, vis_dev, w, h):
        _check(self.lib.oxc_build_hiz_mip0_packed(self.h, _ptr(vis_dev), w, h, self.stream), "oxc_build_hiz_mip0_packed")

    def build_hiz_from_mip0(self):
        _check(self.lib.oxc_build_hiz_from_mip0(self.h, self.stream), "oxc_build_hiz_from_mip0")

    def cull_triangles(self, cam, flags):
        _check(self.lib.oxc_cull_triangles(self.h, _ptr(cam), flags, self.stream), "oxc_cull_triangles")

    def cull_triangles_small_primitive(self, cam, flags, w, h):
        _check(self.lib.oxc_cull_triangles_small_primitive(self.h, _ptr(cam), flags, w, h, self.stream), "oxc_cull_triangles_small_primitive")

    def clear_visbuffer(self, vis_dev, w, h):
        _check(self.lib.oxc_clear_visbuffer(self.h, _ptr(vis_dev), w, h, self.stream), "oxc_clear_visbuffer")

    def raster_visbuffer(self, cam, flags, w, h, vis_dev, small_primitive_cull=False):
        _check(self.lib.oxc_raster_visbuffer(self.h, _ptr(cam), flags, w, h, _ptr(vis_dev), int(small_primitive_cull), self.stream),
               "oxc_raster_visbuffer")

    def set_materials(self, materials, images=None, samplers=None):
        """oxc_set_materials: `materials` abi.MATERIAL_DT array (None switches the alpha test off); `images` a list of
        (device pointer, width, height, format); `samplers` an abi.SAMPLER_DT array or None (linear + repeat)"""
        t, keep = material_table(materials, images, samplers)
        _check(self.lib.oxc_set_materials(self.h, None if t is None else C.byref(t), self.stream), "oxc_set_materials")

    def raster_overdraw(self, cam, flags, w, h, overdraw_dev, after_frame=False):
        _check(self.lib.oxc_raster_overdraw(self.h, _ptr(cam), flags, w, h, _ptr(overdraw_dev), int(after_frame), self.stream), "oxc_raster_overdraw")

    def clear_overdraw(self, overdraw_dev, w, h):
        _check(self.lib.oxc_clear_overdraw(self.h, _ptr(overdraw_dev), w, h, self.stream), "oxc_clear_overdraw")

    def raster_visbuffer_clip_pass(self, cam, flags, w, h, vis_dev):
        _check(self.lib.oxc_raster_visbuffer_clip_pass(self.h, _ptr(cam), flags, w, h, _ptr(vis_dev), self.stream),
               "oxc_raster_visbuffer_clip_pass")

    def resolve_visbuffer(self, vis_dev, w, h, vis32_dev, depth_dev):
        _check(self.lib.oxc_resolve_visbuffer(self.h, _ptr(vis_dev), w, h, _ptr(vis32_dev), _ptr(depth_dev), self.stream),
               "oxc_resolve_visbuffer")

    def clear_visbuffer_with_depth(self, vis_dev, depth_dev, w, h):
        _check(self.lib.oxc_clear_visbuffer_with_depth(self.h, _ptr(vis_dev), _ptr(depth_dev), w, h, self.stream),
               "oxc_clear_visbuffer_with_depth")

    def merge_depth(self, vis_dev, depth_dev, w, h):
        _check(self.lib.oxc_merge_depth(self.h, _ptr(vis_dev), _ptr(depth_dev), w, h, self.stream), "oxc_merge_depth")

    def cull_meshlets_multiview(self, views, directional):
        v = np.ascontiguousarray(views)
        _check(self.lib.oxc_cull_meshlets_multiview(self.h, _ptr(v), len(v), int(directional), self.stream),
               "oxc_cull_meshlets_multiview")

    def cull_meshlets_hpb(self, cam, clipmaps, dirty_flags, hpb_dev, hpb_size, hpb_levels):
        cm = np.ascontiguousarray(clipmaps)
        df = np.ascontiguousarray(dirty_flags, dtype=np.uint32)
        _check(self.lib.oxc_cull_meshlets_hpb(self.h, _ptr(cam), _ptr(cm), _ptr(df), len(cm), _ptr(hpb_dev), hpb_size, hpb_levels,
                                              self.stream), "oxc_cull_meshlets_hpb")

    def cull_terrain(self, terrain, patch_minmax_dev, cam, flags, visible_patches_dev, mask_dev, draw_cmd_dev):
        t = np.ascontiguousarray(terrain)
        _check(self.lib.oxc_cull_terrain(self.h, _ptr(t), _ptr(patch_minmax_dev), _ptr(cam), flags, _ptr(visible_patches_dev),
                                         _ptr(mask_dev), _ptr(draw_cmd_dev), self.stream), "oxc_cull_terrain")

    def draw_terrain(self, heightmap_dev, res_x, res_y, settings, visible_patches_dev, draw_cmd_dev, cam, w, h, vis_dev):
        """oxc_draw_terrain: tessellates the visible patches of oxc_cull_terrain over the R16 heightmap (res_x x res_y uint16 on the
        device) and rasterises them into the packed vis buffer; settings is an abi.TERRAIN_DRAW_SETTINGS_DT record"""
        st = np.ascontiguousarray(settings)
        _check(self.lib.oxc_draw_terrain(self.h, _ptr(heightmap_dev), res_x, res_y, _ptr(st), _ptr(visible_patches_dev), _ptr(draw_cmd_dev),
                                         _ptr(cam), w, h, _ptr(vis_dev), self.stream), "oxc_draw_terrain")

    def decode_visbuffer(self, cam, w, h, targets, vis64_dev=None, vis32_dev=None):
        """targets: dict with any of lambda_, ddx, ddy, uv_normal, uv_grad -> device pointers (float4 planes)."""
        t = abi.DecodeTargets(*[targets.get(k) for k in ("lambda_", "ddx", "ddy", "uv_normal", "uv_grad")])
        _check(self.lib.oxc_decode_visbuffer(self.h, _ptr(cam), _ptr(vis64_dev), _ptr(vis32_dev), w, h, C.byref(t), self.stream),
               "oxc_decode_visbuffer")

    def decode_gbuffer(self, cam, w, h, targets, vis64_dev=None, vis32_dev=None):
        """oxc_decode_gbuffer: targets a dict with any of albedo, normal, emissive, metallic_roughness_occlusion -> device pointers
        (float4 planes); the material table of the last set_materials"""
        t = abi.GBufferTargets(*[targets.get(k) for k in abi.GBUFFER_PLANES])
        _check(self.lib.oxc_decode_gbuffer(self.h, _ptr(cam), _ptr(vis64_dev), _ptr(vis32_dev), w, h, C.byref(t), self.stream),
               "oxc_decode_gbuffer")

    def mark_visible_pages(self, inv_pv, resolution, clipmaps, vsm, depth_dev, page_tables_dev, occupancy_dev, request_count_dev, requests_dev,
                           request_capacity):
        ipv = np.ascontiguousarray(inv_pv, dtype=np.float32)
        res = np.ascontiguousarray(resolution, dtype=np.float32)
        cm = np.ascontiguousarray(clipmaps)
        vc = np.ascontiguousarray(vsm)
        _check(self.lib.oxc_mark_visible_pages(self.h, _ptr(ipv), _ptr(res), _ptr(cm), _ptr(vc), _ptr(depth_dev), _ptr(page_tables_dev),
                                               _ptr(occupancy_dev), _ptr(request_count_dev), _ptr(requests_dev), request_capacity, self.stream),
               "oxc_mark_visible_pages")

    # ---- virtual shadow map page bookkeeping (oxc_vsm_*); `vsm` is an abi.VSM_CONTEXT_DT record, pointers are device pointers ----
    def vsm_begin_frame(self, vsm, sun_moved, page_tables_dev, occupancy_dev, physical_page_count, request_count_dev):
        vc = np.ascontiguousarray(vsm)
        _check(self.lib.oxc_vsm_begin_frame(self.h, _ptr(vc), int(bool(sun_moved)), _ptr(page_tables_dev), _ptr(occupancy_dev), physical_page_count,
                                            _ptr(request_count_dev), self.stream), "oxc_vsm_begin_frame")

    def vsm_invalidate_pages(self, vsm, clipmaps, dirty_dev, dirty_count, previous_transforms_dev, page_tables_dev):
        vc, cm = np.ascontiguousarray(vsm), np.ascontiguousarray(clipmaps)
        _check(self.lib.oxc_vsm_invalidate_pages(self.h, _ptr(vc), _ptr(cm), _ptr(dirty_dev), dirty_count, _ptr(previous_transforms_dev),
                                                 _ptr(page_tables_dev), self.stream), "oxc_vsm_invalidate_pages")

    def vsm_allocate_pages(self, vsm, page_tables_dev, occupancy_dev, physical_page_count, requests_dev, request_capacity, allocator_dev,
                           free_list_dev, dirty_coords_dev, dirty_flags_dev):
        vc = np.ascontiguousarray(vsm)
        _check(self.lib.oxc_vsm_allocate_pages(self.h, _ptr(vc), _ptr(page_tables_dev), _ptr(occupancy_dev), physical_page_count, _ptr(requests_dev),
                                               request_capacity, _ptr(allocator_dev), _ptr(free_list_dev), _ptr(dirty_coords_dev),
                                               _ptr(dirty_flags_dev), self.stream), "oxc_vsm_allocate_pages")

    def vsm_clear_dirty_pages(self, vsm, allocator_dev, dirty_coords_dev, atlas_dev):
        vc = np.ascontiguousarray(vsm)
        _check(self.lib.oxc_vsm_clear_dirty_pages(self.h, _ptr(vc), _ptr(allocator_dev), _ptr(dirty_coords_dev), _ptr(atlas_dev), self.stream),
               "oxc_vsm_clear_dirty_pages")

    def cull_meshlets_hpb_dirty_dev(self, cam, clipmaps, dirty_flags_dev, hpb_dev, hpb_size, hpb_levels):
        cm = np.ascontiguousarray(clipmaps)
        _check(self.lib.oxc_cull_meshlets_hpb_dirty_dev(self.h, _ptr(cam), _ptr(cm), _ptr(dirty_flags_dev), len(cm), _ptr(hpb_dev), hpb_size,
                                                        hpb_levels, self.stream), "oxc_cull_meshlets_hpb_dirty_dev")

    def vsm_draw_pages(self, vsm, coarse, clipmaps, dirty_flags_dev, page_tables_dev, atlas_dev):
        """oxc_vsm_draw_pages: the survivors of the last HPB cull drawn into the physical atlas (device pointers)"""
        vc, cm = np.ascontiguousarray(vsm), np.ascontiguousarray(clipmaps)
        _check(self.lib.oxc_vsm_draw_pages(self.h, _ptr(vc), _ptr(coarse), _ptr(cm), _ptr(dirty_flags_dev), _ptr(page_tables_dev), _ptr(atlas_dev),
                                           self.stream), "oxc_vsm_draw_pages")

    def vsm_draw_stats(self):
        """oxc_vsm_draw_stats: dict(items=, pairs=) of the last oxc_vsm_draw_pages"""
        out = np.zeros(2, dtype=np.uint32)
        _check(self.lib.oxc_vsm_draw_stats(self.h, _ptr(out), self.stream), "oxc_vsm_draw_stats")
        return dict(items=int(out[0]), pairs=int(out[1]))

    def vsm_resolve_shadows(self, vsm, inv_pv, resolution, clipmaps, depth_dev, normals_dev, page_tables_dev, atlas_dev, shadow_dev):
        """oxc_vsm_resolve_shadows: the PCSS shadow factor per pixel of vsm's depth_extent into shadow_dev (device pointers; normals_dev:
        float4 per pixel, oct(world normal) in .zw)"""
        vc, cm = np.ascontiguousarray(vsm), np.ascontiguousarray(clipmaps)
        ipv, res = np.ascontiguousarray(inv_pv, dtype=np.float32), np.ascontiguousarray(resolution, dtype=np.float32)
        _check(self.lib.oxc_vsm_resolve_shadows(self.h, _ptr(vc), _ptr(ipv), _ptr(res), _ptr(cm), _ptr(depth_dev), _ptr(normals_dev),
                                                _ptr(page_tables_dev), _ptr(atlas_dev), _ptr(shadow_dev), self.stream), "oxc_vsm_resolve_shadows")

    def generate_ambient_occlusion(self, gtao_camera, settings, depth_dev, normals_dev, w, h, targets):
        """oxc_generate_ambient_occlusion: prefilter, sector pass and denoise of a w x h frame.  gtao_camera / settings: abi.GtaoCamera /
        abi.GtaoSettings; targets: dict depth_mips, edges, noisy_occlusion, ambient_occlusion -> device pointers (or abi.GtaoTargets)"""
        t = targets if isinstance(targets, abi.GtaoTargets) else abi.GtaoTargets(*[targets.get(k) for k in
                                                                                    ("depth_mips", "edges", "noisy_occlusion", "ambient_occlusion")])
        _check(self.lib.oxc_generate_ambient_occlusion(self.h, C.byref(gtao_camera), C.byref(settings), _ptr(depth_dev), _ptr(normals_dev), w, h,
                                                       C.byref(t), self.stream), "oxc_generate_ambient_occlusion")

    def apply_pbr(self, pbr_camera, settings, lights_dev, inputs, w, h, out_dev):
        """oxc_apply_pbr: the lit RGBA (float4 per pixel) of a w x h frame into out_dev.  pbr_camera / settings: abi.PbrCamera /
        abi.PbrSettings; lights_dev: settings.light_count abi.Light records on the device; inputs: dict depth, albedo, normal, emissive,
        metallic_roughness_occlusion, ambient_occlusion, shadow, contact_shadow -> device pointers (or abi.PbrInputs), missing = NULL"""
        t = inputs if isinstance(inputs, abi.PbrInputs) else abi.PbrInputs(*[inputs.get(k) for k in abi.PBR_INPUTS])
        _check(self.lib.oxc_apply_pbr(self.h, C.byref(pbr_camera), C.byref(settings), _ptr(lights_dev), C.byref(t), w, h, _ptr(out_dev),
                                      self.stream), "oxc_apply_pbr")

    def apply_pbr_atmosphere(self, pbr_camera, settings, atmosphere, lights_dev, inputs, sky, w, h, out_dev):
        """oxc_apply_pbr_atmosphere: the lit RGBA (float4 per pixel) of a w x h frame under the atmosphere into out_dev.  As apply_pbr, plus
        atmosphere (abi.Atmosphere) and sky: dict transmittance, sky_view, aerial_perspective, sky_cube -> device pointers (or
        abi.PbrSky); settings must carry SCENE_HAS_ATMOSPHERE"""
        t = inputs if isinstance(inputs, abi.PbrInputs) else abi.PbrInputs(*[inputs.get(k) for k in abi.PBR_INPUTS])
        k = sky if isinstance(sky, abi.PbrSky) else abi.PbrSky(*[sky.get(n) for n in abi.PBR_SKY_PLANES])
        _check(self.lib.oxc_apply_pbr_atmosphere(self.h, C.byref(pbr_camera), C.byref(settings), C.byref(atmosphere), _ptr(lights_dev),
                                                 C.byref(t), C.byref(k), w, h, _ptr(out_dev), self.stream), "oxc_apply_pbr_atmosphere")

    def eye_adaptation(self, frame_dev, w, h, settings, delta_time, exposure_dev, histogram_dev):
        """oxc_eye_adaptation: the 256-bin luminance histogram of a w x h float4 frame into histogram_dev (zeroed by the call) and the
        exposure record (abi.Exposure, 8 B at exposure_dev) updated in place.  settings: abi.EyeAdaptationSettings"""
        _check(self.lib.oxc_eye_adaptation(self.h, _ptr(frame_dev), w, h, C.byref(settings), float(np.float32(delta_time)), _ptr(exposure_dev),
                                           _ptr(histogram_dev), self.stream), "oxc_eye_adaptation")

    def bloom(self, frame_dev, w, h, settings, exposure_dev, downsampled_dev, upsampled_dev):
        """oxc_bloom: the prefilter, downsample and upsample chains of a w x h float4 frame into the two chains (abi.bloom_levels layout,
        abi.bloom_chain_texels float4 each); the bloom image is upsampled level 0.  settings: abi.BloomSettings; exposure_dev is read
        under SCENE_HAS_EYE_ADAPTATION only"""
        t = abi.BloomTargets(*[None if a is None else int(a) for a in (downsampled_dev, upsampled_dev)])
        _check(self.lib.oxc_bloom(self.h, _ptr(frame_dev), w, h, C.byref(settings), _ptr(exposure_dev), C.byref(t), self.stream), "oxc_bloom")

    def tonemap(self, frame_dev, w, h, settings, exposure_dev, bloom_dev, out_dev):
        """oxc_tonemap: the exposure, bloom composite, curve and lens effects of a w x h float4 frame into out_dev (w x h float4).
        settings: abi.TonemapSettings; exposure_dev is read under SCENE_HAS_EYE_ADAPTATION only, bloom_dev ((w // 2) x (h // 2) float4,
        upsampled level 0 of bloom's chain) under SCENE_HAS_BLOOM only"""
        _check(self.lib.oxc_tonemap(self.h, _ptr(frame_dev), w, h, C.byref(settings), _ptr(exposure_dev), _ptr(bloom_dev), _ptr(out_dev),
                                    self.stream), "oxc_tonemap")

    def fxaa(self, frame_dev, w, h, out_dev):
        """oxc_fxaa: FXAA of a w x h float4 frame into out_dev (w x h float4, sharing no byte with the frame)"""
        _check(self.lib.oxc_fxaa(self.h, _ptr(frame_dev), w, h, _ptr(out_dev), self.stream), "oxc_fxaa")

    def atmosphere_transmittance(self, atmosphere, lut_dev):
        """oxc_atmosphere_transmittance: the transmittance LUT (binary16 RGBA, atmosphere.transmittance_lut_size) into lut_dev"""
        _check(self.lib.oxc_atmosphere_transmittance(self.h, C.byref(atmosphere), _ptr(lut_dev), self.stream), "oxc_atmosphere_transmittance")

    def atmosphere_sky_luts(self, atmosphere, camera, sun_direction, sun_intensity, transmittance_dev, sky_view_dev, aerial_perspective_dev):
        """oxc_atmosphere_sky_luts: the sky-view and aerial-perspective LUTs (binary16 RGBA) over the transmittance LUT.  camera:
        abi.PbrCamera; sun_direction: 3 floats, as given"""
        sun = (C.c_float * 3)(*[float(np.float32(v)) for v in sun_direction])
        _check(self.lib.oxc_atmosphere_sky_luts(self.h, C.byref(atmosphere), C.byref(camera), sun, float(np.float32(sun_intensity)),
                                                _ptr(transmittance_dev), _ptr(sky_view_dev), _ptr(aerial_perspective_dev), self.stream),
               "oxc_atmosphere_sky_luts")

    def atmosphere_sky_ibl(self, atmosphere, camera, sun_direction, sun_intensity, sun_ambient_strength, frame_index, transmittance_dev,
                           sky_view_dev, cube_dev):
        """oxc_atmosphere_sky_ibl: the next sky IBL cube (6 x 32 x 32 binary16 RGBA, read and written in place at cube_dev; zeroed = no
        history) over the transmittance and sky-view LUTs.  camera: abi.PbrCamera (only its position is read); sun_direction: 3 floats,
        as given; the reference passes sun_ambient_strength 0.15 and its frame counter as frame_index"""
        sun = (C.c_float * 3)(*[float(np.float32(v)) for v in sun_direction])
        _check(self.lib.oxc_atmosphere_sky_ibl(self.h, C.byref(atmosphere), C.byref(camera), sun, float(np.float32(sun_intensity)),
                                               float(np.float32(sun_ambient_strength)), int(frame_index) & 0xFFFFFFFF, _ptr(transmittance_dev),
                                               _ptr(sky_view_dev), _ptr(cube_dev), self.stream), "oxc_atmosphere_sky_ibl")

    def contact_shadows(self, contact_camera, settings, depth_dev, w, h, out_dev):
        """oxc_contact_shadows: 1 - the contact shadow (f32 per pixel) of a w x h frame into out_dev.  contact_camera / settings:
        abi.ContactShadowCamera / abi.ContactShadowSettings"""
        _check(self.lib.oxc_contact_shadows(self.h, C.byref(contact_camera), C.byref(settings), _ptr(depth_dev), w, h, _ptr(out_dev), self.stream),
               "oxc_contact_shadows")

    def build_hpb(self, page_table_dev, size, layers, hpb_dev, levels):
        _check(self.lib.oxc_build_hpb(self.h, _ptr(page_table_dev), size, layers, _ptr(hpb_dev), levels, self.stream), "oxc_build_hpb")

    def check_status(self):
        """Raises OxcError when a kernel raised a sticky OXC_STATUS_* bit (and clears it); returns the flags (0) otherwise."""
        f = C.c_uint32(0)
        _check(self.lib.oxc_check_status(self.h, self.stream, C.byref(f)), "oxc_check_status")
        return f.value

    def status_flags(self):
        """The sticky status word without raising / clearing."""
        return int(self.download(self.out.status_flags, np.uint32, 1)[0])

    # ---- multi-GPU exchange (oxc_mgpu_*) ----
    @staticmethod
    def mgpu_unique_id():
        """128-byte communicator id (rank 0 creates it; the host hands it to the other ranks)."""
        buf = (C.c_uint8 * abi.MGPU_ID_BYTES)()
        _check(load().oxc_mgpu_get_unique_id(buf), "oxc_mgpu_get_unique_id")
        return bytes(buf)

    def mgpu_init(self, rank, world, unique_id, survivor_capacity=0):
        buf = (C.c_uint8 * abi.MGPU_ID_BYTES).from_buffer_copy(bytes(unique_id))
        _check(self.lib.oxc_mgpu_init(self.h, rank, world, buf, survivor_capacity), "oxc_mgpu_init")
        return self.mgpu_info()

    def mgpu_info(self):
        info = abi.MgpuInfo()
        _check(self.lib.oxc_mgpu_info(self.h, C.byref(info)), "oxc_mgpu_info")
        return info

    def mgpu_exchange_hiz(self, vis_dev, w, h):
        _check(self.lib.oxc_mgpu_exchange_hiz(self.h, _ptr(vis_dev), w, h, self.stream), "oxc_mgpu_exchange_hiz")

    def mgpu_stage_survivors(self, slot=0):
        _check(self.lib.oxc_mgpu_stage_survivors(self.h, slot, self.stream), "oxc_mgpu_stage_survivors")

    def mgpu_exchange_frame(self, vis_dev, w, h, slot=0, stream=None, already_staged=False):
        _check(self.lib.oxc_mgpu_exchange_frame(self.h, _ptr(vis_dev), w, h, slot, 1 if already_staged else 0,
                                                self.stream if stream is None else stream), "oxc_mgpu_exchange_frame")

    def mgpu_set_survivor_capacity(self, capacity):
        _check(self.lib.oxc_mgpu_set_survivor_capacity(self.h, capacity), "oxc_mgpu_set_survivor_capacity")
        return self.mgpu_info()

    def mgpu_shutdown(self):
        _check(self.lib.oxc_mgpu_shutdown(self.h), "oxc_mgpu_shutdown")

    def mgpu_gathered(self, slot=0):
        """(counts[world, 4] = total, early, late, gathered ; list of per-rank id arrays) of the last exchange_frame into `slot`."""
        info = self.mgpu_info()
        cnt = self.download(info.gathered_counts[slot], np.uint32, info.world * 4).reshape(info.world, 4)
        ids = self.download(info.gathered_ids[slot], np.uint32, info.world * info.survivor_capacity).reshape(info.world, info.survivor_capacity)
        return cnt, [ids[r, : cnt[r, 3]] for r in range(info.world)]

    def debug_stats_ptr(self):
        return self.lib.oxc_debug_stats_ptr(self.h)

    def mark_hiz_dirty(self):
        _check(self.lib.oxc_mark_hiz_dirty(self.h), "oxc_mark_hiz_dirty")

    def bind_camera_buffer(self, camera_dev):
        """oxc_bind_camera_buffer: a device OxcCullCamera the main-view passes read instead of their argument (None unbinds)"""
        _check(self.lib.oxc_bind_camera_buffer(self.h, _ptr(camera_dev)), "oxc_bind_camera_buffer")

    # ---- plumbing ----
    def sync(self):
        _check(self.lib.oxc_sync(self.h, self.stream), "oxc_sync")

    def alloc(self, nbytes):
        p = C.c_void_p()
        _check(self.lib.oxc_device_alloc(self.h, nbytes, C.byref(p)), "oxc_device_alloc")
        return p.value

    def free(self, ptr):
        _check(self.lib.oxc_device_free(self.h, _ptr(ptr)), "oxc_device_free")

    def upload(self, dev_ptr, host: np.ndarray):
        host = np.ascontiguousarray(host)
        _check(self.lib.oxc_copy(self.h, _ptr(dev_ptr), _ptr(host), host.nbytes, 0, self.stream), "oxc_copy h2d")
        self.sync()

    def download(self, dev_ptr, dtype, count):
        out = np.empty(count, dtype=dtype)
        if count:
            _check(self.lib.oxc_copy(self.h, _ptr(out), _ptr(dev_ptr), out.nbytes, 1, self.stream), "oxc_copy d2h")
        self.sync()
        return out

    # ---- typed readbacks of OxcOutputs ----
    def visibility(self):
        return self.download(self.out.visibility, abi.VISIBILITY_DT, 1)

    def meshlet_instances(self, n):
        return self.download(self.out.meshlet_instances, abi.MESHLET_INSTANCE_DT, n)

    def visible_indices(self, n):
        return self.download(self.out.visible_meshlet_instances_indices, np.uint32, n)

    def mask(self):
        return self.download(self.out.meshlet_instance_visibility_mask, np.uint32, self.out.visibility_mask_words)

    def set_mask(self, mask):
        self.upload(self.out.meshlet_instance_visibility_mask, np.ascontiguousarray(mask, dtype=np.uint32))

    def mesh_instances(self, n):
        return self.download(self.out.mesh_instances, abi.MESH_INSTANCE_DT, n)

    def cull_meshlets_cmd(self):
        return self.download(self.out.cull_meshlets_cmd, abi.DISPATCH_CMD_DT, 1)

    def cull_triangles_cmd(self):
        return self.download(self.out.cull_triangles_cmd, abi.DISPATCH_CMD_DT, 1)

    def draw_cmd(self):
        return self.download(self.out.draw_cmd, abi.DRAW_CMD_DT, 1)

    def reordered_indices(self, n):
        return self.download(self.out.reordered_indices, np.uint32, n)

    def hiz_levels(self):
        o = self.out
        total = 0
        for l in range(o.hiz_levels):
            total = o.hiz_level_offset[l] + max(1, o.hiz_width >> l) * max(1, o.hiz_height >> l)
        flat = self.download(o.hiz, np.float32, total)
        return [flat[o.hiz_level_offset[l]: o.hiz_level_offset[l] + max(1, o.hiz_width >> l) * max(1, o.hiz_height >> l)]
                .reshape(max(1, o.hiz_height >> l), max(1, o.hiz_width >> l)) for l in range(o.hiz_levels)]

    def upload_hiz(self, flat):
        self.upload(self.out.hiz, np.ascontiguousarray(flat, dtype=np.float32))

    def view_bits(self, n):
        return self.download(self.out.view_visibility_bits, np.uint32, n)

    def view_counts(self):
        return self.download(self.out.view_visible_counts, np.uint32, abi.MAX_VIEWS)

    def raster_triangle_count(self):
        return int(self.download(self.out.raster_triangle_count, np.uint64, 1)[0])


class Renderer:
    """OxrRenderer wrapper: the host mirror of RendererInstance (HOST buffers in, HOST buffers out)."""

    def __init__(self, device, scene, alloc_reordered_indices=False, max_views=0):
        self.lib = load()
        hw, hh = scene.hiz_extent()
        info = abi.CreateInfo(max(1, scene.mesh_instance_count), max(1, scene.max_meshlet_instance_count), hw, hh,
                              int(alloc_reordered_indices), max_views)
        h = C.c_void_p()
        rc = self.lib.oxr_create(device, C.byref(info), scene.width, scene.height, C.byref(h))
        _check(rc, "oxr_create")
        self.h = h
        self.scene = scene
        from . import synth

        desc, self._keep = synth.scene_desc(scene)
        _check(self.lib.oxr_update(self.h, C.byref(desc)), "oxr_update")
        self.ctx = Context.from_handle(self.lib.oxr_context(self.h))

    def update_transforms(self, transforms, first=0):
        t = transforms if isinstance(transforms, np.ndarray) and transforms.flags.c_contiguous else np.ascontiguousarray(transforms)
        _check(self.lib.oxr_update_transforms(self.h, _ptr(t), first, len(t)), "oxr_update_transforms")

    def set_materials(self, materials, images=None, samplers=None):
        """oxr_set_materials (see Context.set_materials)"""
        t, keep = material_table(materials, images, samplers)
        _check(self.lib.oxr_set_materials(self.h, None if t is None else C.byref(t)), "oxr_set_materials")

    def overdraw(self, cam):
        """oxr_overdraw: the encode pass's fragment counter of the frame rendered last (uint32 [height, width])"""
        out = np.zeros((self.scene.height, self.scene.width), dtype=np.uint32)
        _check(self.lib.oxr_overdraw(self.h, _ptr(cam), _ptr(out)), "oxr_overdraw")
        return out

    def set_terrain(self, heightmap, patch_minmax=None, settings=None):
        """oxr_set_terrain: heightmap uint16 [res_y, res_x], patch_minmax float32 [patches, 2], settings an abi.TERRAIN_DRAW_SETTINGS_DT
        record; heightmap None removes the terrain"""
        if heightmap is None:
            _check(self.lib.oxr_set_terrain(self.h, None, 0, 0, None, None), "oxr_set_terrain")
            return
        hm = np.ascontiguousarray(heightmap, dtype=np.uint16)
        mm = np.ascontiguousarray(patch_minmax, dtype=np.float32)
        st = np.ascontiguousarray(settings)
        _check(self.lib.oxr_set_terrain(self.h, _ptr(hm), hm.shape[1], hm.shape[0], _ptr(mm), _ptr(st)), "oxr_set_terrain")

    def set_external_depth(self, depth):
        d = None if depth is None else np.ascontiguousarray(depth, dtype=np.float32)
        _check(self.lib.oxr_set_external_depth(self.h, _ptr(d)), "oxr_set_external_depth")

    def render(self, cam, occluder_depth=None, want_image=True, want_indices=True, out=None):
        """out: optional dict(vis32=, depth=, idx=) of preallocated (e.g. pinned) host arrays to fill."""
        sc = self.scene
        out = out or {}
        vis32 = out.get("vis32", np.empty((sc.height, sc.width), dtype=np.uint32) if want_image else None)
        depth = out.get("depth", np.empty((sc.height, sc.width), dtype=np.float32) if want_image else None)
        idx = out.get("idx", np.empty(max(1, sc.max_meshlet_instance_count), dtype=np.uint32) if want_indices else None)
        occ = occluder_depth
        if occ is not None and not (isinstance(occ, np.ndarray) and occ.dtype == np.float32 and occ.flags.c_contiguous):
            occ = np.ascontiguousarray(occ, dtype=np.float32)
        res = abi.FrameResult()
        _check(self.lib.oxr_render(self.h, _ptr(cam), _ptr(occ), _ptr(vis32), _ptr(depth), _ptr(idx),
                                   len(idx) if idx is not None else 0, C.byref(res)), "oxr_render")
        n = res.early + res.late
        return dict(vis32=vis32, depth=depth, visible=idx[:n] if idx is not None else None, total=res.total, early=res.early,
                    late=res.late, draw_index_count_early=res.draw_index_count_early,
                    draw_index_count_late=res.draw_index_count_late, raster_triangles=res.raster_triangles)

    def submit(self, cam, out):
        """Pipelined frame: out = dict(vis32=, depth=, idx=) of PINNED host arrays for this frame.  Returns a ticket."""
        t = C.c_int(-1)
        idx = out.get("idx")
        _check(self.lib.oxr_submit(self.h, _ptr(cam), _ptr(out.get("vis32")), _ptr(out.get("depth")), _ptr(idx),
                                   len(idx) if idx is not None else 0, C.byref(t)), "oxr_submit")
        return t.value

    def wait(self, ticket):
        res = abi.FrameResult()
        _check(self.lib.oxr_wait(self.h, ticket, C.byref(res)), "oxr_wait")
        return dict(total=res.total, early=res.early, late=res.late, raster_triangles=res.raster_triangles,
                    draw_index_count_early=res.draw_index_count_early, draw_index_count_late=res.draw_index_count_late)

    def vsm_update_pages(self, vsm, clipmaps, inv_projection_view, resolution, sun_moved=False, dirty_mesh_instances=(), hpb_levels=7):
        """oxr_vsm_update_pages: one VSM frame from the depth of the last rendered frame; returns vsm_pages()"""
        c = abi.VsmPageContext()
        vc = np.ascontiguousarray(vsm, dtype=abi.VSM_CONTEXT_DT)
        cm = np.zeros(abi.VSM_MAX_CLIPMAPS, dtype=abi.CLIPMAP_DT)
        cm[: len(clipmaps)] = clipmaps
        C.memmove(c.vsm, vc.ctypes.data, vc.nbytes)
        C.memmove(c.clipmaps, cm.ctypes.data, cm.nbytes)
        c.inv_projection_view[:] = [float(x) for x in np.asarray(inv_projection_view, dtype=np.float32).reshape(16)]
        c.resolution[:] = [float(x) for x in np.asarray(resolution, dtype=np.float32).reshape(2)]
        dirty = np.ascontiguousarray(dirty_mesh_instances, dtype=np.uint32)
        c.sun_moved, c.dirty_mesh_instance_count = int(bool(sun_moved)), len(dirty)
        c.dirty_mesh_instances = dirty.ctypes.data if len(dirty) else None
        c.hpb_levels = hpb_levels
        _check(self.lib.oxr_vsm_update_pages(self.h, C.byref(c)), "oxr_vsm_update_pages")
        return self.vsm_pages()

    def vsm_draw_shadows(self, coarse):
        """oxr_vsm_draw_shadows: the shadow casters of the last vsm_update_pages drawn into the renderer's atlas (coarse: the
        clipmap-9 camera, Shadowmaps.cpp:433-463)"""
        _check(self.lib.oxr_vsm_draw_shadows(self.h, _ptr(coarse)), "oxr_vsm_draw_shadows")

    def vsm_resolve_shadows(self, cam):
        """oxr_vsm_resolve_shadows: the shadow factor (float32 [height, width]) of the frame rendered last with `cam`, from the pages,
        clipmaps and atlas of the last vsm_update_pages / vsm_draw_shadows"""
        out = np.zeros((self.scene.height, self.scene.width), dtype=np.float32)
        _check(self.lib.oxr_vsm_resolve_shadows(self.h, _ptr(cam), _ptr(out)), "oxr_vsm_resolve_shadows")
        return out

    def decode_gbuffer(self, cam):
        """oxr_decode_gbuffer: the G-buffer of the frame rendered last with `cam` as four float32 [height, width, 4] arrays (albedo,
        normal, emissive, metallic_roughness_occlusion) from the table of the last set_materials"""
        out = [np.zeros((self.scene.height, self.scene.width, 4), dtype=np.float32) for _ in abi.GBUFFER_PLANES]
        _check(self.lib.oxr_decode_gbuffer(self.h, _ptr(cam), *[_ptr(o) for o in out]), "oxr_decode_gbuffer")
        return tuple(out)

    def generate_ambient_occlusion(self, cam, gtao_camera, settings):
        """oxr_generate_ambient_occlusion: the ambient occlusion (float32 [height, width]) of the frame rendered last with `cam`
        (gtao_camera: abi.GtaoCamera with that frame's projection, view and far clip; settings: abi.GtaoSettings)"""
        out = np.zeros((self.scene.height, self.scene.width), dtype=np.float32)
        _check(self.lib.oxr_generate_ambient_occlusion(self.h, _ptr(cam), C.byref(gtao_camera), C.byref(settings), _ptr(out)),
               "oxr_generate_ambient_occlusion")
        return out

    def contact_shadows(self, contact_camera, settings):
        """oxr_contact_shadows: 1 - the contact shadow (float32 [height, width]) over the depth of the frame rendered last
        (contact_camera: abi.ContactShadowCamera of that frame's camera; settings: abi.ContactShadowSettings)"""
        out = np.zeros((self.scene.height, self.scene.width), dtype=np.float32)
        _check(self.lib.oxr_contact_shadows(self.h, C.byref(contact_camera), C.byref(settings), _ptr(out)), "oxr_contact_shadows")
        return out

    def atmosphere_luts(self, atmosphere, camera, sun_direction, sun_intensity):
        """oxr_atmosphere_luts: (transmittance [64, 256, 4], sky view [192, 312, 4], aerial perspective [32, 32, 32, 4]) as float16
        arrays.  The transmittance LUT is the renderer's bake with the default record; the per-frame LUTs use `atmosphere` (abi.Atmosphere,
        its sizes replaced by the renderer's), camera (abi.PbrCamera) and the sun"""
        t = np.zeros((64, 256, 4), np.float16)
        sv = np.zeros((192, 312, 4), np.float16)
        ap = np.zeros((32, 32, 32, 4), np.float16)
        sun = (C.c_float * 3)(*[float(np.float32(v)) for v in sun_direction])
        _check(self.lib.oxr_atmosphere_luts(self.h, C.byref(atmosphere), C.byref(camera), sun, float(np.float32(sun_intensity)), _ptr(t),
                                            _ptr(sv), _ptr(ap)), "oxr_atmosphere_luts")
        return t, sv, ap

    def atmosphere_sky_ibl(self, atmosphere, camera, sun_direction, sun_intensity):
        """oxr_atmosphere_sky_ibl: the renderer's sky IBL cube after this call, float16 [6, 32, 32, 4].  The per-frame LUTs are made as
        atmosphere_luts makes them; the cube persists across calls (zeroed at the first) and the call's frame_index is the number of
        earlier calls on this renderer"""
        cube = np.zeros(abi.SKY_IBL_CUBE_SHAPE, np.float16)
        sun = (C.c_float * 3)(*[float(np.float32(v)) for v in sun_direction])
        _check(self.lib.oxr_atmosphere_sky_ibl(self.h, C.byref(atmosphere), C.byref(camera), sun, float(np.float32(sun_intensity)), _ptr(cube)),
               "oxr_atmosphere_sky_ibl")
        return cube

    def apply_pbr_atmosphere(self, cam, settings, atmosphere, lights=None, cast_shadows=False, gtao_camera=None, gtao_settings=None,
                             pbr_camera=None, contact_camera=None, contact_settings=None):
        """oxr_apply_pbr_atmosphere: the per-frame LUTs and the cube update (as atmosphere_sky_ibl, advancing its counter), the chain of
        apply_pbr, then the atmospheric PBR apply with the record (abi.Atmosphere); settings must carry SCENE_HAS_ATMOSPHERE and
        SCENE_HAS_DIRECTIONAL_LIGHT.  Returns float32 [height, width, 4]"""
        from oxylus_b200 import synth

        n = 0 if lights is None else len(lights)
        settings = abi.PbrSettings.from_buffer_copy(settings)
        settings.light_count = n
        pc = pbr_camera if pbr_camera is not None else synth.pbr_camera(cam)
        out = np.zeros((self.scene.height, self.scene.width, 4), dtype=np.float32)
        opt = lambda v: C.byref(v) if v is not None else None
        _check(self.lib.oxr_apply_pbr_atmosphere(self.h, _ptr(cam), C.byref(pc), C.byref(settings), C.byref(atmosphere),
                                                 C.cast(lights, C.c_void_p) if n else None, int(bool(cast_shadows)), opt(gtao_camera),
                                                 opt(gtao_settings), opt(contact_camera), opt(contact_settings), _ptr(out)),
               "oxr_apply_pbr_atmosphere")
        return out

    def eye_adaptation(self, settings, delta_time):
        """oxr_eye_adaptation: eye adaptation on the post chain's source (the lit plane of the last apply_pbr* call, or the FXAA plane
        after fxaa), into the renderer's persistent exposure record ((1, 1) at the first call); returns the record after the call
        (abi.Exposure)"""
        rec = abi.Exposure()
        _check(self.lib.oxr_eye_adaptation(self.h, C.byref(settings), float(np.float32(delta_time)), C.byref(rec)), "oxr_eye_adaptation")
        return rec

    def bloom(self, settings):
        """oxr_bloom: the bloom image (upsampled level 0, float32 [height // 2, width // 2, 4]) of the post chain's source, with the
        renderer's exposure record under SCENE_HAS_EYE_ADAPTATION"""
        out = np.zeros((self.scene.height // 2, self.scene.width // 2, 4), dtype=np.float32)
        _check(self.lib.oxr_bloom(self.h, C.byref(settings), _ptr(out)), "oxr_bloom")
        return out

    def tonemap(self, settings):
        """oxr_tonemap: the tonemapped frame (float32 [height, width, 4]) of the post chain's source, with the renderer's exposure
        record under SCENE_HAS_EYE_ADAPTATION and its bloom image under SCENE_HAS_BLOOM"""
        out = np.zeros((self.scene.height, self.scene.width, 4), dtype=np.float32)
        _check(self.lib.oxr_tonemap(self.h, C.byref(settings), _ptr(out)), "oxr_tonemap")
        return out

    def fxaa(self):
        """oxr_fxaa: FXAA (float32 [height, width, 4]) of the lit plane of the last apply_pbr* call; the FXAA plane then becomes the
        source of eye_adaptation, bloom and tonemap until the next apply_pbr*"""
        out = np.zeros((self.scene.height, self.scene.width, 4), dtype=np.float32)
        _check(self.lib.oxr_fxaa(self.h, _ptr(out)), "oxr_fxaa")
        return out

    def apply_pbr(self, cam, settings, lights=None, cast_shadows=False, gtao_camera=None, gtao_settings=None, pbr_camera=None,
                  contact_camera=None, contact_settings=None):
        """oxr_apply_pbr: the lit frame (float32 [height, width, 4]) of the frame rendered last with `cam`: G-buffer decode, the shadow
        resolve when cast_shadows (state of the last vsm_update_pages / vsm_draw_shadows), GTAO under SCENE_HAS_GTAO (gtao_camera,
        gtao_settings), then PBR apply with settings (abi.PbrSettings; light_count is set from `lights`, an abi.Light array).
        pbr_camera defaults to synth.pbr_camera(cam).  Given contact_camera or contact_settings (abi.ContactShadowCamera /
        abi.ContactShadowSettings), it calls oxr_apply_pbr_with_contact_shadows, which runs the contact-shadow pass under
        SCENE_HAS_CONTACT_SHADOWS"""
        from oxylus_b200 import synth

        n = 0 if lights is None else len(lights)
        settings = abi.PbrSettings.from_buffer_copy(settings)
        settings.light_count = n
        pc = pbr_camera if pbr_camera is not None else synth.pbr_camera(cam)
        out = np.zeros((self.scene.height, self.scene.width, 4), dtype=np.float32)
        args = [self.h, _ptr(cam), C.byref(pc), C.byref(settings), C.cast(lights, C.c_void_p) if n else None, int(bool(cast_shadows)),
                C.byref(gtao_camera) if gtao_camera is not None else None, C.byref(gtao_settings) if gtao_settings is not None else None]
        if contact_camera is None and contact_settings is None:
            _check(self.lib.oxr_apply_pbr(*args, _ptr(out)), "oxr_apply_pbr")
        else:
            _check(self.lib.oxr_apply_pbr_with_contact_shadows(*args, C.byref(contact_camera) if contact_camera is not None else None,
                                                               C.byref(contact_settings) if contact_settings is not None else None, _ptr(out)),
                   "oxr_apply_pbr_with_contact_shadows")
        return out

    def vsm_pages(self):
        """oxr_vsm_pages: abi.VsmPages of device pointers and sizes"""
        out = abi.VsmPages()
        _check(self.lib.oxr_vsm_pages(self.h, C.byref(out)), "oxr_vsm_pages")
        return out

    def close(self):
        if getattr(self, "h", None):
            self.lib.oxr_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
