"""numpy / ctypes mirrors of include/oxcull.h (which mirrors Oxylus/include/Scene/SceneGPU.hpp).

Sizes are asserted against the reference's scalar-layout sizes (SURVEY.md §8): MeshletBounds 16 B
(SceneGPU.hpp:84-90), MeshInstance 20 B (:111-117), Meshlet 16 B (:119-124), MeshLOD 64 B (:126-140),
Mesh 64 B (:142-152), CullCamera 96 B (:222-229).
"""
import ctypes as C

import numpy as np

TRANSFORM_DT = np.dtype([("world", "<f4", (16,))])
MESHLET_BOUNDS_DT = np.dtype(
    [
        ("aabb_center", "<u2", (3,)),
        ("cone_axis_xy", "i1", (2,)),
        ("aabb_extent", "<u2", (3,)),
        ("cone_axis_z", "i1"),
        ("cone_cutoff", "i1"),
    ]
)
MESH_BOUNDS_DT = np.dtype([("aabb_center", "<f4", (3,)), ("aabb_extent", "<f4", (3,))])
VISIBILITY_DT = np.dtype([("total", "<u4"), ("early", "<u4"), ("late", "<u4")])
MESHLET_INSTANCE_DT = np.dtype([("mesh_instance_index", "<u4"), ("meshlet_index", "<u4")])
MESH_INSTANCE_DT = np.dtype(
    [
        ("mesh_index", "<u4"),
        ("lod_index", "<u4"),
        ("material_index", "<u4"),
        ("transform_index", "<u4"),
        ("meshlet_instance_visibility_offset", "<u4"),
    ]
)
MESHLET_DT = np.dtype(
    [
        ("indirect_vertex_index_offset", "<u4"),
        ("local_triangle_index_offset", "<u4"),
        ("vertex_count", "<u4"),
        ("triangle_count", "<u4"),
    ]
)
MESH_LOD_DT = np.dtype(
    [
        ("indices", "<u8"),
        ("meshlets", "<u8"),
        ("meshlet_bounds", "<u8"),
        ("local_triangle_indices", "<u8"),
        ("indirect_vertex_indices", "<u8"),
        ("indices_count", "<u4"),
        ("meshlet_count", "<u4"),
        ("meshlet_bounds_count", "<u4"),
        ("local_triangle_indices_count", "<u4"),
        ("indirect_vertex_indices_count", "<u4"),
        ("error", "<f4"),
    ]
)
MESH_DT = np.dtype(
    [
        ("vertex_positions", "<u8"),
        ("vertex_normals", "<u8"),
        ("texture_coords", "<u8"),
        ("vertex_count", "<u4"),
        ("lod_count", "<u4"),
        ("lods", "<u8"),
        ("bounds", MESH_BOUNDS_DT),
    ]
)
CULL_CAMERA_DT = np.dtype(
    [
        ("projection_view", "<f4", (16,)),
        ("position", "<f4", (3,)),
        ("acceptable_lod_error", "<f4"),
        ("resolution", "<f4", (2,)),
        ("near_clip", "<f4"),
        ("mesh_instance_count", "<u4"),
    ]
)
DISPATCH_CMD_DT = np.dtype([("x", "<u4"), ("y", "<u4"), ("z", "<u4")])
DRAW_CMD_DT = np.dtype(
    [
        ("index_count", "<u4"),
        ("instance_count", "<u4"),
        ("first_index", "<u4"),
        ("vertex_offset", "<i4"),
        ("first_instance", "<u4"),
    ]
)

TERRAIN_DT = np.dtype([("world_min", "<f4", (2,)), ("world_size", "<f4", (2,)), ("patch_count", "<u4", (2,)),
                       ("base_height", "<f4"), ("height_scale", "<f4")])
DRAW_INDIRECT_DT = np.dtype([("vertex_count", "<u4"), ("instance_count", "<u4"), ("first_vertex", "<u4"), ("first_instance", "<u4")])
CLIPMAP_DT = np.dtype([("projection_view_mat", "<f4", (16,)), ("page_offset", "<i4", (2,)), ("z_near", "<f4")])
assert CLIPMAP_DT.itemsize == 76
assert TERRAIN_DT.itemsize == 32 and DRAW_INDIRECT_DT.itemsize == 16
# OxcTerrainDrawSettings: TerrainData's fields the terrain draw reads and Camera::fov (degrees)
TERRAIN_DRAW_SETTINGS_DT = np.dtype([("terrain", TERRAIN_DT), ("inv_world_size", "<f4", (2,)), ("target_edge_pixels", "<f4"),
                                     ("max_tessellation", "<f4"), ("fov", "<f4")])
assert TERRAIN_DRAW_SETTINGS_DT.itemsize == 52


def terrain_draw_settings(terrain, target_edge_pixels=16.0, max_tessellation=64.0, fov=60.0):
    """OxcTerrainDrawSettings of a TERRAIN_DT record with the reference's defaults (Terrain.hpp: 16 px, 64; Camera fov 60 degrees);
    inv_world_size = 1 / world_size in binary32, as Passes/Terrain.cpp:20 forms it"""
    s = np.zeros(1, dtype=TERRAIN_DRAW_SETTINGS_DT)
    s["terrain"] = np.asarray(terrain, dtype=TERRAIN_DT).reshape(1)
    size = s["terrain"]["world_size"][0].astype(np.float32)
    with np.errstate(divide="ignore"):
        s["inv_world_size"][0] = np.float32(1.0) / size
    s["target_edge_pixels"], s["max_tessellation"], s["fov"] = target_edge_pixels, max_tessellation, fov
    return s
assert TRANSFORM_DT.itemsize == 64
assert MESHLET_BOUNDS_DT.itemsize == 16
assert VISIBILITY_DT.itemsize == 12
assert MESHLET_INSTANCE_DT.itemsize == 8
assert MESH_INSTANCE_DT.itemsize == 20
assert MESHLET_DT.itemsize == 16
assert MESH_LOD_DT.itemsize == 64
assert MESH_DT.itemsize == 64
assert CULL_CAMERA_DT.itemsize == 96
assert DISPATCH_CMD_DT.itemsize == 12
assert DRAW_CMD_DT.itemsize == 20

# CullFlag — SceneGPU.hpp:345-353
CULL_NONE = 0
CULL_TEST_FRUSTUM = 1 << 0
CULL_SELECT_LOD = 1 << 1
CULL_TEST_OCCLUSION = 1 << 2
CULL_LATE_PASS = 1 << 3
CULL_TEST_ALL = CULL_TEST_FRUSTUM | CULL_SELECT_LOD | CULL_TEST_OCCLUSION

HIZ_MAX_LEVELS = 13
MAX_VIEWS = 16
VIS_PRIMITIVE_BITS = 8
VIS_WIDE_PRIMITIVE_BITS = 6
VIS_CLEAR = 0xFFFFFFFF
STATUS_MESHLET_OVERFLOW, STATUS_BAD_GEOMETRY, STATUS_SURVIVOR_OVERFLOW, STATUS_ID_OVERFLOW, STATUS_PEER_TIMEOUT = 1, 2, 4, 8, 16
STATUS_CLIP_OVERFLOW = 32
STATUS_BAD_MATERIAL = 64

# Material — SceneGPU.hpp:67-82 / scene.slang:51-66 (56 B); MaterialFlag scene.slang:34-49
MATERIAL_DT = np.dtype(
    [
        ("albedo_color", "<u2", (4,)),
        ("emissive_color", "<u2", (3,)),
        ("roughness_factor", "<u2"),
        ("metallic_factor", "<u2"),
        ("alpha_cutoff", "<u2"),
        ("flags", "<u4"),
        ("sampler_index", "<u4"),
        ("albedo_image_index", "<u4"),
        ("normal_image_index", "<u4"),
        ("emissive_image_index", "<u4"),
        ("metallic_roughness_image_index", "<u4"),
        ("occlusion_image_index", "<u4"),
        ("uv_size", "<u2", (2,)),
        ("uv_offset", "<u2", (2,)),
    ]
)
assert MATERIAL_DT.itemsize == 56
MATERIAL_HAS_ALBEDO_IMAGE, MATERIAL_ALPHA_MASK = 1, 1 << 8
IMAGE_RGBA8_UNORM, IMAGE_R8_UNORM, IMAGE_RGBA8_SRGB, IMAGE_RG8_UNORM = 0, 1, 2, 3
MATERIAL_HAS_NORMAL_IMAGE, MATERIAL_HAS_EMISSIVE_IMAGE, MATERIAL_HAS_METALLIC_ROUGHNESS_IMAGE, MATERIAL_HAS_OCCLUSION_IMAGE = 1 << 1, 1 << 2, 1 << 3, 1 << 4
MATERIAL_NORMAL_TWO_COMPONENT, MATERIAL_NORMAL_FLIP_Y = 1 << 5, 1 << 6
FILTER_LINEAR, FILTER_NEAREST = 0, 1
ADDRESS_REPEAT, ADDRESS_CLAMP_TO_EDGE, ADDRESS_MIRRORED_REPEAT = 0, 1, 2
MIPMAP_LINEAR, MIPMAP_NEAREST = 0, 1
ALPHA_IMAGE_DT = np.dtype([("texels", "<u8"), ("width", "<u4"), ("height", "<u4"), ("format", "<u4"), ("level_count", "<u4")])
SAMPLER_DT = np.dtype([("mag_filter", "<u4"), ("min_filter", "<u4"), ("mipmap_mode", "<u4"), ("address_u", "<u4"), ("address_v", "<u4")])


def sampler(mag=FILTER_LINEAR, min=FILTER_LINEAR, mip=MIPMAP_LINEAR, u=ADDRESS_REPEAT, v=ADDRESS_REPEAT):  # noqa: A002
    """one SAMPLER_DT record (defaults = the reference's default sampler, Texture.hpp:38-45)"""
    return (mag, min, mip, u, v)


class MaterialTable(C.Structure):
    """OxcMaterialTable"""

    _fields_ = [
        ("materials", C.c_void_p),
        ("material_count", C.c_uint32),
        ("images", C.c_void_p),
        ("image_count", C.c_uint32),
        ("samplers", C.c_void_p),
        ("sampler_count", C.c_uint32),
    ]


# VSMPageState — Shaders/rmvsm.slang:16-28 ([Flags] enum)
VSM_PAGE_VISIBLE = 1
VSM_PAGE_DIRTY = 2
VSM_PAGE_BACKED = 4
VSM_PAGE_INVALIDATED = 8
VSM_PAGE_ALLOCATION_FAILED = 16
VSM_MAX_CLIPMAPS = 10


class SceneDesc(C.Structure):
    """OxcSceneDesc"""

    _fields_ = [
        ("meshes", C.c_void_p),
        ("mesh_count", C.c_uint32),
        ("mesh_instances", C.c_void_p),
        ("mesh_instance_count", C.c_uint32),
        ("transforms", C.c_void_p),
        ("transform_count", C.c_uint32),
        ("blob", C.c_void_p),
        ("blob_size", C.c_uint64),
    ]


class CreateInfo(C.Structure):
    """OxcCreateInfo"""

    _fields_ = [
        ("max_mesh_instances", C.c_uint32),
        ("max_meshlet_instances", C.c_uint32),
        ("hiz_width", C.c_uint32),
        ("hiz_height", C.c_uint32),
        ("alloc_reordered_indices", C.c_uint32),
        ("max_views", C.c_uint32),
        ("max_mask_bits", C.c_uint32),
        ("wide_ids", C.c_uint32),
    ]


class Outputs(C.Structure):
    """OxcOutputs"""

    _fields_ = [
        ("visibility", C.c_void_p),
        ("cull_meshlets_cmd", C.c_void_p),
        ("cull_triangles_cmd", C.c_void_p),
        ("draw_cmd", C.c_void_p),
        ("meshlet_instances", C.c_void_p),
        ("visible_meshlet_instances_indices", C.c_void_p),
        ("meshlet_instance_visibility_mask", C.c_void_p),
        ("reordered_indices", C.c_void_p),
        ("mesh_instances", C.c_void_p),
        ("hiz", C.c_void_p),
        ("hiz_level_offset", C.c_uint32 * HIZ_MAX_LEVELS),
        ("hiz_levels", C.c_uint32),
        ("hiz_width", C.c_uint32),
        ("hiz_height", C.c_uint32),
        ("visibility_mask_words", C.c_uint32),
        ("view_visibility_bits", C.c_void_p),
        ("view_visible_counts", C.c_void_p),
        ("raster_triangle_count", C.c_void_p),
        ("status_flags", C.c_void_p),
        ("vis_primitive_bits", C.c_uint32),
    ]


VSM_CONTEXT_DT = np.dtype([("page_size", "<i4"), ("page_table_size", "<i4"), ("physical_page_table_size", "<i4"), ("curr_clipmap_index", "<i4"),
                           ("clipmap_count", "<i4"), ("depth_extent", "<i4", (2,)), ("first_clipmap_width", "<f4"),
                           ("clipmap_selection_bias", "<f4"), ("virtual_extent", "<f4"), ("z_length", "<f4"),
                           ("directional_light_dir", "<f4", (3,))])
assert VSM_CONTEXT_DT.itemsize == 56
# rmvsm.slang:228-236 VSMPageAllocator (OxcVsmAllocator): counters, then device pointers of the three lists
VSM_ALLOCATOR_DT = np.dtype([("active_request_count", "<u4"), ("dirty_physical_page_count", "<u4"), ("free_page_count", "<u4"),
                             ("alloc_cursor", "<u4"), ("requests", "<u8"), ("dirty_physical_page_coords", "<u8"), ("free_page_list", "<u8")])
assert VSM_ALLOCATOR_DT.itemsize == 40


class VsmPageContext(C.Structure):
    """OxrVsmPageContext (oxr_vsm_update_pages)"""

    _fields_ = [
        ("vsm", C.c_uint8 * VSM_CONTEXT_DT.itemsize),
        ("clipmaps", C.c_uint8 * (CLIPMAP_DT.itemsize * VSM_MAX_CLIPMAPS)),
        ("inv_projection_view", C.c_float * 16),
        ("resolution", C.c_float * 2),
        ("sun_moved", C.c_uint32),
        ("dirty_mesh_instance_count", C.c_uint32),
        ("dirty_mesh_instances", C.c_void_p),
        ("hpb_levels", C.c_uint32),
    ]


class VsmPages(C.Structure):
    """OxrVsmPages: device pointers of the renderer's virtual shadow map state"""

    _fields_ = [
        ("page_tables", C.c_void_p), ("hpb", C.c_void_p), ("page_occupancy", C.c_void_p), ("requests", C.c_void_p), ("allocator", C.c_void_p),
        ("free_page_list", C.c_void_p), ("dirty_physical_page_coords", C.c_void_p), ("clipmap_dirty_flags", C.c_void_p),
        ("physical_atlas", C.c_void_p),
        ("page_table_size", C.c_uint32), ("clipmap_count", C.c_uint32), ("physical_page_count", C.c_uint32), ("physical_atlas_size", C.c_uint32),
        ("hpb_levels", C.c_uint32), ("request_capacity", C.c_uint32),
    ]


assert C.sizeof(VsmPageContext) == 912 and C.sizeof(VsmPages) == 96


class MgpuInfo(C.Structure):
    """OxcMgpuInfo"""

    _fields_ = [
        ("active", C.c_uint32), ("rank", C.c_uint32), ("world", C.c_uint32), ("survivor_capacity", C.c_uint32),
        ("hiz_over_peer_memory", C.c_uint32),
        ("gathered_counts", C.c_void_p * 2),
        ("gathered_ids", C.c_void_p * 2),
    ]


MGPU_ID_BYTES = 128


class DecodeTargets(C.Structure):
    """OxcDecodeTargets: device pointers of the five float4 planes (any may be NULL)"""

    _fields_ = [("lambda_", C.c_void_p), ("ddx", C.c_void_p), ("ddy", C.c_void_p), ("uv_normal", C.c_void_p), ("uv_grad", C.c_void_p)]


class GBufferTargets(C.Structure):
    """OxcGBufferTargets: device pointers of the four float4 G-buffer planes (any may be NULL)"""

    _fields_ = [("albedo", C.c_void_p), ("normal", C.c_void_p), ("emissive", C.c_void_p), ("metallic_roughness_occlusion", C.c_void_p)]


assert C.sizeof(GBufferTargets) == 32
GBUFFER_PLANES = ("albedo", "normal", "emissive", "metallic_roughness_occlusion")


GTAO_MAX_SLICES = 16
GTAO_MAX_SAMPLES_PER_SIDE = 8
GTAO_LEVELS = 5


class GtaoSettings(C.Structure):
    """OxcGtaoSettings (SceneGPU.hpp:286-293 VBGTAOSettings)"""

    _fields_ = [("thickness", C.c_float), ("slice_count", C.c_uint32), ("samples_per_slice_side", C.c_uint32), ("effect_radius", C.c_float),
                ("noise_index", C.c_uint32), ("final_power", C.c_float)]


class GtaoCamera(C.Structure):
    """OxcGtaoCamera: Camera::projection and Camera::view (column-major) and far_clip"""

    _fields_ = [("projection", C.c_float * 16), ("view", C.c_float * 16), ("far_clip", C.c_float)]


class GtaoTargets(C.Structure):
    """OxcGtaoTargets: device pointers of the depth mips, edges (u32), noisy occlusion (binary16) and final occlusion planes"""

    _fields_ = [("depth_mips", C.c_void_p), ("edges", C.c_void_p), ("noisy_occlusion", C.c_void_p), ("ambient_occlusion", C.c_void_p)]


assert C.sizeof(GtaoSettings) == 24 and C.sizeof(GtaoCamera) == 132 and C.sizeof(GtaoTargets) == 32

# update_vbgtao_info's quality presets (PBR.cpp:149-170): (slice_count, samples_per_slice_side); the cvar default is 3, "ultra"
GTAO_PRESETS = {0: (1, 2), 1: (2, 2), 2: (3, 3), 3: (9, 3)}


def gtao_settings(quality_level=3, thickness=0.25, radius=0.5, final_power=1.2, noise_index=0):
    """GtaoSettings as update_vbgtao_info fills them from the cvars (RendererCVar.cpp:36-41 defaults); noise_index stays 0 until
    there is TAA (PBR.cpp:172-174)"""
    slices, samples = GTAO_PRESETS[int(quality_level)]
    return GtaoSettings(thickness, slices, samples, radius, noise_index, final_power)


def gtao_camera(projection, view, far_clip):
    c = GtaoCamera()
    c.projection[:] = [float(x) for x in np.asarray(projection, dtype=np.float32).reshape(16)]
    c.view[:] = [float(x) for x in np.asarray(view, dtype=np.float32).reshape(16)]
    c.far_clip = float(np.float32(far_clip))
    return c


def gtao_mip_layout(width, height):
    """[(offset, width, height)] of mips 0..4 in the packed depth_mips plane, and the total texel count"""
    out, off = [], 0
    for k in range(GTAO_LEVELS):
        w, h = max(1, width >> k), max(1, height >> k)
        out.append((off, w, h))
        off += w * h
    return out, off


MAX_LIGHTS = 256  # GPU::MAX_LIGHTS
# SceneFlags (SceneGPU.hpp:253-267)
SCENE_HAS_DIRECTIONAL_LIGHT = 1 << 0
SCENE_HAS_ATMOSPHERE = 1 << 1
SCENE_HAS_EYE_ADAPTATION = 1 << 2
SCENE_HAS_BLOOM = 1 << 3
SCENE_HAS_FXAA = 1 << 4
SCENE_HAS_GTAO = 1 << 5
SCENE_HAS_FILM_GRAIN = 1 << 6
SCENE_HAS_CHROMATIC_ABERRATION = 1 << 7
SCENE_HAS_VIGNETTE = 1 << 8
SCENE_HAS_CONTACT_SHADOWS = 1 << 9
SCENE_HAS_SKY = 1 << 10
SCENE_TRANSPARENT_BACKGROUND = 1 << 11
# LightKind
LIGHT_DIRECTIONAL, LIGHT_POINT, LIGHT_SPOT = 0, 1, 2


class Light(C.Structure):
    """OxcLight (GPU::Light, SceneGPU.hpp:241-251)"""

    _fields_ = [("position", C.c_float * 3), ("intensity", C.c_float), ("color", C.c_float * 3), ("range", C.c_float), ("direction", C.c_float * 3),
                ("inner_cone_angle", C.c_float), ("outer_cone_angle", C.c_float), ("kind", C.c_uint32), ("pad", C.c_uint32 * 2)]


class PbrSettings(C.Structure):
    """OxcPbrSettings: scene flags, sun direction and intensity, base ambient colour, the Sky record and the light count"""

    _fields_ = [("scene_flags", C.c_uint32), ("sun_direction", C.c_float * 3), ("sun_intensity", C.c_float), ("base_ambient_color", C.c_float * 3),
                ("sky_solid_color", C.c_float * 4), ("sky_ambient_color", C.c_float * 3), ("sky_has_texture", C.c_uint32), ("light_count", C.c_uint32)]


class PbrCamera(C.Structure):
    """OxcPbrCamera: Camera::inv_projection_view (column-major) and the camera position"""

    _fields_ = [("inv_projection_view", C.c_float * 16), ("position", C.c_float * 3)]


class PbrInputs(C.Structure):
    """OxcPbrInputs: device pointers of depth, albedo, normal, emissive, metallic/roughness/occlusion, ambient occlusion, shadow and contact
    shadow"""

    _fields_ = [(k, C.c_void_p) for k in ("depth", "albedo", "normal", "emissive", "metallic_roughness_occlusion", "ambient_occlusion", "shadow",
                                          "contact_shadow")]


assert C.sizeof(Light) == 64 and C.sizeof(PbrSettings) == 68 and C.sizeof(PbrCamera) == 76 and C.sizeof(PbrInputs) == 64
PBR_INPUTS = tuple(k for k, _ in PbrInputs._fields_)


def pbr_settings(scene_flags=SCENE_HAS_DIRECTIONAL_LIGHT | SCENE_HAS_GTAO, sun_direction=(0.3, 0.8, 0.52), sun_intensity=10.0, base_ambient=0.03,
                 sky_solid_color=(0.0, 0.0, 0.0, 1.0), sky_ambient_color=(0.0, 0.0, 0.0), sky_has_texture=False, light_count=0):
    """PbrSettings as apply_pbr fills them (PBR.cpp:436-486: base ambient 0.03, DirectionalLight::intensity 10 by default)"""
    s = PbrSettings()
    s.scene_flags = int(scene_flags)
    s.sun_direction[:] = [float(np.float32(v)) for v in sun_direction]
    s.sun_intensity = float(sun_intensity)
    s.base_ambient_color[:] = [float(np.float32(base_ambient))] * 3 if np.isscalar(base_ambient) else [float(v) for v in base_ambient]
    s.sky_solid_color[:] = [float(v) for v in sky_solid_color]
    s.sky_ambient_color[:] = [float(v) for v in sky_ambient_color]
    s.sky_has_texture = int(bool(sky_has_texture))
    s.light_count = int(light_count)
    return s


def pbr_camera(inv_projection_view, position):
    c = PbrCamera()
    c.inv_projection_view[:] = [float(x) for x in np.asarray(inv_projection_view, dtype=np.float32).reshape(16)]
    c.position[:] = [float(x) for x in np.asarray(position, dtype=np.float32).reshape(3)]
    return c


CONTACT_SHADOW_MAX_STEPS = 64  # the editor's range of the steps cvar (ViewportPanel.cpp:748)


class ContactShadowCamera(C.Structure):
    """OxcContactShadowCamera: Camera::inv_projection_view, view and projection (column-major) and near_clip"""

    _fields_ = [("inv_projection_view", C.c_float * 16), ("view", C.c_float * 16), ("projection", C.c_float * 16), ("near_clip", C.c_float)]


class ContactShadowSettings(C.Structure):
    """OxcContactShadowSettings: the contact_shadows pass's push constants (sun direction, steps, thickness, length)"""

    _fields_ = [("sun_direction", C.c_float * 3), ("steps", C.c_uint32), ("thickness", C.c_float), ("length", C.c_float)]


assert C.sizeof(ContactShadowCamera) == 196 and C.sizeof(ContactShadowSettings) == 24


def contact_shadow_camera(inv_projection_view, view, projection, near_clip):
    c = ContactShadowCamera()
    for name, m in (("inv_projection_view", inv_projection_view), ("view", view), ("projection", projection)):
        getattr(c, name)[:] = [float(x) for x in np.asarray(m, dtype=np.float32).reshape(16)]
    c.near_clip = float(np.float32(near_clip))
    return c


def contact_shadow_settings(sun_direction=(0.3, 0.8, 0.52), steps=8, thickness=0.1, length=0.01):
    """ContactShadowSettings with the reference's cvar defaults (RendererCVar.cpp:30-34: 8 steps, thickness 0.1, length 0.01)"""
    s = ContactShadowSettings()
    s.sun_direction[:] = [float(np.float32(v)) for v in sun_direction]
    s.steps, s.thickness, s.length = int(steps), float(np.float32(thickness)), float(np.float32(length))
    return s


ATMOSPHERE_MAX_LUT_SIZE = 4096
ATMOSPHERE_MAX_AERIAL_DEPTH = 256


class Atmosphere(C.Structure):
    """OxcAtmosphere (GPU::Atmosphere, SceneGPU.hpp:158-181, scalar layout)"""

    _fields_ = [("rayleigh_scatter", C.c_float * 3), ("rayleigh_density", C.c_float), ("mie_scatter", C.c_float * 3), ("mie_density", C.c_float),
                ("mie_extinction", C.c_float), ("mie_asymmetry", C.c_float), ("ozone_absorption", C.c_float * 3), ("ozone_height", C.c_float),
                ("ozone_thickness", C.c_float), ("terrain_albedo", C.c_float * 3), ("planet_radius", C.c_float), ("atmos_radius", C.c_float),
                ("aerial_perspective_start_km", C.c_float), ("aerial_perspective_exposure", C.c_float),
                ("transmittance_lut_size", C.c_uint32 * 3), ("sky_view_lut_size", C.c_uint32 * 3), ("multiscattering_lut_size", C.c_uint32 * 3),
                ("aerial_perspective_lut_size", C.c_uint32 * 3)]


assert C.sizeof(Atmosphere) == 136

# GPU::Atmosphere{} (SceneGPU.hpp:158-181) and the reference's LUT extents (RendererInstance.hpp: transmittance 256 x 64, sky view
# 312 x 192, multiple scattering 32 x 32, aerial perspective 32 x 32 x 32)
ATMOSPHERE_DEFAULTS = dict(rayleigh_scatter=(0.005802, 0.013558, 0.033100), rayleigh_density=8.0, mie_scatter=(0.003996, 0.003996, 0.003996),
                           mie_density=1.2, mie_extinction=0.004440, mie_asymmetry=3.6, ozone_absorption=(0.000650, 0.001881, 0.000085),
                           ozone_height=25.0, ozone_thickness=15.0, terrain_albedo=(0.3, 0.3, 0.3), planet_radius=6360.0, atmos_radius=6460.0,
                           aerial_perspective_start_km=8.0, aerial_perspective_exposure=1.0, transmittance_lut_size=(256, 64, 1),
                           sky_view_lut_size=(312, 192, 1), multiscattering_lut_size=(32, 32, 1), aerial_perspective_lut_size=(32, 32, 32))


class PbrSky(C.Structure):
    """OxcPbrSky: the atmospheric PBR apply's sky planes (device pointers, binary16 RGBA, 8-byte aligned)"""
    _fields_ = [("transmittance", C.c_void_p), ("sky_view", C.c_void_p), ("aerial_perspective", C.c_void_p), ("sky_cube", C.c_void_p)]


PBR_SKY_PLANES = ("transmittance", "sky_view", "aerial_perspective", "sky_cube")
assert C.sizeof(PbrSky) == 32


# the sky IBL cube (oxc_atmosphere_sky_ibl): 6 faces x 32 x 32 binary16 RGBA texels, 64 sky-view samples per texel per call
SKY_IBL_CUBE_RES = 32
SKY_IBL_SAMPLES = 64
SKY_IBL_CUBE_SHAPE = (6, SKY_IBL_CUBE_RES, SKY_IBL_CUBE_RES, 4)
SKY_IBL_CUBE_BYTES = 6 * SKY_IBL_CUBE_RES * SKY_IBL_CUBE_RES * 8
# the sun_ambient_strength the reference passes (Passes/PBR.cpp:56)
SKY_IBL_SUN_AMBIENT_STRENGTH = 0.15


class EyeAdaptationSettings(C.Structure):
    """OxcEyeAdaptationSettings (GPU::EyeAdaptationSettings)"""
    _fields_ = [("min_exposure", C.c_float), ("max_exposure", C.c_float), ("adaptation_speed", C.c_float), ("ev100_bias", C.c_float)]


class Exposure(C.Structure):
    """OxcExposure: the persistent exposure record (HistogramLuminance), 8 B"""
    _fields_ = [("adapted_luminance", C.c_float), ("exposure", C.c_float)]


class BloomSettings(C.Structure):
    """OxcBloomSettings: the bloom cvars the passes read and the scene flags (only HasEyeAdaptation is read)"""
    _fields_ = [("threshold", C.c_float), ("soft_threshold", C.c_float), ("clamp_value", C.c_float), ("radius", C.c_float),
                ("scene_flags", C.c_uint32)]


class BloomTargets(C.Structure):
    """OxcBloomTargets: the two chains (device pointers, float4 texels, 16-byte aligned)"""
    _fields_ = [("downsampled", C.c_void_p), ("upsampled", C.c_void_p)]


assert C.sizeof(EyeAdaptationSettings) == 16 and C.sizeof(Exposure) == 8 and C.sizeof(BloomSettings) == 20 and C.sizeof(BloomTargets) == 16
HISTOGRAM_BIN_COUNT = 256
BLOOM_MAX_LEVELS = 15


def eye_adaptation_settings(min_exposure=-11.5, max_exposure=18.0, adaptation_speed=1.1, ev100_bias=1.0):
    """EyeAdaptationSettings with the AutoExposureComponent defaults"""
    return EyeAdaptationSettings(*[float(np.float32(v)) for v in (min_exposure, max_exposure, adaptation_speed, ev100_bias)])


def bloom_settings(threshold=1.0, soft_threshold=0.125, clamp_value=4.0, radius=0.75, scene_flags=0):
    """BloomSettings with the reference's cvar defaults (bloom_threshold, bloom_soft_threshold, bloom_clamp, bloom_radius)"""
    return BloomSettings(*[float(np.float32(v)) for v in (threshold, soft_threshold, clamp_value, radius)], int(scene_flags))


def bloom_levels(width: int, height: int):
    """[(w, h, first texel)] of the levels of a width x height frame's bloom chains (oxc_bloom's layout)"""
    w, h = width // 2, height // 2
    out, off = [], 0
    for k in range(max(w, h).bit_length()):
        lw, lh = max(1, w >> k), max(1, h >> k)
        out.append((lw, lh, off))
        off += lw * lh
    return out


def bloom_chain_texels(width: int, height: int) -> int:
    """float4 texels of one bloom chain (oxc_bloom_chain_texels)"""
    return sum(w * h for w, h, _ in bloom_levels(width, height))


TONEMAP_NONE, TONEMAP_ACES, TONEMAP_AGX, TONEMAP_GT7 = 0, 1, 2, 3


class TonemapSettings(C.Structure):
    """OxcTonemapSettings: the tonemap's scene flags and curve, the pp.* cvars and the lens components' settings"""
    _fields_ = [("scene_flags", C.c_uint32), ("tonemap_type", C.c_uint32), ("exposure", C.c_float), ("bloom_intensity", C.c_float),
                ("chromatic_aberration_amount", C.c_float), ("vignette_amount", C.c_float), ("film_grain_scale", C.c_float),
                ("film_grain_amount", C.c_float), ("film_grain_seed", C.c_uint32)]


assert C.sizeof(TonemapSettings) == 36


def tonemap_settings(scene_flags=0, tonemap_type=TONEMAP_AGX, exposure=1.0, bloom_intensity=0.1, chromatic_aberration_amount=0.5,
                     vignette_amount=0.5, film_grain_scale=0.7, film_grain_amount=0.6, film_grain_seed=0):
    """TonemapSettings with the reference's defaults: TonemappingComponent's AgX, the pp.exposure and pp.bloom_intensity cvars, the
    vignette, chromatic aberration and film grain components; the seed is the frame count % 16"""
    f = [float(np.float32(v)) for v in (exposure, bloom_intensity, chromatic_aberration_amount, vignette_amount, film_grain_scale,
                                        film_grain_amount)]
    return TonemapSettings(int(scene_flags), int(tonemap_type), *f, int(film_grain_seed) & 0xFFFFFFFF)


def atmosphere(**overrides):
    """Atmosphere with the GPU::Atmosphere{} defaults and the reference's LUT sizes; any field may be overridden by name"""
    a = Atmosphere()
    for name, value in dict(ATMOSPHERE_DEFAULTS, **overrides).items():
        if name not in ATMOSPHERE_DEFAULTS:
            raise TypeError(f"Atmosphere has no field {name}")
        if name.endswith("_size"):
            getattr(a, name)[:] = [int(v) for v in value]
        elif np.ndim(value):
            getattr(a, name)[:] = [float(np.float32(v)) for v in value]
        else:
            setattr(a, name, float(np.float32(value)))
    return a


MESH_MAX_LODS = 8


class MeshInput(C.Structure):
    """OxbMeshInput"""

    _fields_ = [
        ("positions", C.c_void_p),
        ("normals", C.c_void_p),
        ("texcoords", C.c_void_p),
        ("vertex_count", C.c_uint32),
        ("lod_count", C.c_uint32),
        ("lod_indices", C.c_void_p * MESH_MAX_LODS),
        ("lod_index_counts", C.c_uint32 * MESH_MAX_LODS),
        ("lod_errors", C.c_float * MESH_MAX_LODS),
        ("cluster_mode", C.c_uint32),
        ("auto_lods", C.c_uint32),
    ]


class OrcHiz(C.Structure):
    """OrcHiz (oracle/oxc_oracle.h) — also used as a plain layout helper"""

    _fields_ = [
        ("data", C.c_void_p),
        ("width", C.c_uint32),
        ("height", C.c_uint32),
        ("levels", C.c_uint32),
        ("level_offset", C.c_uint32 * HIZ_MAX_LEVELS),
    ]


class FrameResult(C.Structure):
    """OxrFrameResult"""

    _fields_ = [
        ("total", C.c_uint32),
        ("early", C.c_uint32),
        ("late", C.c_uint32),
        ("draw_index_count_early", C.c_uint32),
        ("draw_index_count_late", C.c_uint32),
        ("raster_triangles", C.c_uint64),
    ]


def hiz_extent(width: int, height: int):
    """RendererInstance.cpp:573-577: bit_ceil((W+1)>>1) per axis."""

    def bit_ceil(v):
        return 1 if v <= 1 else 1 << (int(v) - 1).bit_length()

    return bit_ceil((width + 1) >> 1), bit_ceil((height + 1) >> 1)


def hiz_layout(w: int, h: int):
    """(levels, offsets[levels], total_texels) — Texture.hpp:144-146 + min(.,13)."""
    levels = min(int(max(w, h)).bit_length(), HIZ_MAX_LEVELS)
    offs, off = [], 0
    for l in range(levels):
        offs.append(off)
        off += max(1, w >> l) * max(1, h >> l)
    return levels, offs, off
