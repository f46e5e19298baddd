"""Seeded synthetic scenes for the meshlet visibility pipeline (SURVEY.md §8d).

Produces exactly the tables RendererInstance::update receives
(Oxylus/src/Scene/Scene.cpp:1226-1290): GPU::Mesh[] / GPU::MeshInstance[] / TransformWorld[] plus the
geometry blob whose layout follows build_gltf_mesh's blob packing
(Oxylus/src/Asset/AssetManager_GLTF.cpp:748-768): per mesh  positions(u16x4) | per LOD: meshlets,
meshlet_bounds, local_triangle_indices (u8 packed, padded to 4), indirect_vertex_indices | MeshLOD[].
Mesh/MeshLOD u64 members are byte offsets into the blob (rebased by oxc_set_scene).

All randomness is SplitMix64 (one stream per array), seed 0x0C115EED + config index.
This module is PRODUCT code (bench.py uses it): it never touches oracle/.
"""
from dataclasses import dataclass, field

import numpy as np

from . import abi

SEED_BASE = 0x0C115EED
_GOLDEN = np.uint64(0x9E3779B97F4A7C15)


def splitmix64(seed: int, stream: int, n: int) -> np.ndarray:
    """n SplitMix64 outputs of the generator seeded with hash(seed, stream)."""
    with np.errstate(over="ignore"):
        s0 = np.uint64(seed & 0xFFFFFFFFFFFFFFFF) + np.uint64(stream) * np.uint64(0xD1B54A32D192ED03)
        z = s0 + (np.arange(1, n + 1, dtype=np.uint64) * _GOLDEN)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return z


def uniform(seed, stream, n, lo=0.0, hi=1.0):
    u = (splitmix64(seed, stream, n) >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)
    return lo + (hi - lo) * u


def randint(seed, stream, n, lo, hi):
    """integers in [lo, hi]"""
    return (lo + (splitmix64(seed, stream, n) % np.uint64(hi - lo + 1)).astype(np.int64)).astype(np.int64)


def quantize_half(x: np.ndarray) -> np.ndarray:
    """f32 -> IEEE half bits (round-to-nearest-even).  Only the DECODE side
    (com::dequantize_half, common/math.slang:193-201) matters for cull parity."""
    return np.asarray(x, dtype=np.float32).astype(np.float16).view(np.uint16)


def perspective_reverse_z(fov_deg=60.0, aspect=16.0 / 9.0, near=0.1, far=1000.0) -> np.ndarray:
    """Camera::update (Oxylus/src/Render/Camera.cpp:36-54): glm::perspective(fov, aspect, far, near) with
    GLM_FORCE_DEPTH_ZERO_TO_ONE (Oxylus/xmake.lua:58), then P[1][1] *= -1.  Column-major 16 floats (f32 math)."""
    f32 = np.float32
    t = f32(np.tan(f32(np.radians(f32(fov_deg))) / f32(2.0)))
    z_near, z_far = f32(far), f32(near)  # swapped: reversed-z
    m = np.zeros((4, 4), dtype=np.float32)  # m[col][row]
    m[0][0] = f32(1.0) / (f32(aspect) * t)
    m[1][1] = f32(1.0) / t
    m[2][2] = z_far / (z_near - z_far)
    m[2][3] = f32(-1.0)
    m[3][2] = -(z_far * z_near) / (z_far - z_near)
    m[1][1] *= f32(-1.0)
    return m.reshape(16)


def look_at(eye, center, up) -> np.ndarray:
    """glm::lookAt (RH), column-major 16 floats."""
    eye, center, up = (np.asarray(v, dtype=np.float64) for v in (eye, center, up))
    f = center - eye
    f /= np.linalg.norm(f)
    s = np.cross(f, up)
    s /= np.linalg.norm(s)
    u = np.cross(s, f)
    m = np.eye(4, dtype=np.float64)  # m[col][row]
    m[0][0], m[1][0], m[2][0] = s
    m[0][1], m[1][1], m[2][1] = u
    m[0][2], m[1][2], m[2][2] = -f
    m[3][0], m[3][1], m[3][2] = -np.dot(s, eye), -np.dot(u, eye), np.dot(f, eye)
    return m.astype(np.float32).reshape(16)


def mat_mul_cm(a16, b16):
    """column-major 4x4 product in f32 (host-side camera setup only)."""
    a = np.asarray(a16, dtype=np.float32).reshape(4, 4).T
    b = np.asarray(b16, dtype=np.float32).reshape(4, 4).T
    return (a @ b).T.astype(np.float32).reshape(16)


def camera_matrices(width, height, yaw_deg=0.0, eye=(0.0, 0.0, 0.0), fov=60.0, near=0.1, far=1000.0):
    """(projection, view), column-major 16 floats each: the two matrices make_camera multiplies into projection_view"""
    yaw = np.radians(yaw_deg)
    fwd = np.array([-np.sin(yaw), 0.0, -np.cos(yaw)])
    view = look_at(eye, np.asarray(eye) + fwd, (0.0, 1.0, 0.0))
    proj = perspective_reverse_z(fov, width / height, near, far)
    return proj, view


def make_camera(width, height, mesh_instance_count, yaw_deg=0.0, eye=(0.0, 0.0, 0.0), fov=60.0, near=0.1, far=1000.0):
    """CullCamera as RendererInstance::render fills it (RendererInstance.cpp:783-790)."""
    cam = np.zeros(1, dtype=abi.CULL_CAMERA_DT)
    proj, view = camera_matrices(width, height, yaw_deg, eye, fov, near, far)
    cam["projection_view"][0] = mat_mul_cm(proj, view)
    cam["position"][0] = eye
    cam["acceptable_lod_error"] = 2.0  # RendererInstance.cpp:1394
    cam["resolution"][0] = (width, height)
    cam["near_clip"] = near
    cam["mesh_instance_count"] = mesh_instance_count
    return cam


def pbr_camera(cull_camera):
    """abi.PbrCamera of a make_camera camera: the binary64 inverse of its projection_view (column-major), rounded to binary32, and its
    position"""
    inv = np.linalg.inv(cull_camera["projection_view"][0].reshape(4, 4).T.astype(np.float64)).T.astype(np.float32).reshape(16)
    return abi.pbr_camera(inv, cull_camera["position"][0])


def make_lights(rng, n, eye=(0.0, 0.0, 0.0), yaw_deg=0.0, spot_fraction=0.5, distance=(3.0, 60.0), radius=(2.0, 25.0), intensity=(0.5, 40.0)):
    """n seeded point and spot lights (abi.Light array) placed in front of a make_camera camera at `eye` / `yaw_deg`: positions up to
    45 degrees off the view axis at `distance`, 0.5..6 m above the eye's height, ranges in `radius` (each lights part of the view),
    colours in [0.2, 1], spots aimed at a point on the axis with cone angles of 0.1..0.9 rad (inner <= outer)"""
    lights = (abi.Light * n)()
    yaw = np.radians(yaw_deg)
    for i in range(n):
        d = rng.uniform(*distance)
        a = yaw + rng.uniform(-np.pi / 4, np.pi / 4)
        p = np.asarray(eye, np.float64) + (-np.sin(a) * d, rng.uniform(0.5, 6.0), -np.cos(a) * d)
        L = lights[i]
        L.position[:] = [float(np.float32(v)) for v in p]
        L.intensity = float(np.float32(rng.uniform(*intensity)))
        L.color[:] = [float(np.float32(v)) for v in rng.uniform(0.2, 1.0, 3)]
        L.range = float(np.float32(rng.uniform(*radius)))
        if rng.random() < spot_fraction:
            L.kind = abi.LIGHT_SPOT
            target = np.asarray(eye, np.float64) + (-np.sin(yaw) * rng.uniform(*distance), -2.0, -np.cos(yaw) * rng.uniform(*distance))
            L.direction[:] = [float(np.float32(v)) for v in target - p]
            inner = rng.uniform(0.1, 0.6)
            L.inner_cone_angle, L.outer_cone_angle = float(np.float32(inner)), float(np.float32(inner + rng.uniform(0.0, 0.3)))
        else:
            L.kind = abi.LIGHT_POINT
    return lights


def make_ortho_view(direction, center, half_size, depth_range, mesh_instance_count, resolution=2048):
    """Orthographic reverse-Z shadow-cascade style view (Camera.cpp:44-52 shape) for the multi-view config.
    position carries the light direction (-dir), as the reference does for directional cone tests
    (Shadowmaps.cpp:433-463)."""
    d = np.asarray(direction, dtype=np.float64)
    d /= np.linalg.norm(d)
    up = np.array([0.0, 1.0, 0.0]) if abs(d[1]) < 0.9 else np.array([1.0, 0.0, 0.0])
    eye = np.asarray(center, dtype=np.float64) - d * depth_range * 0.5
    view = look_at(eye, eye + d, up)
    # glm::ortho(l, r, b, t, zNear=far, zFar=near) ZO, reversed
    l, r, b, t = -half_size, half_size, -half_size, half_size
    zn, zf = depth_range, 0.0
    m = np.eye(4, dtype=np.float64)
    m[0][0] = 2.0 / (r - l)
    m[1][1] = 2.0 / (t - b)
    m[2][2] = -1.0 / (zf - zn)
    m[3][0] = -(r + l) / (r - l)
    m[3][1] = -(t + b) / (t - b)
    m[3][2] = -zn / (zf - zn)
    m[1][1] *= -1.0
    cam = np.zeros(1, dtype=abi.CULL_CAMERA_DT)
    cam["projection_view"][0] = mat_mul_cm(m.astype(np.float32).reshape(16), view)
    cam["position"][0] = -d
    cam["acceptable_lod_error"] = 2.0
    cam["resolution"][0] = (resolution, resolution)
    cam["near_clip"] = 0.0
    cam["mesh_instance_count"] = mesh_instance_count
    return cam


def make_vsm_clipmaps(light_dir, camera_position, count=10, first_clipmap_width=10.0, max_shadow_dist=1000.0, page_table_size=64):
    """The directional light's virtual clipmaps as the reference builds them (Passes/Shadowmaps.cpp:9-60): light_dir points TOWARDS the
    light (the view looks along -light_dir), glm::lookAtRH from the origin, glm::orthoRH_ZO(+-extent, near = -max_shadow_dist,
    far = +max_shadow_dist) with y flipped, so a point closer to the light has the SMALLER depth; the projection is shifted by whole
    pages so that the camera sits in the centre page, and page_offset is that shift.  Returns an abi.CLIPMAP_DT array."""
    fwd = -np.asarray(light_dir, dtype=np.float64)
    fwd /= np.linalg.norm(fwd)
    up = (0.0, 1.0, 0.0) if 1.0 - abs(fwd[1]) >= 1e-5 else (0.0, 0.0, 1.0)
    view = look_at((0.0, 0.0, 0.0), fwd, up).reshape(4, 4).T.astype(np.float64)  # row-major
    cm = np.zeros(count, dtype=abi.CLIPMAP_DT)
    for k in range(count):
        e = first_clipmap_width * float(1 << k)
        n, f = -max_shadow_dist, max_shadow_dist
        proj = np.eye(4)
        proj[0, 0], proj[1, 1], proj[2, 2], proj[2, 3] = 1.0 / e, -1.0 / e, -1.0 / (f - n), -n / (f - n)  # orthoRH_ZO, [1][1] *= -1
        clip = proj @ view @ np.append(np.asarray(camera_position, dtype=np.float64), 1.0)
        offset = np.trunc(clip[:2] / clip[3] * 0.5 * page_table_size).astype(np.int32)  # glm::ivec2 truncates
        shift = np.eye(4)
        shift[:2, 3] = -(offset / page_table_size) * 2.0
        cm["projection_view_mat"][k] = (shift @ proj @ view).astype(np.float32).T.reshape(16)
        cm["page_offset"][k] = offset
        cm["z_near"][k] = n
    return cm


# 7x7 grid patch: 49 vertices, 72 triangles, the last 8 dropped -> 64 (SURVEY §8d)
_GRID = 7
_VERTS = _GRID * _GRID


def _patch_topology():
    tris = []
    for j in range(_GRID - 1):
        for i in range(_GRID - 1):
            p00 = j * _GRID + i
            p10 = p00 + 1
            p01 = p00 + _GRID
            p11 = p01 + 1
            tris.append((p00, p10, p11))  # CCW about t x b
            tris.append((p00, p11, p01))
    return np.asarray(tris[:64], dtype=np.uint8)


_TOPO = _patch_topology()


@dataclass
class Scene:
    meshes: np.ndarray
    mesh_instances: np.ndarray
    transforms: np.ndarray
    blob: np.ndarray  # uint8
    max_meshlet_instance_count: int  # Σ LOD0 meshlets (Scene.cpp:1226-1264)
    width: int
    height: int
    seed: int
    occluder_depth: np.ndarray = None  # H x W f32 reverse-Z depth of the synthetic occluders
    info: dict = field(default_factory=dict)

    @property
    def mesh_instance_count(self):
        return len(self.mesh_instances)

    def camera(self, yaw_deg=0.0):
        return make_camera(self.width, self.height, self.mesh_instance_count, yaw_deg)

    def hiz_extent(self):
        return abi.hiz_extent(self.width, self.height)


def _align(n, a):
    return (n + a - 1) // a * a


def _build_unique_meshes(seed, counts, lod_counts, ragged):
    """Vectorised over all meshlets of all LODs of all unique meshes.
    Returns (meshes, blob)."""
    n_mesh = len(counts)
    # per (mesh, lod) meshlet counts: LOD k has ceil(count / 2^k) meshlets
    lod_meshlets = [[max(1, -(-int(counts[m]) // (1 << k))) for k in range(int(lod_counts[m]))] for m in range(n_mesh)]
    total = int(sum(sum(l) for l in lod_meshlets))

    # --- geometry of every meshlet (patch) ---
    org = np.stack([uniform(seed, 10 + a, total, -4.0, 4.0) for a in range(3)], axis=1)
    size = np.exp(uniform(seed, 13, total, np.log(0.02), np.log(0.3)))
    # random orthonormal frame from a quaternion
    q = np.stack([uniform(seed, 14 + a, total, -1.0, 1.0) for a in range(4)], axis=1)
    q /= np.maximum(np.linalg.norm(q, axis=1, keepdims=True), 1e-9)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    t = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y + z * w), 2 * (x * z - y * w)], axis=1)
    b = np.stack([2 * (x * y - z * w), 1 - 2 * (x * x + z * z), 2 * (y * z + x * w)], axis=1)
    nrm = np.cross(t, b)
    curv = uniform(seed, 18, total, -0.6, 0.6)
    gi, gj = np.meshgrid(np.arange(_GRID), np.arange(_GRID), indexing="xy")
    u0 = (gi.reshape(-1) / (_GRID - 1) - 0.5)[None, :]
    v0 = (gj.reshape(-1) / (_GRID - 1) - 0.5)[None, :]
    ju = uniform(seed, 19, total * _VERTS, -0.03, 0.03).reshape(total, _VERTS)
    jv = uniform(seed, 20, total * _VERTS, -0.03, 0.03).reshape(total, _VERTS)
    jn = uniform(seed, 21, total * _VERTS, -0.01, 0.01).reshape(total, _VERTS)
    u = u0 + ju
    v = v0 + jv
    hgt = curv[:, None] * (u * u + v * v) + jn
    pos = (
        org[:, None, :]
        + size[:, None, None] * (u[:, :, None] * t[:, None, :] + v[:, :, None] * b[:, None, :] + hgt[:, :, None] * nrm[:, None, :])
    ).astype(np.float32)  # total x 49 x 3

    tri_count = np.full(total, 64, dtype=np.int64)
    if ragged:
        tri_count = randint(seed, 22, total, 1, 64)

    # bounds (AssetManager_GLTF.cpp:692-741): AABB over vertices referenced by the meshlet's triangles
    tp = pos[:, _TOPO.reshape(-1), :].reshape(total, 64, 3, 3)  # total x tri x corner x xyz
    valid = (np.arange(64)[None, :] < tri_count[:, None])
    big = np.float32(3.0e38)
    tmin = np.where(valid[:, :, None, None], tp, big).min(axis=(1, 2))
    tmax = np.where(valid[:, :, None, None], tp, -big).max(axis=(1, 2))
    center = (tmax + tmin) * np.float32(0.5)
    extent = tmax - tmin
    # normal cone (meshopt_computeMeshletBounds shape): axis = mean triangle normal, cutoff = sqrt(1 - mindp^2)
    e1 = tp[:, :, 1, :] - tp[:, :, 0, :]
    e2 = tp[:, :, 2, :] - tp[:, :, 0, :]
    tn = np.cross(e1.astype(np.float64), e2.astype(np.float64))
    tn /= np.maximum(np.linalg.norm(tn, axis=2, keepdims=True), 1e-30)
    tn = np.where(valid[:, :, None], tn, 0.0)
    axis = tn.sum(axis=1)
    axis /= np.maximum(np.linalg.norm(axis, axis=1, keepdims=True), 1e-30)
    dp = np.where(valid, (tn * axis[:, None, :]).sum(axis=2), 1.0)
    mindp = dp.min(axis=1)
    axis_s8 = np.clip(np.rint(axis * 127.0), -127, 127).astype(np.int8)
    axis_q = axis_s8.astype(np.float64) / 127.0
    axis_err = np.abs(axis_q - axis).sum(axis=1)
    cutoff = np.sqrt(np.maximum(0.0, 1.0 - mindp * mindp))
    cutoff_s8 = np.minimum(127, np.floor(cutoff * 127.0 + axis_err * 127.0 + 1.0)).astype(np.int64)
    # 25 % cone-disabled (and degenerate cones, mindp <= 0.1, as meshopt does)
    disable = (uniform(seed, 23, total) < 0.25) | (mindp <= 0.1)
    cutoff_s8 = np.where(disable, 127, cutoff_s8).astype(np.int8)

    bounds = np.zeros(total, dtype=abi.MESHLET_BOUNDS_DT)
    bounds["aabb_center"] = quantize_half(center)
    bounds["aabb_extent"] = quantize_half(extent)
    bounds["cone_axis_xy"] = axis_s8[:, :2]
    bounds["cone_axis_z"] = axis_s8[:, 2]
    bounds["cone_cutoff"] = cutoff_s8

    pos_q = np.zeros((total, _VERTS, 4), dtype=np.uint16)
    pos_q[:, :, :3] = quantize_half(pos)
    # vertex attributes the vis-buffer decode reads (AssetManager_GLTF.cpp:579-581 packing): analytic normal of the
    # height field, 10:10:10 unorm (scene.slang:486-489 decodes c / 511 - 1); uv = grid parameter as half2
    nv = nrm[:, None, :] - (2.0 * curv[:, None] * u)[:, :, None] * t[:, None, :] - (2.0 * curv[:, None] * v)[:, :, None] * b[:, None, :]
    nv /= np.maximum(np.linalg.norm(nv, axis=2, keepdims=True), 1e-30)
    nq = np.clip(np.rint((nv + 1.0) * 511.0), 0, 1022).astype(np.uint32)
    normals_q = (nq[:, :, 0] << 20) | (nq[:, :, 1] << 10) | nq[:, :, 2]
    uv_q = quantize_half(np.stack([u + 0.5, v + 0.5], axis=2).astype(np.float32))  # total x 49 x 2 u16

    # --- pack the blob ---
    meshes = np.zeros(n_mesh, dtype=abi.MESH_DT)
    chunks, off = [], 0

    def put(arr, align=16):
        nonlocal off
        pad = _align(off, align) - off
        if pad:
            chunks.append(np.zeros(pad, dtype=np.uint8))
            off += pad
        start = off
        raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
        chunks.append(raw)
        off += raw.size
        return start

    cursor = 0
    for m in range(n_mesh):
        n_all = sum(lod_meshlets[m])
        sl = slice(cursor, cursor + n_all)
        meshes[m]["vertex_positions"] = put(pos_q[sl].reshape(-1, 4))
        meshes[m]["vertex_normals"] = put(normals_q[sl].reshape(-1))
        meshes[m]["texture_coords"] = put(uv_q[sl].reshape(-1, 2))
        meshes[m]["vertex_count"] = n_all * _VERTS
        meshes[m]["lod_count"] = lod_counts[m]
        lods = np.zeros(int(lod_counts[m]), dtype=abi.MESH_LOD_DT)
        lcur = cursor
        for k, nk in enumerate(lod_meshlets[m]):
            ls = slice(lcur, lcur + nk)
            tcs = tri_count[ls]
            meshlets = np.zeros(nk, dtype=abi.MESHLET_DT)
            # micro indices: (triangle_count*3 + 3) & ~3 bytes per meshlet (AssetManager_GLTF.cpp:689)
            sizes = (tcs * 3 + 3) & ~3
            offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
            micro = np.zeros(int(sizes.sum()), dtype=np.uint8)
            if not ragged:
                micro[:] = np.tile(_TOPO.reshape(-1), nk)
            else:
                flat = _TOPO.reshape(-1)
                for i in range(nk):
                    micro[offs[i] : offs[i] + tcs[i] * 3] = flat[: tcs[i] * 3]
            meshlets["local_triangle_index_offset"] = offs
            vbase = (np.arange(lcur - cursor, lcur - cursor + nk, dtype=np.int64)) * _VERTS
            meshlets["indirect_vertex_index_offset"] = np.arange(nk, dtype=np.int64) * _VERTS
            meshlets["vertex_count"] = _VERTS
            meshlets["triangle_count"] = tcs
            vidx = (vbase[:, None] + np.arange(_VERTS)[None, :]).astype(np.uint32).reshape(-1)
            lods[k]["meshlets"] = put(meshlets)
            lods[k]["meshlet_bounds"] = put(bounds[ls])
            lods[k]["local_triangle_indices"] = put(micro)
            lods[k]["indirect_vertex_indices"] = put(vidx)
            lods[k]["meshlet_count"] = nk
            lods[k]["meshlet_bounds_count"] = nk
            lods[k]["local_triangle_indices_count"] = micro.size
            lods[k]["indirect_vertex_indices_count"] = vidx.size
            lods[k]["error"] = 0.0 if k == 0 else 0.002 * (4.0**k)
            lcur += nk
        meshes[m]["lods"] = put(lods)
        # mesh bounds from LOD0 (AssetManager_GLTF.cpp:743-746)
        l0 = slice(cursor, cursor + lod_meshlets[m][0])
        mn = tmin[l0].min(axis=0)
        mx = tmax[l0].max(axis=0)
        meshes[m]["bounds"]["aabb_center"] = (mx + mn) * np.float32(0.5)
        meshes[m]["bounds"]["aabb_extent"] = mx - mn
        cursor += n_all
    blob = np.concatenate(chunks) if chunks else np.zeros(0, dtype=np.uint8)
    pad = _align(blob.size, 16) - blob.size
    if pad:
        blob = np.concatenate([blob, np.zeros(pad, dtype=np.uint8)])
    return meshes, blob, [l[0] for l in lod_meshlets]


def make_scene(
    n_meshlets: int,
    config_index: int = 2,
    width: int = 1920,
    height: int = 1080,
    n_unique_meshes: int = 256,
    meshlets_per_mesh=(64, 256),
    max_lods: int = 1,
    ragged: bool = False,
    n_occluders: int = 32,
    placement: str = "frustum",
    seed: int = None,
    instance_scale: float = 1.0,
) -> Scene:
    """Scene with exactly n_meshlets LOD0 meshlet instances (Σ over mesh instances).

    placement="frustum": instance centres inside the view frustum of the yaw-0 camera (every mesh
    instance intersects the frustum, so cull_meshes emits all n_meshlets with single-LOD meshes);
    placement="box": the SURVEY §8d 400x100x400 box 200 units ahead (≈45 % of instances outside).
    instance_scale multiplies every mesh instance's uniform scale: weak-scaling runs shrink instances by world^-1/2 so
    the screen coverage — hence the share of meshlets that survive occlusion, per GPU — stays what it is on one GPU.
    """
    seed = SEED_BASE + config_index if seed is None else seed
    lo, hi = meshlets_per_mesh
    n_unique_meshes = max(1, min(n_unique_meshes, max(1, n_meshlets // max(1, (lo + hi) // 2))))
    counts = randint(seed, 1, n_unique_meshes, lo, hi)
    counts = np.minimum(counts, max(1, n_meshlets))
    # mesh instances: random mesh each until the total would exceed n; remainder -> filler mesh
    est = int(n_meshlets / counts.mean() * 1.3) + 16
    pick = randint(seed, 2, est, 0, n_unique_meshes - 1)
    csum = np.cumsum(counts[pick])
    n_inst = int(np.searchsorted(csum, n_meshlets, side="right"))
    while n_inst == est:  # pragma: no cover (est is generous)
        est *= 2
        pick = randint(seed, 2, est, 0, n_unique_meshes - 1)
        csum = np.cumsum(counts[pick])
        n_inst = int(np.searchsorted(csum, n_meshlets, side="right"))
    used = int(csum[n_inst - 1]) if n_inst > 0 else 0
    rem = n_meshlets - used
    pick = pick[:n_inst]
    lod_counts = np.ones(n_unique_meshes, dtype=np.int64)
    if max_lods > 1:
        lod_counts = randint(seed, 3, n_unique_meshes, 1, max_lods)
    if rem > 0:
        counts = np.concatenate([counts, [rem]])
        lod_counts = np.concatenate([lod_counts, [1]])
        pick = np.concatenate([pick, [len(counts) - 1]])
        n_inst += 1
    meshes, blob, lod0 = _build_unique_meshes(seed, counts, lod_counts, ragged)
    lod0 = np.asarray(lod0, dtype=np.int64)

    # transforms: rotation x uniform scale x translation
    q = np.stack([uniform(seed, 30 + a, n_inst, -1.0, 1.0) for a in range(4)], axis=1)
    q /= np.maximum(np.linalg.norm(q, axis=1, keepdims=True), 1e-9)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    s = uniform(seed, 34, n_inst, 0.5, 2.0) * float(instance_scale)
    rot = np.empty((n_inst, 3, 3))
    rot[:, 0, 0] = 1 - 2 * (y * y + z * z); rot[:, 0, 1] = 2 * (x * y - z * w); rot[:, 0, 2] = 2 * (x * z + y * w)
    rot[:, 1, 0] = 2 * (x * y + z * w); rot[:, 1, 1] = 1 - 2 * (x * x + z * z); rot[:, 1, 2] = 2 * (y * z - x * w)
    rot[:, 2, 0] = 2 * (x * z - y * w); rot[:, 2, 1] = 2 * (y * z + x * w); rot[:, 2, 2] = 1 - 2 * (x * x + y * y)
    if placement == "frustum":
        # depth log-uniform in [15, 600]; x/y inside the frustum cross-section (fov 60, 16:9) with 8 % margin.
        # With patch sizes log-uniform in [0.02, 0.3] this gives ~30 % steady-state visible meshlets at 1M / 1080p
        # (cone ~35 %, frustum, Hi-Z occlusion do the rest) and mostly pixel-sized triangles.
        d = np.exp(uniform(seed, 35, n_inst, np.log(15.0), np.log(600.0)))
        th = np.tan(np.radians(60.0) / 2.0)
        px = uniform(seed, 36, n_inst, -0.92, 0.92) * d * th * (width / height)
        py = uniform(seed, 37, n_inst, -0.92, 0.92) * d * th
        trans = np.stack([px, py, -d], axis=1)
    else:
        trans = np.stack(
            [uniform(seed, 36, n_inst, -200.0, 200.0), uniform(seed, 37, n_inst, -50.0, 50.0),
             uniform(seed, 35, n_inst, -400.0, 0.0)], axis=1)
    world = np.zeros((n_inst, 4, 4), dtype=np.float32)  # [col][row]
    world[:, :3, :3] = np.transpose(rot * s[:, None, None], (0, 2, 1)).astype(np.float32)
    world[:, 3, :3] = trans.astype(np.float32)
    world[:, 3, 3] = 1.0
    transforms = np.zeros(n_inst, dtype=abi.TRANSFORM_DT)
    transforms["world"] = world.reshape(n_inst, 16)

    mesh_instances = np.zeros(n_inst, dtype=abi.MESH_INSTANCE_DT)
    mesh_instances["mesh_index"] = pick
    mesh_instances["transform_index"] = np.arange(n_inst)
    l0 = lod0[pick]
    mesh_instances["meshlet_instance_visibility_offset"] = np.concatenate([[0], np.cumsum(l0)[:-1]])  # Scene.cpp:1255-1260
    total = int(l0.sum())
    assert total == n_meshlets, (total, n_meshlets)

    sc = Scene(meshes, mesh_instances, transforms, blob, total, width, height, seed)
    sc.occluder_depth = make_occluder_depth(seed, width, height, n_occluders)
    sc.info = dict(n_unique_meshes=len(meshes), n_mesh_instances=n_inst, unique_meshlets=int(sum(
        int(-(-int(c) // 1)) for c in counts)), blob_bytes=int(blob.size), placement=placement)
    return sc


def with_ground_caster(scene: Scene, half_size=1200.0, center=(0.0, 0.0, -40.0), grid=32):
    """`scene` plus one more mesh instance: a tessellated plane y = center.y of 2 * half_size per side, the shadow caster under the
    other instances.  grid x grid meshlets of 4 x 8 quads (45 vertices, 64 triangles each) over a local [-1, 1]^2 whose vertex
    coordinates are exact in half precision (multiples of 1 / (8 * grid)); the world matrix scales x and z by half_size."""
    nx, nz = 4 * grid + 1, 8 * grid + 1
    gx, gz = np.meshgrid(np.arange(nx) / (2.0 * grid) - 1.0, np.arange(nz) / (4.0 * grid) - 1.0, indexing="ij")
    pos = np.zeros((nx * nz, 4), dtype=np.uint16)
    pos[:, 0], pos[:, 2] = quantize_half(gx.reshape(-1).astype(np.float32)), quantize_half(gz.reshape(-1).astype(np.float32))
    lx, lz = np.meshgrid(np.arange(5), np.arange(9), indexing="ij")
    local = (lx * 9 + lz).reshape(-1)                    # meshlet-local vertex index of (x, z)
    q = (np.arange(4)[:, None] * 9 + np.arange(8)[None, :]).reshape(-1)
    tris = np.stack([np.stack([q, q + 10, q + 9], 1), np.stack([q, q + 1, q + 10], 1)], 1).reshape(-1, 3).astype(np.uint8)
    mi, mj = np.meshgrid(np.arange(grid), np.arange(grid), indexing="ij")
    mi, mj = mi.reshape(-1), mj.reshape(-1)
    n = grid * grid
    vidx = ((mi[:, None] * 4 + lx.reshape(-1)[None, :]) * nz + mj[:, None] * 8 + lz.reshape(-1)[None, :]).astype(np.uint32)
    assert (local == np.arange(45)).all()
    meshlets = np.zeros(n, dtype=abi.MESHLET_DT)
    meshlets["indirect_vertex_index_offset"] = np.arange(n) * 45
    meshlets["local_triangle_index_offset"] = np.arange(n) * 192
    meshlets["vertex_count"], meshlets["triangle_count"] = 45, 64
    bounds = np.zeros(n, dtype=abi.MESHLET_BOUNDS_DT)
    cx, cz = (mi * 2 + 1) / grid - 1.0, (mj * 2 + 1) / grid - 1.0
    bounds["aabb_center"] = quantize_half(np.stack([cx, np.zeros(n), cz], 1).astype(np.float32))
    bounds["aabb_extent"] = quantize_half(np.tile(np.float32([2.0 / grid, 1.0 / 64, 2.0 / grid]), (n, 1)))
    bounds["cone_cutoff"] = 127  # no cone: a plane is seen from both sides
    chunks, off = [], _align(int(scene.blob.size), 16)

    def put(a):
        nonlocal off
        start = off
        raw = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        pad = (-raw.size) % 16
        chunks.append(np.concatenate([raw, np.zeros(pad, dtype=np.uint8)]))
        off += raw.size + pad
        return start

    mesh = np.zeros(1, dtype=abi.MESH_DT)
    mesh["vertex_positions"] = put(pos)
    mesh["vertex_count"], mesh["lod_count"] = nx * nz, 1
    lod = np.zeros(1, dtype=abi.MESH_LOD_DT)
    lod["meshlets"], lod["meshlet_bounds"] = put(meshlets), put(bounds)
    lod["local_triangle_indices"], lod["indirect_vertex_indices"] = put(np.tile(tris.reshape(-1), n)), put(vidx.reshape(-1))
    lod["meshlet_count"] = lod["meshlet_bounds_count"] = n
    lod["local_triangle_indices_count"], lod["indirect_vertex_indices_count"] = n * 192, n * 45
    mesh["lods"] = put(lod)
    mesh["bounds"]["aabb_center"][0] = (0.0, 0.0, 0.0)
    mesh["bounds"]["aabb_extent"][0] = (2.0, 1.0 / 64, 2.0)
    head = np.concatenate([scene.blob, np.zeros(_align(int(scene.blob.size), 16) - scene.blob.size, dtype=np.uint8)])
    blob = np.concatenate([head] + chunks)
    xf = np.zeros(1, dtype=abi.TRANSFORM_DT)
    w = np.diag([half_size, 1.0, half_size, 1.0]).astype(np.float32)
    w[3, :3] = center  # [col][row]: column 3 = translation
    xf["world"][0] = w.reshape(16)
    inst = np.zeros(1, dtype=abi.MESH_INSTANCE_DT)
    inst["mesh_index"], inst["transform_index"] = len(scene.meshes), len(scene.transforms)
    inst["meshlet_instance_visibility_offset"] = scene.max_meshlet_instance_count
    sc = Scene(np.concatenate([scene.meshes, mesh]), np.concatenate([scene.mesh_instances, inst]), np.concatenate([scene.transforms, xf]),
               blob, scene.max_meshlet_instance_count + n, scene.width, scene.height, scene.seed, scene.occluder_depth, dict(scene.info))
    sc.info["ground_caster"] = dict(half_size=half_size, center=tuple(center), meshlets=n, triangles=n * 64)
    return sc


def make_occluder_depth(seed, width, height, n_occluders=32, near=0.1, far=1000.0):
    """Depth (reverse-Z) of n screen-space occluder rectangles at seeded view distances — the stand-in
    for depth laid down by passes outside this path.  0 = nothing (far)."""
    depth = np.zeros((height, width), dtype=np.float32)
    if n_occluders <= 0:
        return depth
    p = perspective_reverse_z(60.0, width / height, near, far).reshape(4, 4)  # [col][row]
    cx = uniform(seed, 50, n_occluders, 0.0, 1.0)
    cy = uniform(seed, 51, n_occluders, 0.0, 1.0)
    hw = uniform(seed, 52, n_occluders, 0.03, 0.14)
    hh = uniform(seed, 53, n_occluders, 0.05, 0.20)
    dist = np.exp(uniform(seed, 54, n_occluders, np.log(20.0), np.log(150.0)))
    for i in range(n_occluders):
        zc = np.float32(p[2][2]) * np.float32(-dist[i]) + np.float32(p[3][2])
        zn = np.float32(zc / np.float32(dist[i]))
        x0, x1 = int(max(0, (cx[i] - hw[i]) * width)), int(min(width, (cx[i] + hw[i]) * width))
        y0, y1 = int(max(0, (cy[i] - hh[i]) * height)), int(min(height, (cy[i] + hh[i]) * height))
        if x1 > x0 and y1 > y0:
            depth[y0:y1, x0:x1] = np.maximum(depth[y0:y1, x0:x1], zn)
    return depth


def scene_desc(scene: Scene):
    """ctypes OxcSceneDesc over the scene's numpy buffers (keeps them alive via the returned tuple)."""
    keep = (np.ascontiguousarray(scene.meshes), np.ascontiguousarray(scene.mesh_instances),
            np.ascontiguousarray(scene.transforms), np.ascontiguousarray(scene.blob))
    d = abi.SceneDesc()
    d.meshes = keep[0].ctypes.data
    d.mesh_count = len(keep[0])
    d.mesh_instances = keep[1].ctypes.data
    d.mesh_instance_count = len(keep[1])
    d.transforms = keep[2].ctypes.data
    d.transform_count = len(keep[2])
    d.blob = keep[3].ctypes.data
    d.blob_size = keep[3].size
    return d, keep
