"""Terrain scenes shared by the terrain-draw tests and tools/bench_terrain.py: a seeded R16 heightmap, its patch min / max, the
TerrainData record, and the three cameras of the measurement (2 m above the ground looking at the horizon, aerial, grazing)."""
import numpy as np

from oxylus_b200 import abi, synth

DEFAULT_TEXEL_NOISE = 0.0005


def heightmap(res_x, res_y, seed, kind="noise", texel_noise=0.1):
    """uint16 [res_y, res_x]: 'flat' (all 0), 'noise' (smooth hills plus independent texel noise of texel_noise x the height range)
    or 'rough' (independent texels).  The default terrain of the measurement uses DEFAULT_TEXEL_NOISE, 0.2 m over its 400 m range:
    10 % would put 40 m spikes 0.5 m apart, walls that span the screen near the camera."""
    if kind == "flat":
        return np.zeros((res_y, res_x), np.uint16)
    rng = np.random.default_rng(seed)
    if kind == "rough":
        return rng.integers(0, 65536, (res_y, res_x), dtype=np.uint16)
    y, x = np.mgrid[0:res_y, 0:res_x].astype(np.float64)
    h = np.zeros((res_y, res_x))
    for k in range(4):
        fx, fy, ph = rng.uniform(1, 6) * (k + 1), rng.uniform(1, 6) * (k + 1), rng.uniform(0, 2 * np.pi, 2)
        h += np.sin(2 * np.pi * fx * x / res_x + ph[0]) * np.cos(2 * np.pi * fy * y / res_y + ph[1]) / (k + 1)
    h = (h - h.min()) / max(h.max() - h.min(), 1e-9)
    h = (1.0 - texel_noise) * h + texel_noise * rng.random((res_y, res_x))
    return np.clip(h * 65535.0, 0, 65535).astype(np.uint16)


def terrain(patch_count=(64, 64), world_size=(1024.0, 1024.0), height_range=(0.0, 400.0), world_origin=(0.0, 0.0)):
    """TERRAIN_DT record centred on world_origin (Terrain.hpp defaults: 1024 m, 64 x 64 patches, heights 0..400 m)"""
    t = np.zeros(1, abi.TERRAIN_DT)
    t["world_min"] = (world_origin[0] - world_size[0] / 2, world_origin[1] - world_size[1] / 2)
    t["world_size"] = world_size
    t["patch_count"] = patch_count
    t["base_height"] = height_range[0]
    t["height_scale"] = height_range[1] - height_range[0]
    return t


def patch_minmax(hm, patch_count):
    """float32 [patches, 2]: min / max of the normalised heights over the texels each patch's bilinear taps can reach"""
    ry, rx = hm.shape
    px, pz = patch_count
    out = np.zeros((pz * px, 2), np.float32)
    n = hm.astype(np.float32) / np.float32(65535.0)
    for j in range(pz):
        y0, y1 = max(0, j * ry // pz - 1), min(ry, -(-(j + 1) * ry // pz) + 1)
        for i in range(px):
            x0, x1 = max(0, i * rx // px - 1), min(rx, -(-(i + 1) * rx // px) + 1)
            blk = n[y0:y1, x0:x1]
            out[j * px + i] = (blk.min(), blk.max())
    return out


def height_at(hm, t, x, z):
    """approximate terrain height (binary64 bilinear) at world (x, z), for placing cameras"""
    ry, rx = hm.shape
    u = (x - float(t["world_min"][0][0])) / float(t["world_size"][0][0]) * rx - 0.5
    v = (z - float(t["world_min"][0][1])) / float(t["world_size"][0][1]) * ry - 0.5
    i, j = int(np.clip(np.floor(u), 0, rx - 1)), int(np.clip(np.floor(v), 0, ry - 1))
    return float(t["base_height"][0]) + float(hm[j, i]) / 65535.0 * float(t["height_scale"][0])


def camera(width, height, eye, center, fov=60.0, near=0.1, far=4000.0):
    """CullCamera looking from eye at center (world up +y)"""
    c = np.zeros(1, abi.CULL_CAMERA_DT)
    proj = synth.perspective_reverse_z(fov, width / height, near, far)
    view = synth.look_at(eye, center, (0.0, 1.0, 0.0))
    c["projection_view"][0] = synth.mat_mul_cm(proj, view)
    c["position"][0] = eye
    c["acceptable_lod_error"] = 2.0
    c["resolution"][0] = (width, height)
    c["near_clip"] = near
    return c


def views(hm, t, width, height, fov=60.0):
    """{name: camera}: 'horizon' 2 m above the ground looking level, 'aerial' 0.3 x the terrain's size above its top looking down at 45
    degrees (307 m over the default terrain), 'grazing' 20 m above the ground looking down at 8 degrees"""
    size = float(t["world_size"][0][0])
    cx, cz = float(t["world_min"][0][0]) + size / 2, float(t["world_min"][0][1]) + size / 2
    g = height_at(hm, t, cx, cz + size / 4)
    top = float(t["base_height"][0]) + float(t["height_scale"][0])
    out = {}
    e = (cx, g + 2.0, cz + size / 4)
    out["horizon"] = camera(width, height, e, (cx + 10.0, e[1], cz + size / 4 - 100.0), fov)
    e = (cx, top + 0.3 * size, cz + size / 2)
    out["aerial"] = camera(width, height, e, (cx, top - 0.3 * size, cz - 0.1 * size), fov)
    e = (cx - size / 4, g + 20.0, cz + size / 4)
    out["grazing"] = camera(width, height, e, (e[0] + 30.0, e[1] - 20.0, e[2] - 140.0), fov)
    return out


def settings(t, target_edge_pixels=16.0, max_tessellation=64.0, fov=60.0):
    return abi.terrain_draw_settings(t, target_edge_pixels, max_tessellation, fov)
