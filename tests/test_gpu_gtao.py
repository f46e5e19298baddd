"""The GTAO on the device (oxc_generate_ambient_occlusion, oxr_generate_ambient_occlusion) against the CPU oracle
(oracle/oxc_oracle_gtao.c orc_generate_ambient_occlusion): the depth mips, the edges, the noisy occlusion and the final occlusion
compared bit for bit in every case, plus two checks without the oracle (an all-sky frame, a crease between two planes), and the device
against the binary64 restatement of tests/test_oracle_gtao_f64.py on ray-cast scenes up to 4K."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_vsm_pages import Dev

pytestmark = pytest.mark.gpu

PLANES = ("mips", "edges", "noisy", "ao")


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def go():
    """the GTAO oracle (oracle/pyoracle_gtao.py)"""
    import pyoracle_gtao

    pyoracle_gtao.build()
    return pyoracle_gtao


@pytest.fixture(scope="module")
def ctx(capi):
    sc = synth.make_scene(200, config_index=2, width=64, height=64, n_unique_meshes=4)
    hw, hh = sc.hiz_extent()
    c = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
    yield c
    c.close()


def oct_encode(n):
    """oct(n) of unit vectors [..., 3] (common/encoding.slang:17-21)"""
    p = n[..., :2] / np.abs(n).sum(-1, keepdims=True)
    sgn = np.where(p >= 0, 1.0, -1.0)
    return np.where(n[..., 2:3] <= 0, (1 - np.abs(p[..., ::-1])) * sgn, p).astype(np.float32)


def gtao_camera_for(w, h, yaw=0.0, far=1000.0):
    proj, view = synth.camera_matrices(w, h, yaw, far=far)
    return abi.gtao_camera(proj, view, far), proj


def random_frame(rng, w, h, proj, hostile=True):
    """depth of a few slanted planes and boxes at 1..60 m with a quarter of sky, random unit normals oct-encoded in .zw (random .xy);
    hostile frames add NaN, +-Inf, denormal and negative depths and non-finite normals"""
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    z = 4.0 + 20.0 * (ys / max(h, 1)) + 3.0 * np.sin(xs / 13.0) + 8.0 * ((xs // 37 + ys // 23) % 3 == 0)
    z = z * (1.0 + 0.5 * rng.random((h, w)) * (rng.random((h, w)) < 0.05))
    depth = (proj[14] / z - proj[10]).astype(np.float32)
    depth[rng.random((h, w)) < 0.25] = 0.0
    n = rng.normal(size=(h, w, 3))
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    normals = np.zeros((h, w, 4), np.float32)
    normals[..., :2] = rng.random((h, w, 2))
    normals[..., 2:] = oct_encode(n)
    if hostile:
        k = rng.random((h, w))
        depth[k < 0.01] = np.float32(np.nan)
        depth[(k >= 0.01) & (k < 0.02)] = np.float32(np.inf)
        depth[(k >= 0.02) & (k < 0.03)] = np.float32(-np.inf)
        depth[(k >= 0.03) & (k < 0.04)] = np.float32(1e-40)
        depth[(k >= 0.04) & (k < 0.05)] = np.float32(-0.3)
        m = rng.random((h, w))
        normals[m < 0.01, 2] = np.float32(np.nan)
        normals[(m >= 0.01) & (m < 0.02), 3] = np.float32(np.inf)
        normals[(m >= 0.02) & (m < 0.03), 2:] = np.float32(1e-40)
        normals[(m >= 0.03) & (m < 0.04), 2] = np.float32(70000.0)
    return depth, normals


def random_settings(rng, hostile=False):
    s = abi.GtaoSettings(float(rng.uniform(0.02, 1.5)), int(rng.integers(1, abi.GTAO_MAX_SLICES + 1)),
                         int(rng.integers(1, abi.GTAO_MAX_SAMPLES_PER_SIDE + 1)), float(rng.uniform(0.05, 4.0)),
                         int(rng.integers(0, 2**32)), float(rng.uniform(0.3, 4.0)))
    if hostile:
        s.thickness, s.effect_radius, s.final_power = float("nan"), 1e30, float("nan")
    return s


def run_device(ctx, gcam, settings, depth, normals):
    h, w = depth.shape
    d = Dev(ctx)
    layout, total = abi.gtao_mip_layout(w, h)
    t = {"depth_mips": d.put(np.zeros(total, np.float32)), "edges": d.put(np.zeros((h, w), np.uint32)),
         "noisy_occlusion": d.put(np.zeros((h, w), np.uint16)), "ambient_occlusion": d.put(np.zeros((h, w), np.float32))}
    ctx.generate_ambient_occlusion(gcam, settings, d.put(depth), d.put(normals), w, h, t)
    out = dict(mips=ctx.download(t["depth_mips"], np.float32, total), edges=ctx.download(t["edges"], np.uint32, w * h).reshape(h, w),
               noisy=ctx.download(t["noisy_occlusion"], np.uint16, w * h).reshape(h, w),
               ao=ctx.download(t["ambient_occlusion"], np.float32, w * h).reshape(h, w))
    d.free()
    return out


def assert_planes_equal(got, want, label=""):
    for k in PLANES:
        a, b = np.asarray(got[k]), np.asarray(want[k])
        if a.dtype == np.float32:
            a, b = a.view(np.uint32), b.view(np.uint32)
        bad = np.argwhere(a != b)
        assert bad.size == 0, f"{label} {k}: {len(bad)} texels differ, first at {bad[:3].tolist()}"


SIZES = [(1, 1, 3), (17, 9, 0), (640, 360, 1), (1023, 577, 2), (1920, 1080, 3), (3840, 2160, 0)]


@pytest.mark.parametrize("w,h,preset", SIZES, ids=[f"{w}x{h}" for w, h, _ in SIZES])
def test_sizes_and_presets(ctx, go, w, h, preset):
    """every plane equals the oracle at odd and full sizes, each preset at least once, hostile depth and normals included"""
    rng = np.random.default_rng(w * 7 + h)
    gcam, proj = gtao_camera_for(w, h, yaw=float(w % 90))
    depth, normals = random_frame(rng, w, h, proj)
    settings = abi.gtao_settings(preset)
    want = go.generate_ambient_occlusion(gcam, settings, depth, normals)
    assert_planes_equal(run_device(ctx, gcam, settings, depth, normals), want, f"{w}x{h}")
    if w * h > 1000:
        occluded = (want["ao"] < 0.99).mean()
        assert 0.02 < occluded < 0.98, occluded


@pytest.mark.parametrize("seed", range(4))
def test_random_settings(ctx, go, seed):
    """random thickness, radius, slice and sample counts over their whole accepted range, noise_index and final power; the last seed
    uses NaN thickness and power and a radius of 1e30"""
    rng = np.random.default_rng(100 + seed)
    w, h = (211, 97) if seed % 2 else (160, 120)
    gcam, proj = gtao_camera_for(w, h, yaw=17.0 * seed)
    depth, normals = random_frame(rng, w, h, proj, hostile=seed >= 2)
    settings = random_settings(rng, hostile=seed == 3)
    want = go.generate_ambient_occlusion(gcam, settings, depth, normals)
    assert_planes_equal(run_device(ctx, gcam, settings, depth, normals), want, f"seed {seed}")


def test_all_sky_is_unoccluded(ctx):
    """no oracle: a frame of sky gives exactly 1.0 in the noisy and the final plane"""
    w, h = 97, 45
    gcam, _ = gtao_camera_for(w, h)
    got = run_device(ctx, gcam, abi.gtao_settings(3), np.zeros((h, w), np.float32), np.zeros((h, w, 4), np.float32))
    assert (got["noisy"] == 0x3C00).all() and (got["ao"] == 1.0).all()


def crease_frame(w, h, proj):
    """a floor y = -1 and a wall z = -10 in view space (identity view), meeting in a crease; returns depth, normals, the linear depth,
    and which pixels lie on the wall"""
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    u, v = (xs + 0.5) / w, (ys + 0.5) / h
    ry = (v * 2 - 1) / proj[5]
    t_floor = np.where(ry < 0, -1.0 / np.minimum(ry, -1e-9), np.inf)
    t = np.minimum(t_floor, 10.0)
    wall = t_floor >= 10.0
    depth = (proj[14] / t - proj[10]).astype(np.float32)
    n = np.where(wall[..., None], np.float64([0.0, 0.0, 1.0]), np.float64([0.0, 1.0, 0.0]))
    normals = np.zeros((h, w, 4), np.float32)
    normals[..., 2:] = oct_encode(n)
    return depth, normals, t, wall, ry * t


def test_crease_is_more_occluded(ctx):
    """no oracle: on two perpendicular planes every value lies in [0, 1], and pixels along the crease are more occluded than pixels of
    the same plane far from it"""
    w, h = 640, 360
    proj, _ = synth.camera_matrices(w, h)
    gcam = abi.gtao_camera(proj, np.eye(4, dtype=np.float32).reshape(16), 1000.0)
    depth, normals, t, wall, y_world = crease_frame(w, h, proj)
    got = run_device(ctx, gcam, abi.gtao_settings(3), depth, normals)
    ao = got["ao"]
    assert ((ao >= 0) & (ao <= 1)).all()
    height = y_world + 1.0  # height above the floor on the wall
    near_wall, far_wall = wall & (height < 0.15), wall & (height > 1.5)
    near_floor, far_floor = ~wall & (t > 8.5), ~wall & (t < 5.0)
    assert near_wall.sum() > 500 and far_wall.sum() > 500 and near_floor.sum() > 500 and far_floor.sum() > 500
    assert ao[near_wall].mean() < ao[far_wall].mean() - 0.05, (ao[near_wall].mean(), ao[far_wall].mean())
    assert ao[near_floor].mean() < ao[far_floor].mean() - 0.05, (ao[near_floor].mean(), ao[far_floor].mean())


def test_argument_refusals(capi, ctx):
    d = Dev(ctx)
    buf = d.put(np.zeros(1 << 16, np.uint32))
    gcam, _ = gtao_camera_for(64, 32)
    good = dict(depth_mips=buf, edges=buf, noisy_occlusion=buf, ambient_occlusion=buf)

    def refused(fn, match):
        with pytest.raises(capi.OxcError, match=match) as e:
            fn()
        assert "(-1)" in str(e.value)

    s = abi.gtao_settings(3)
    refused(lambda: ctx.generate_ambient_occlusion(gcam, s, None, buf, 64, 32, good), "null argument")
    refused(lambda: ctx.generate_ambient_occlusion(gcam, s, buf, None, 64, 32, good), "null argument")
    for k in good:
        refused(lambda: ctx.generate_ambient_occlusion(gcam, s, buf, buf, 64, 32, dict(good, **{k: None})), "null target")
    refused(lambda: ctx.generate_ambient_occlusion(gcam, s, buf, buf, 0, 32, good), "empty extent")
    refused(lambda: ctx.generate_ambient_occlusion(gcam, s, buf, buf, 64, 0, good), "empty extent")
    for field, value in (("slice_count", 0), ("slice_count", abi.GTAO_MAX_SLICES + 1), ("samples_per_slice_side", 0),
                         ("samples_per_slice_side", abi.GTAO_MAX_SAMPLES_PER_SIDE + 1)):
        bad = abi.gtao_settings(3)
        setattr(bad, field, value)
        refused(lambda: ctx.generate_ambient_occlusion(gcam, bad, buf, buf, 64, 32, good), field)
    refused(lambda: ctx.generate_ambient_occlusion(gcam, s, buf, buf + 4, 64, 32, good), "16-byte")
    refused(lambda: ctx.generate_ambient_occlusion(gcam, s, buf + 2, buf, 64, 32, good), "4-byte")
    refused(lambda: ctx.generate_ambient_occlusion(gcam, s, buf, buf, 64, 32, dict(good, edges=buf + 2)), "4-byte")
    refused(lambda: ctx.generate_ambient_occlusion(gcam, s, buf, buf, 64, 32, dict(good, noisy_occlusion=buf + 1)), "2-byte")
    d.free()


def test_graph_capture_equals_eager(capi, ctx):
    """the three passes captured into a CUDA graph at their first call and replayed with new depth equal eager runs"""
    import torch

    w, h = 320, 180
    rng = np.random.default_rng(5)
    gcam, proj = gtao_camera_for(w, h)
    depth0, normals = random_frame(rng, w, h, proj, hostile=False)
    depth1 = np.roll(depth0, 11, axis=0)
    settings = abi.gtao_settings(3, noise_index=7)
    eager = [run_device(ctx, gcam, settings, dep, normals) for dep in (depth0, depth1)]
    d = Dev(ctx)
    layout, total = abi.gtao_mip_layout(w, h)
    dep_dev, nrm_dev = d.put(depth0), d.put(normals)
    t = abi.GtaoTargets(d.put(np.zeros(total, np.float32)), d.put(np.zeros((h, w), np.uint32)), d.put(np.zeros((h, w), np.uint16)),
                        d.put(np.zeros((h, w), np.float32)))
    s = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
        gctx.generate_ambient_occlusion(gcam, settings, dep_dev, nrm_dev, w, h, t)
    for k, dep in enumerate((depth0, depth1)):
        ctx.upload(dep_dev, dep)
        g.replay()
        torch.cuda.synchronize()
        got = dict(mips=ctx.download(t.depth_mips, np.float32, total), edges=ctx.download(t.edges, np.uint32, w * h).reshape(h, w),
                   noisy=ctx.download(t.noisy_occlusion, np.uint16, w * h).reshape(h, w),
                   ao=ctx.download(t.ambient_occlusion, np.float32, w * h).reshape(h, w))
        assert_planes_equal(got, eager[k], f"replay {k}")
    assert not np.array_equal(eager[0]["ao"], eager[1]["ao"])
    del g
    d.free()


def test_renderer_frame(capi, go):
    """oxr_generate_ambient_occlusion on a rendered frame (normals from the decode's uv_normal plane) equals the oracle over the
    frame's depth and oxc_decode_gbuffer's normal plane, and the next camera frame equals the one of a renderer without the call"""
    from tests.test_gpu_gbuffer import Table, scene_with_materials

    sc = synth.with_ground_caster(scene_with_materials(20000, 48, 10, config_index=2, width=640, height=360, n_unique_meshes=16),
                                  half_size=1200.0, center=(0.0, -2.0, -40.0))
    sc.mesh_instances["material_index"][-1] = 0
    cam0, cam1 = sc.camera(0.0), sc.camera(1.5)
    gcam, _ = gtao_camera_for(sc.width, sc.height, yaw=0.0)
    settings = abi.gtao_settings(3)
    renderers, tables, last = [capi.Renderer(0, sc), capi.Renderer(0, sc)], [], []
    for k, r in enumerate(renderers):
        tables.append(Table(r.ctx, 10))
        r.set_materials(tables[-1].materials, tables[-1].dev_images, tables[-1].samplers)
        out = r.render(cam0, want_indices=False)
        if k == 0:
            depth = out["depth"].copy()
            got = r.generate_ambient_occlusion(cam0, gcam, settings)
            normal_plane = r.decode_gbuffer(cam0)[1]
            again = r.generate_ambient_occlusion(cam0, gcam, settings)
        o = r.render(cam1)
        last.append((o["vis32"].copy(), o["depth"].copy(), np.sort(o["visible"])))
    for a, b in zip(*last):
        np.testing.assert_array_equal(a, b)
    want = go.generate_ambient_occlusion(gcam, settings, depth, normal_plane)
    np.testing.assert_array_equal(got.view(np.uint32), want["ao"].view(np.uint32))
    np.testing.assert_array_equal(again.view(np.uint32), got.view(np.uint32))
    held = depth != 0
    assert held.mean() > 0.3 and (got[held] < 0.9).sum() > 1000
    for t, r in zip(tables, renderers):
        t.free()
        r.close()


ANALYTIC = [("box", 211, 97, 3), ("turned", 1920, 1080, 2), ("spheres", 1920, 1080, 1), ("corridor", 3840, 2160, 0)]


@pytest.mark.parametrize("name,w,h,preset", ANALYTIC, ids=[f"analytic_{n}_{w}x{h}" for n, w, h, _ in ANALYTIC])
def test_analytic_against_restatement(ctx, name, w, h, preset):
    """every plane of the device agrees with the binary64 restatement on a ray-cast scene, by the rules of test_oracle_gtao_f64"""
    from tests import test_oracle_gtao_f64 as f64

    cam, depth, normals = f64.scene(name, w, h)
    settings = abi.gtao_settings(preset)
    got = run_device(ctx, f64.gtao_camera(cam), settings, depth, normals)
    f64.compare(got, f64.restate(cam, settings, depth, normals), settings, depth, f"{name} {w}x{h}")


def test_renderer_frame_against_restatement(capi):
    """oxr_generate_ambient_occlusion on a rendered frame agrees with the binary64 restatement over the frame's depth and the decode's
    normal plane"""
    from tests import test_oracle_gtao_f64 as f64
    from tests.test_gpu_gbuffer import Table, scene_with_materials

    sc = synth.with_ground_caster(scene_with_materials(20000, 48, 10, config_index=2, width=640, height=360, n_unique_meshes=16),
                                  half_size=1200.0, center=(0.0, -2.0, -40.0))
    sc.mesh_instances["material_index"][-1] = 0
    cam0 = sc.camera(0.0)
    proj, view = synth.camera_matrices(sc.width, sc.height, 0.0)
    cam = f64.camera_dict(proj, view)
    settings = abi.gtao_settings(3)
    r = capi.Renderer(0, sc)
    table = Table(r.ctx, 10)
    r.set_materials(table.materials, table.dev_images, table.samplers)
    depth = r.render(cam0, want_indices=False)["depth"].copy()
    got = r.generate_ambient_occlusion(cam0, f64.gtao_camera(cam), settings)
    normal_plane = r.decode_gbuffer(cam0)[1]
    zw = normal_plane[..., 2:4]
    finite = np.isfinite(zw).all(-1)
    # the ground's normals are NaN (the NaN rules decide its occlusion) and some of the others are not binary16-exact
    assert (~finite).mean() > 0.2 and (zw.astype(np.float16).astype(np.float32) != zw).any(-1)[finite].mean() > 0.01
    stats = f64.compare(dict(ao=got), f64.restate(cam, settings, depth, normal_plane), settings, depth, "renderer frame")
    print("renderer frame", stats)
    held = depth != 0
    assert held.mean() > 0.3 and (got[held] < 0.9).sum() > 1000
    table.free()
    r.close()
