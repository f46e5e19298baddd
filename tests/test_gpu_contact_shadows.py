"""The contact-shadow pass on the device (oxc_contact_shadows, oxr_contact_shadows, oxr_apply_pbr_with_contact_shadows) against the CPU
oracle (oracle/oxc_oracle_contact_shadows.c orc_contact_shadows), bit for bit in every case: sizes from 1 x 1 to 4K, random and hostile
depth and settings, steps 1 / 2 / 8 / 64, refusals, graph capture, the renderer's pass and its lit frame against the oracle chain; plus
one check without the oracle (contact on the casters of the ground-caster frame, none on open ground)."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_vsm_pages import Dev

pytestmark = pytest.mark.gpu

NEAR = 0.1


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def co():
    """the contact-shadow oracle (oracle/pyoracle_contact_shadows.py)"""
    import pyoracle_contact_shadows

    pyoracle_contact_shadows.build()
    return pyoracle_contact_shadows


@pytest.fixture(scope="module")
def ctx(capi):
    sc = synth.make_scene(200, config_index=2, width=64, height=64, n_unique_meshes=4)
    hw, hh = sc.hiz_extent()
    c = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
    yield c
    c.close()


def contact_camera_for(w, h, yaw=0.0, eye=(0.0, 0.0, 0.0), near=NEAR):
    """(abi.ContactShadowCamera, projection) of a make_camera camera: the binary64 inverse of its projection_view rounded to binary32"""
    proj, view = synth.camera_matrices(w, h, yaw, eye=eye, near=near)
    pv = synth.mat_mul_cm(proj, view)
    inv = np.linalg.inv(pv.reshape(4, 4).T.astype(np.float64)).T.astype(np.float32).reshape(16)
    return abi.contact_shadow_camera(inv, view, proj, near), proj


def random_depth(rng, w, h, proj, hostile=True):
    """reversed-Z depth of slanted planes and boxes at 2..40 m with steps between them and a quarter of sky; hostile frames add NaN,
    +-Inf, denormal and negative depths"""
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    z = 2.0 + 30.0 * (ys / max(h, 1)) + 2.0 * np.sin(xs / 11.0) + 3.0 * ((xs // 31 + ys // 19) % 3 == 0)
    z = z * (1.0 + 0.3 * rng.random((h, w)) * (rng.random((h, w)) < 0.05))
    depth = (proj[14] / z - proj[10]).astype(np.float32)
    depth[rng.random((h, w)) < 0.25] = 0.0
    if hostile:
        k = rng.random((h, w))
        depth[k < 0.01] = np.float32(np.nan)
        depth[(k >= 0.01) & (k < 0.02)] = np.float32(np.inf)
        depth[(k >= 0.02) & (k < 0.03)] = np.float32(-np.inf)
        depth[(k >= 0.03) & (k < 0.04)] = np.float32(1e-40)
        depth[(k >= 0.04) & (k < 0.05)] = np.float32(-0.3)
    return depth


def random_settings(rng, steps=None, hostile=False):
    """a random sun, ray length 0.05..3 m and thickness 0.02..1; hostile: NaN thickness, infinite length and a zero sun in turn"""
    s = abi.contact_shadow_settings(rng.normal(size=3), int(rng.integers(1, abi.CONTACT_SHADOW_MAX_STEPS + 1)) if steps is None else steps,
                                    float(rng.uniform(0.02, 1.0)), float(rng.uniform(0.05, 3.0)))
    if hostile:
        k = int(rng.integers(0, 3))
        if k == 0:
            s.thickness = float("nan")
        elif k == 1:
            s.length = float("inf")
        else:
            s.sun_direction[:] = [0.0, 0.0, 0.0]
    return s


def box_on_plane(w, h, box=True):
    """reversed-Z depth of a ground plane y = -1 and (box) a box [-1, 1] x [-1, 0.5] x [-9, -7], ray-cast in binary64 from the origin
    (identity view), with sky above the horizon; returns depth, the ground mask and the world x / z of every pixel"""
    proj, view = synth.camera_matrices(w, h)
    inv = np.linalg.inv(synth.mat_mul_cm(proj, view).reshape(4, 4).T.astype(np.float64))
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    cx, cy = (xs + 0.5) / w * 2 - 1, (ys + 0.5) / h * 2 - 1
    far = inv @ np.stack([cx, cy, np.full_like(cx, 0.5), np.ones_like(cx)]).reshape(4, -1)
    d = (far[:3] / far[3]).T.reshape(h, w, 3)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        t_ground = np.where(d[..., 1] < 0, -1.0 / d[..., 1], np.inf)
        lo, hi = np.float64([-1.0, -1.0, -9.0]), np.float64([1.0, 0.5, -7.0])
        t1, t2 = lo / d, hi / d
        tn = np.nanmax(np.minimum(t1, t2), axis=-1)
        tf = np.nanmin(np.maximum(t1, t2), axis=-1)
    t_box = np.where((tn <= tf) & (tf > 0) & box, tn, np.inf)
    t = np.minimum(t_ground, t_box)
    p = d * t[..., None]
    zv = -p[..., 2]  # the view is the identity
    depth = np.where(np.isfinite(t), proj[14] / np.where(np.isfinite(t), zv, 1.0) - proj[10], 0.0).astype(np.float32)
    ground = np.isfinite(t_ground) & (t_ground < t_box)
    return depth, ground, p[..., 0], p[..., 2]


def run_device(ctx, ccam, settings, depth):
    h, w = depth.shape
    d = Dev(ctx)
    out = d.put(np.zeros((h, w), np.float32))
    ctx.contact_shadows(ccam, settings, d.put(depth), w, h, out)
    got = ctx.download(out, np.float32, w * h).reshape(h, w)
    d.free()
    return got


def assert_equal(got, want, label=""):
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, f"{label}: {len(bad)} pixels differ, first at {bad[:3].tolist()}"


SIZES = [(1, 1, 1), (17, 9, 2), (640, 360, 8), (1920, 1080, 64), (3840, 2160, 8)]


@pytest.mark.parametrize("w,h,steps", SIZES, ids=[f"{w}x{h}" for w, h, _ in SIZES])
@pytest.mark.parametrize("hostile", [False, True], ids=["random", "hostile"])
def test_sizes(ctx, co, w, h, steps, hostile):
    """the device equals the oracle on every pixel, random and hostile depth and settings"""
    rng = np.random.default_rng(w * 7 + h + hostile)
    ccam, proj = contact_camera_for(w, h, yaw=float(w % 90))
    depth = random_depth(rng, w, h, proj, hostile=hostile)
    settings = random_settings(rng, steps=steps, hostile=hostile and w > 1)
    want = co.contact_shadows(ccam, settings, depth)
    assert_equal(run_device(ctx, ccam, settings, depth), want, f"{w}x{h}")
    assert ((want >= 0) & (want <= 1)).all()
    if w * h > 1000 and not hostile:
        assert 0.005 < (want < 1).mean() < 0.9, (want < 1).mean()


@pytest.mark.parametrize("steps", [1, 2, 8, 64])
def test_steps(ctx, co, steps):
    """each step count on a 211 x 97 frame, with the reference's defaults and a longer ray"""
    rng = np.random.default_rng(40 + steps)
    ccam, proj = contact_camera_for(211, 97, yaw=11.0)
    depth = random_depth(rng, 211, 97, proj, hostile=False)
    for settings in (abi.contact_shadow_settings(steps=steps), abi.contact_shadow_settings((0.5, 0.6, -0.2), steps, 0.3, 2.0)):
        assert_equal(run_device(ctx, ccam, settings, depth), co.contact_shadows(ccam, settings, depth), f"steps {steps}")


@pytest.mark.parametrize("seed", range(4))
def test_random_settings(ctx, co, seed):
    """random settings over the whole accepted range, on random frames; the odd seeds with hostile depth and settings"""
    rng = np.random.default_rng(100 + seed)
    w, h = (211, 97) if seed % 2 else (160, 120)
    ccam, proj = contact_camera_for(w, h, yaw=17.0 * seed)
    depth = random_depth(rng, w, h, proj, hostile=seed % 2 == 1)
    settings = random_settings(rng, hostile=seed % 2 == 1)
    assert_equal(run_device(ctx, ccam, settings, depth), co.contact_shadows(ccam, settings, depth), f"seed {seed}")


def test_box_on_plane(ctx, co):
    """the analytic box on a plane with a grazing sun behind it: the device equals the oracle, the ground next to the box's base on the
    side away from the sun is in contact and open ground far from the box is exactly 1"""
    w, h = 640, 360
    ccam, _ = contact_camera_for(w, h)
    depth, ground, x, z = box_on_plane(w, h)
    settings = abi.contact_shadow_settings((0.3, 0.2, -1.0), 16, 0.1, 1.0)
    got = run_device(ctx, ccam, settings, depth)
    assert_equal(got, co.contact_shadows(ccam, settings, depth), "box")
    base = ground & (np.abs(x) < 0.9) & (z > -7.0) & (z < -6.8)
    open_ground = ground & ((np.abs(x) > 4.0) | (z > -5.0))
    assert base.sum() > 50 and (got[base] < 1).all()
    assert open_ground.sum() > 10000 and (got[open_ground] == 1).all()


def test_argument_refusals(capi, ctx):
    d = Dev(ctx)
    buf = d.put(np.zeros(1 << 14, np.float32))
    ccam, _ = contact_camera_for(64, 32)
    s = abi.contact_shadow_settings()

    def refused(fn, match):
        with pytest.raises(capi.OxcError, match=match) as e:
            fn()
        assert "(-1)" in str(e.value)

    launches = capi.kernel_launch_count()
    refused(lambda: ctx.contact_shadows(ccam, s, None, 64, 32, buf), "null argument")
    refused(lambda: ctx.contact_shadows(ccam, s, buf, 64, 32, None), "null argument")
    refused(lambda: ctx.contact_shadows(ccam, s, buf, 0, 32, buf), "empty extent")
    refused(lambda: ctx.contact_shadows(ccam, s, buf, 64, 0, buf), "empty extent")
    refused(lambda: ctx.contact_shadows(ccam, s, buf, 32769, 1, buf), "above 32768")
    refused(lambda: ctx.contact_shadows(ccam, s, buf, 1, 32769, buf), "above 32768")
    for steps in (0, abi.CONTACT_SHADOW_MAX_STEPS + 1, 2**32 - 1):
        refused(lambda: ctx.contact_shadows(ccam, abi.contact_shadow_settings(steps=steps), buf, 64, 32, buf), "steps")
    refused(lambda: ctx.contact_shadows(ccam, s, buf + 2, 64, 32, buf), "4-byte")
    refused(lambda: ctx.contact_shadows(ccam, s, buf, 64, 32, buf + 1), "4-byte")
    assert capi.kernel_launch_count() == launches
    d.free()


def test_graph_capture_equals_eager(capi, ctx, co):
    """the pass captured into a CUDA graph at its first call and replayed with new depth equals eager runs and the oracle"""
    import torch

    w, h = 320, 180
    rng = np.random.default_rng(5)
    ccam, proj = contact_camera_for(w, h)
    depth0 = random_depth(rng, w, h, proj, hostile=False)
    depth1 = np.roll(depth0, 11, axis=0)
    settings = abi.contact_shadow_settings((0.2, 0.9, 0.3), 8, 0.2, 1.5)
    eager = [run_device(ctx, ccam, settings, dep) for dep in (depth0, depth1)]
    d = Dev(ctx)
    dep_dev, out = d.put(depth0), d.put(np.zeros((h, w), np.float32))
    s = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
        gctx.contact_shadows(ccam, settings, dep_dev, w, h, out)
    for k, dep in enumerate((depth0, depth1)):
        ctx.upload(dep_dev, dep)
        g.replay()
        torch.cuda.synchronize()
        assert_equal(ctx.download(out, np.float32, w * h).reshape(h, w), eager[k], f"replay {k}")
    assert not np.array_equal(eager[0], eager[1])
    assert_equal(eager[1], co.contact_shadows(ccam, settings, depth1), "eager vs oracle")
    del g
    d.free()


def ground_caster_scene():
    from tests.test_gpu_gbuffer import scene_with_materials

    sc = synth.with_ground_caster(scene_with_materials(20000, 48, 10, config_index=2, width=640, height=360, n_unique_meshes=16),
                                  half_size=1200.0, center=(0.0, -2.0, -40.0))
    sc.mesh_instances["material_index"][-1] = 0
    return sc


SUN = (0.2, 0.3, -1.0)  # a low sun behind the casters, so their contact shadows fall on the ground in front of them


def test_renderer_contact_shadows(capi, co):
    """oxr_contact_shadows on a rendered frame of the ground-caster scene equals the oracle over that frame's depth, twice; the next
    camera frame equals the one of a renderer without the call.  Without the oracle: contact < 1 on the casters, 1 on open ground"""
    sc = ground_caster_scene()
    cam0, cam1 = sc.camera(0.0), sc.camera(1.5)
    ccam, _ = contact_camera_for(sc.width, sc.height)
    settings = abi.contact_shadow_settings(SUN, 16, 0.1, 0.5)
    renderers, last = [capi.Renderer(0, sc), capi.Renderer(0, sc)], []
    for k, r in enumerate(renderers):
        out = r.render(cam0, want_indices=False)
        if k == 0:
            depth = out["depth"].copy()
            got = r.contact_shadows(ccam, settings)
            again = r.contact_shadows(ccam, settings)
        o = r.render(cam1)
        last.append((o["vis32"].copy(), o["depth"].copy(), np.sort(o["visible"])))
    for a, b in zip(*last):
        np.testing.assert_array_equal(a, b)
    assert_equal(got, co.contact_shadows(ccam, settings, depth), "renderer frame")
    assert_equal(again, got, "second call")
    # the ground: pixels whose depth is the plane y = -2 of the ground caster; the casters: every other pixel holding depth.  The
    # scene's instances float above the ground, so their contact shadows fall on themselves (faces turned away from the sun), not on
    # the ground; open ground away from them stays at 1 (measured on the oracle's frame: 781 caster pixels in contact, 18 of 103,956
    # open-ground pixels)
    proj, _ = synth.camera_matrices(sc.width, sc.height)
    ys = (np.arange(sc.height) + 0.5) / sc.height * 2 - 1
    with np.errstate(divide="ignore"):
        zlin = proj[14] / (depth.astype(np.float64) + proj[10])
    plane = np.abs(zlin * (ys / proj[5])[:, None] + 2.0) < 0.02 * zlin
    caster = (depth != 0) & ~plane
    grow = caster.copy()
    for _ in range(6):
        grow = grow | np.roll(grow, 1, 0) | np.roll(grow, -1, 0) | np.roll(grow, 1, 1) | np.roll(grow, -1, 1)
    open_ground = plane & ~grow
    assert open_ground.sum() > 50000 and (got[caster] < 1).sum() > 100, (open_ground.sum(), (got[caster] < 1).sum())
    assert (got[open_ground] == 1).mean() > 0.999, (got[open_ground] == 1).mean()
    for r in renderers:
        r.close()


def test_renderer_apply_pbr_with_contact_shadows(capi, co):
    """oxr_apply_pbr_with_contact_shadows under HasContactShadows equals orc_apply_pbr fed with the oracle's contact plane (over
    oxr_decode_gbuffer's planes and the oracle GTAO), and the same oxc_* calls made by hand on the renderer's outputs; without the flag
    it equals oxr_apply_pbr; oxr_apply_pbr still refuses the flag; the next camera frame is unchanged"""
    import pyoracle_gtao
    import pyoracle_pbr

    from tests.test_gpu_gbuffer import Table
    from tests.test_gpu_gtao import gtao_camera_for
    from tests.test_gpu_pbr import assert_equal as pbr_equal
    from tests.test_gpu_pbr import run_device as pbr_device
    from tests.test_gpu_pbr import settings_for

    pyoracle_gtao.build()
    pyoracle_pbr.build()
    sc = ground_caster_scene()
    cam0, cam1 = sc.camera(0.0), sc.camera(1.5)
    ccam, _ = contact_camera_for(sc.width, sc.height)
    cset = abi.contact_shadow_settings(SUN, 8, 0.1, 0.5)
    gcam, _ = gtao_camera_for(sc.width, sc.height, yaw=0.0)
    gset = abi.gtao_settings(2)
    lights = synth.make_lights(np.random.default_rng(3), 8, eye=(0.0, -1.0, 0.0))
    # the contact plane darkens the sun's term, which HasDirectionalLight switches on (without cast_shadows the shadow reads 1)
    flags = abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_GTAO | abi.SCENE_HAS_CONTACT_SHADOWS
    settings = settings_for(flags, len(lights))
    settings.sun_direction[:] = list(SUN)
    plain = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_GTAO, len(lights))
    plain.sun_direction[:] = list(SUN)
    pcam = synth.pbr_camera(cam0)
    renderers, tables, last = [capi.Renderer(0, sc), capi.Renderer(0, sc)], [], []
    for k, r in enumerate(renderers):
        tables.append(Table(r.ctx, 10))
        r.set_materials(tables[-1].materials, tables[-1].dev_images, tables[-1].samplers)
        out = r.render(cam0, want_indices=False)
        if k == 0:
            depth = out["depth"].copy()
            got = r.apply_pbr(cam0, settings, lights, gtao_camera=gcam, gtao_settings=gset, contact_camera=ccam, contact_settings=cset)
            without = r.apply_pbr(cam0, plain, lights, gtao_camera=gcam, gtao_settings=gset, contact_camera=ccam, contact_settings=cset)
            reference = r.apply_pbr(cam0, plain, lights, gtao_camera=gcam, gtao_settings=gset)
            with pytest.raises(capi.OxcError, match="oxr_apply_pbr"):
                r.apply_pbr(cam0, settings, lights, gtao_camera=gcam, gtao_settings=gset)
            for cc, cs in ((ccam, None), (None, cset), (ccam, abi.contact_shadow_settings(steps=0))):
                with pytest.raises(capi.OxcError, match="with_contact_shadows"):
                    r.apply_pbr(cam0, settings, lights, gtao_camera=gcam, gtao_settings=gset, contact_camera=cc, contact_settings=cs)
            gb = r.decode_gbuffer(cam0)
            ao_r = r.generate_ambient_occlusion(cam0, gcam, gset)
            contact_r = r.contact_shadows(ccam, cset)
        o = r.render(cam1)
        last.append((o["vis32"].copy(), o["depth"].copy(), np.sort(o["visible"])))
    for a, b in zip(*last):
        np.testing.assert_array_equal(a, b)
    contact = co.contact_shadows(ccam, cset, depth)
    assert_equal(contact_r, contact, "contact plane")
    ao = pyoracle_gtao.generate_ambient_occlusion(gcam, gset, depth, gb[1])["ao"]
    planes = dict(depth=depth, albedo=gb[0], normal=gb[1], emissive=gb[2], metallic_roughness_occlusion=gb[3])
    want = pyoracle_pbr.apply_pbr(pcam, settings, lights, depth, gb[0], gb[1], gb[2], gb[3], ao, None, contact)
    pbr_equal(got, want, "oracle chain")
    pbr_equal(without, reference, "without the flag")
    by_hand = pbr_device(renderers[0].ctx, pcam, settings, lights, dict(planes, ambient_occlusion=ao_r, shadow=None, contact_shadow=contact_r),
                         omit=("shadow",))
    pbr_equal(by_hand, got, "composed by hand")
    held = depth != 0
    # most contact falls on faces turned away from the sun, whose sun term is already 0 (measured: 310 pixels in contact, 26 changed)
    assert (contact[held] < 1).sum() > 100 and (np.abs(got - without).sum(-1) > 0).sum() > 10
    for t, r in zip(tables, renderers):
        t.free()
        r.close()
