"""PBR apply on the device (oxc_apply_pbr, oxr_apply_pbr) against the CPU oracle (oracle/oxc_oracle_pbr.c orc_apply_pbr), bit for bit
in every case: sizes from 1 x 1 to 4K, random planes with 0 / 1 / 256 mixed lights, every subset of the flags the pass reads, NULL
optional planes, hostile planes and lights, refusals, graph capture and the renderer chain; plus checks without the oracle (emissive
only, lights out of range, sky and transparent pixels)."""
import itertools

import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_gtao import oct_encode
from tests.test_gpu_vsm_pages import Dev

pytestmark = pytest.mark.gpu

FLAGS = (abi.SCENE_HAS_DIRECTIONAL_LIGHT, abi.SCENE_HAS_CONTACT_SHADOWS, abi.SCENE_HAS_SKY, abi.SCENE_TRANSPARENT_BACKGROUND)
OPTIONAL = ("ambient_occlusion", "shadow", "contact_shadow")


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def po():
    """the PBR oracle (oracle/pyoracle_pbr.py)"""
    import pyoracle_pbr

    pyoracle_pbr.build()
    return pyoracle_pbr


@pytest.fixture(scope="module")
def ctx(capi):
    sc = synth.make_scene(200, config_index=2, width=64, height=64, n_unique_meshes=4)
    hw, hh = sc.hiz_extent()
    c = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
    yield c
    c.close()


def mixed_lights(rng, n, hostile=False):
    """synth.make_lights plus, when n > 2, a directional and an unknown kind among them; hostile lights get NaN / Inf / denormal /
    negative fields"""
    lights = synth.make_lights(rng, n)
    if n > 2:
        lights[1].kind = abi.LIGHT_DIRECTIONAL
        lights[2].kind = 7
    if hostile:
        for i in range(0, n, 3):
            L = lights[i]
            field = i // 3 % 6
            if field == 0:
                L.range = float("nan")
            elif field == 1:
                L.intensity = float("inf")
            elif field == 2:
                L.position[0] = float("nan")
            elif field == 3:
                L.inner_cone_angle, L.outer_cone_angle = 0.4, 0.4
            elif field == 4:
                L.direction[:] = [0.0, 0.0, 0.0]
            else:
                L.range, L.color[1] = -3.0, 1e-40
    return lights


def random_planes(rng, w, h, yaw=0.0, hostile=False):
    """(pbr camera, planes) of a w x h frame: depth of slanted planes at 3..60 m with a quarter of sky, random albedo, oct-encoded
    random normals in .xy and nearby smooth normals in .zw, sparse emissive, metallic / roughness slightly beyond [0, 1], ambient
    occlusion, shadow and contact factors; hostile frames add NaN / Inf / denormal values to every plane"""
    cam = synth.make_camera(w, h, 1, yaw)
    proj, _ = synth.camera_matrices(w, h, yaw)
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    z = 3.0 + 50.0 * (ys / max(h, 1)) ** 2 + 4.0 * np.sin(xs / 17.0) + 6.0 * ((xs // 29 + ys // 19) % 3 == 0)
    depth = (proj[14] / z - proj[10]).astype(np.float32)
    depth[rng.random((h, w)) < 0.25] = 0.0
    n = rng.normal(size=(h, w, 3)) + (0.0, 1.5, 0.0)
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    s = n + rng.normal(scale=0.2, size=(h, w, 3))
    s /= np.linalg.norm(s, axis=-1, keepdims=True)
    normal = np.concatenate([oct_encode(n), oct_encode(s)], -1).astype(np.float32)
    planes = dict(depth=depth, albedo=rng.random((h, w, 4)).astype(np.float32), normal=normal,
                  emissive=(rng.random((h, w, 4)) * (rng.random((h, w, 1)) < 0.1)).astype(np.float32),
                  metallic_roughness_occlusion=rng.uniform(-0.1, 1.1, (h, w, 4)).astype(np.float32),
                  ambient_occlusion=rng.random((h, w)).astype(np.float32), shadow=np.where(rng.random((h, w)) < 0.3, 0.0, rng.random((h, w))).astype(np.float32),
                  contact_shadow=rng.random((h, w)).astype(np.float32))
    if hostile:
        bad = np.float32([np.nan, np.inf, -np.inf, 1e-40, -1e-40, 70000.0, -2.0])
        for k, a in planes.items():
            m = rng.random(a.shape) < 0.02
            a[m] = rng.choice(bad, int(m.sum()))
    return synth.pbr_camera(cam), planes


def settings_for(flags, n_lights, rng=None):
    s = abi.pbr_settings(scene_flags=flags, sun_direction=(0.35, 0.8, 0.48), sun_intensity=7.5, sky_solid_color=(0.2, 0.4, 0.9, 1.0),
                         sky_ambient_color=(0.05, 0.07, 0.1), light_count=n_lights)
    if rng is not None:
        s.sun_direction[:] = [float(np.float32(v)) for v in rng.normal(size=3)]
        s.sun_intensity = float(np.float32(rng.uniform(0.0, 20.0)))
    return s


def run_device(ctx, pcam, settings, lights, planes, omit=()):
    h, w = planes["depth"].shape
    d = Dev(ctx)
    inputs = {k: (None if k in omit else d.put(v)) for k, v in planes.items()}
    ldev = d.put(np.frombuffer(bytes(lights), np.uint8)) if lights is not None and len(lights) else None
    out = d.put(np.zeros((h, w, 4), np.float32))
    ctx.apply_pbr(pcam, settings, ldev, inputs, w, h, out)
    got = ctx.download(out, np.float32, w * h * 4).reshape(h, w, 4)
    d.free()
    return got


def oracle(po, pcam, settings, lights, planes, omit=()):
    p = {k: (None if k in omit else v) for k, v in planes.items()}
    return po.apply_pbr(pcam, settings, lights, p["depth"], p["albedo"], p["normal"], p["emissive"], p["metallic_roughness_occlusion"],
                        p["ambient_occlusion"], p["shadow"], p["contact_shadow"])


def assert_equal(got, want, label=""):
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, f"{label}: {len(bad)} values differ, first at {bad[:3].tolist()}"


SIZES = [(1, 1, 1), (17, 9, 17), (640, 360, 256), (1920, 1080, 64), (3840, 2160, 16)]


@pytest.mark.parametrize("w,h,n", SIZES, ids=[f"{w}x{h}" for w, h, _ in SIZES])
def test_sizes(ctx, po, w, h, n):
    """every pixel equals the oracle at odd and full sizes, directional light, GTAO plane and lights"""
    rng = np.random.default_rng(w * 3 + h)
    pcam, planes = random_planes(rng, w, h, yaw=float(w % 50))
    lights = mixed_lights(rng, n)
    s = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_GTAO, n)
    want = oracle(po, pcam, s, lights, planes)
    assert_equal(run_device(ctx, pcam, s, lights, planes), want, f"{w}x{h}")
    if w * h > 1000:
        lit = want[..., :3].sum(-1)
        assert np.isfinite(lit).mean() > 0.5 and (lit > 0.1).mean() > 0.2


@pytest.mark.parametrize("n", [0, 1, 256])
@pytest.mark.parametrize("flags", range(16), ids=[f"flags{k}" for k in range(16)])
def test_flag_subsets(ctx, po, flags, n):
    """every subset of HasDirectionalLight / HasContactShadows / HasSky / TransparentBackground with 0, 1 and 256 mixed lights, plus
    bits the pass ignores (bloom, FXAA, ...)"""
    rng = np.random.default_rng(1000 + flags * 7 + n)
    w, h = 61, 37
    pcam, planes = random_planes(rng, w, h, yaw=5.0 * flags)
    lights = mixed_lights(rng, n)
    f = sum(b for k, b in enumerate(FLAGS) if flags >> k & 1) | abi.SCENE_HAS_BLOOM | abi.SCENE_HAS_FXAA | abi.SCENE_HAS_VIGNETTE
    s = settings_for(f, n, rng)
    s.sky_has_texture = flags % 3 == 0
    assert_equal(run_device(ctx, pcam, s, lights, planes), oracle(po, pcam, s, lights, planes), f"flags {f:#x}")


@pytest.mark.parametrize("omit", [(), ("ambient_occlusion",), ("shadow",), ("ambient_occlusion", "shadow"), ("contact_shadow",)])
def test_null_optional_planes(ctx, po, omit):
    """NULL ambient occlusion and shadow read as 1.0; the contact plane may be NULL without HasContactShadows"""
    rng = np.random.default_rng(77 + len(omit))
    pcam, planes = random_planes(rng, 97, 45)
    lights = mixed_lights(rng, 9)
    s = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_GTAO, 9)
    assert_equal(run_device(ctx, pcam, s, lights, planes, omit), oracle(po, pcam, s, lights, planes, omit), str(omit))


@pytest.mark.parametrize("seed", range(3))
def test_hostile(ctx, po, seed):
    """NaN / Inf / denormal values in every plane and in light fields, random sun and flags: the same bits as the oracle"""
    rng = np.random.default_rng(500 + seed)
    pcam, planes = random_planes(rng, 123, 77, hostile=True)
    n = (5, 64, 256)[seed]
    lights = mixed_lights(rng, n, hostile=True)
    s = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_CONTACT_SHADOWS * (seed % 2) | abi.SCENE_HAS_SKY * (seed == 2), n, rng)
    s.sky_solid_color[1] = float("nan")
    got = run_device(ctx, pcam, s, lights, planes)
    assert_equal(got, oracle(po, pcam, s, lights, planes), f"seed {seed}")
    nan = got.view(np.uint32)[np.isnan(got)]
    assert (nan == 0x7FFFFFFF).all() and nan.size > 0


def test_emissive_only(ctx):
    """no oracle: with Li = 0, no lights and zero ambient, rgb equals the emissive plane bit for bit and alpha is 1"""
    rng = np.random.default_rng(3)
    pcam, planes = random_planes(rng, 160, 90)
    s = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT, 0)
    s.sun_intensity = 0.0
    s.base_ambient_color[:] = [0.0, 0.0, 0.0]
    got = run_device(ctx, pcam, s, None, planes)
    held = planes["depth"] != 0
    assert_equal(got[held][:, :3], planes["emissive"][held][:, :3], "emissive")
    assert (got[..., 3] == 1.0).all()


def test_lights_out_of_range(ctx):
    """no oracle: pixels beyond every light's range equal the frame without lights bit for bit, and the lights change the others"""
    rng = np.random.default_rng(4)
    w, h = 320, 180
    pcam, planes = random_planes(rng, w, h)
    lights = synth.make_lights(rng, 24, radius=(1.0, 6.0))
    s0, s1 = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT, 0), settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT, len(lights))
    base, lit = run_device(ctx, pcam, s0, None, planes), run_device(ctx, pcam, s1, lights, planes)
    inv = np.asarray(pcam.inv_projection_view, np.float64).reshape(4, 4).T
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    ndc = np.stack([(xs + 0.5) / w * 2 - 1, (ys + 0.5) / h * 2 - 1, planes["depth"], np.ones((h, w))], -1) @ inv.T
    world = ndc[..., :3] / ndc[..., 3:]
    far = np.ones((h, w), bool)
    for L in lights:
        far &= np.linalg.norm(world - np.asarray(L.position[:]), axis=-1) > L.range * 1.001
    far &= planes["depth"] != 0
    assert far.sum() > 1000 and (~far).sum() > 1000
    assert_equal(lit[far], base[far], "beyond range")
    assert (lit[~far & (planes["depth"] != 0)] != base[~far & (planes["depth"] != 0)]).any()


def test_sky_and_transparent_pixels(ctx):
    """no oracle: HasSky sky pixels hold solid_color (or 1 with a sky texture), TransparentBackground sky pixels hold 0 and win over
    HasSky; pixels holding depth are lit"""
    rng = np.random.default_rng(5)
    pcam, planes = random_planes(rng, 96, 64)
    sky = planes["depth"] == 0
    for flags, tex, want in ((abi.SCENE_HAS_SKY, False, (0.2, 0.4, 0.9, 1.0)), (abi.SCENE_HAS_SKY, True, (1.0, 1.0, 1.0, 1.0)),
                             (abi.SCENE_TRANSPARENT_BACKGROUND, False, (0.0, 0.0, 0.0, 0.0)),
                             (abi.SCENE_TRANSPARENT_BACKGROUND | abi.SCENE_HAS_SKY, True, (0.0, 0.0, 0.0, 0.0))):
        s = settings_for(flags | abi.SCENE_HAS_DIRECTIONAL_LIGHT, 0)
        s.sky_has_texture = tex
        got = run_device(ctx, pcam, s, None, planes)
        assert_equal(got[sky], np.broadcast_to(np.float32(want), got[sky].shape).copy(), f"flags {flags:#x}")
        assert (got[~sky][:, 3] == 1.0).all()


def test_argument_refusals(capi, ctx):
    d = Dev(ctx)
    buf = d.put(np.zeros(1 << 16, np.uint32))
    pcam = synth.pbr_camera(synth.make_camera(64, 32, 1))
    good = {k: buf for k in abi.PBR_INPUTS}
    s = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT, 4)

    def refused(fn, match):
        with pytest.raises(capi.OxcError, match=match) as e:
            fn()
        assert "(-1)" in str(e.value)

    for k in ("depth", "albedo", "normal", "emissive", "metallic_roughness_occlusion"):
        refused(lambda: ctx.apply_pbr(pcam, s, buf, dict(good, **{k: None}), 64, 32, buf), "null input plane")
    refused(lambda: ctx.apply_pbr(pcam, s, buf, good, 64, 32, None), "null argument")
    refused(lambda: ctx.apply_pbr(pcam, s, None, good, 64, 32, buf), "null lights")
    sc = settings_for(abi.SCENE_HAS_CONTACT_SHADOWS, 0)
    refused(lambda: ctx.apply_pbr(pcam, sc, None, dict(good, contact_shadow=None), 64, 32, buf), "contact_shadow")
    refused(lambda: ctx.apply_pbr(pcam, s, buf, good, 0, 32, buf), "empty extent")
    refused(lambda: ctx.apply_pbr(pcam, s, buf, good, 64, 0, buf), "empty extent")
    refused(lambda: ctx.apply_pbr(pcam, s, buf, good, 32769, 1, buf), "above 32768")
    many = settings_for(0, abi.MAX_LIGHTS + 1)
    refused(lambda: ctx.apply_pbr(pcam, many, buf, good, 64, 32, buf), "light_count")
    atm = settings_for(abi.SCENE_HAS_ATMOSPHERE, 0)
    refused(lambda: ctx.apply_pbr(pcam, atm, None, good, 64, 32, buf), "HasAtmosphere")
    for k in ("albedo", "normal", "emissive", "metallic_roughness_occlusion"):
        refused(lambda: ctx.apply_pbr(pcam, s, buf, dict(good, **{k: buf + 4}), 64, 32, buf), "16-byte")
    refused(lambda: ctx.apply_pbr(pcam, s, buf, good, 64, 32, buf + 8), "16-byte")
    refused(lambda: ctx.apply_pbr(pcam, s, buf + 4, good, 64, 32, buf), "16-byte")
    for k in ("depth", "ambient_occlusion", "shadow", "contact_shadow"):
        refused(lambda: ctx.apply_pbr(pcam, s, buf, dict(good, **{k: buf + 2}), 64, 32, buf), "4-byte")
    d.free()


def test_graph_capture_equals_eager(capi, ctx, po):
    """the pass captured into a CUDA graph at its first call and replayed with new planes and lights equals eager runs"""
    import torch

    w, h = 320, 180
    rng = np.random.default_rng(6)
    pcam, p0 = random_planes(rng, w, h)
    _, p1 = random_planes(rng, w, h, yaw=3.0)
    l0, l1 = mixed_lights(rng, 32), mixed_lights(rng, 32)
    s = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_GTAO, 32)
    eager = [run_device(ctx, pcam, s, lt, pl) for pl, lt in ((p0, l0), (p1, l1))]
    d = Dev(ctx)
    inputs = {k: d.put(v) for k, v in p0.items()}
    ldev = d.put(np.frombuffer(bytes(l0), np.uint8))
    out = d.put(np.zeros((h, w, 4), np.float32))
    st = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=st.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st, capture_error_mode="thread_local"):
        gctx.apply_pbr(pcam, s, ldev, inputs, w, h, out)
    for k, (pl, lt) in enumerate(((p0, l0), (p1, l1))):
        for name, v in pl.items():
            ctx.upload(inputs[name], v)
        ctx.upload(ldev, np.frombuffer(bytes(lt), np.uint8))
        g.replay()
        torch.cuda.synchronize()
        assert_equal(ctx.download(out, np.float32, w * h * 4).reshape(h, w, 4), eager[k], f"replay {k}")
    assert not np.array_equal(eager[0], eager[1])
    assert_equal(eager[1], oracle(po, pcam, s, l1, p1), "eager vs oracle")
    del g
    d.free()


def test_renderer_chain(capi, po):
    """oxr_apply_pbr on a rendered frame of the 20,000-instance scene over a ground plane, with the shadow resolve and GTAO: equal to
    orc_apply_pbr over oxr_decode_gbuffer's planes, the oracle resolve (pyoracle_vsm_resolve over the renderer's page table and atlas
    and the G-buffer's normal plane) and the oracle GTAO over that plane; equal to the same oxc_* calls composed by hand on the
    renderer's outputs; the next camera frame equals the one of a renderer without the call"""
    import pyoracle_gtao
    import pyoracle_vsm_resolve as vr

    from tests.test_gpu_gbuffer import Table, scene_with_materials
    from tests.test_gpu_gtao import gtao_camera_for
    from tests.test_gpu_vsm_draw import coarse_camera
    from tests.test_gpu_vsm_pages import _sequence_frames, vsm_context

    vr.build()
    pyoracle_gtao.build()
    sc = synth.with_ground_caster(scene_with_materials(20000, 48, 10, config_index=2, width=640, height=360, n_unique_meshes=16),
                                  half_size=1200.0, center=(0.0, -2.0, -40.0))
    sc.mesh_instances["material_index"][-1] = 0
    fr = next(iter(_sequence_frames(sc, 1)))
    cam0, cam1 = sc.camera(0.0), sc.camera(1.5)
    gcam, _ = gtao_camera_for(sc.width, sc.height, yaw=0.0)
    gset = abi.gtao_settings(3)
    vsm = vsm_context(width=sc.width, height=sc.height)
    coarse = coarse_camera(sc.mesh_instance_count)
    rng = np.random.default_rng(9)
    lights = synth.make_lights(rng, 40, eye=(0.0, -1.0, 0.0))
    settings = settings_for(abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_GTAO, len(lights))
    pcam = synth.pbr_camera(cam0)
    renderers, tables, last = [capi.Renderer(0, sc), capi.Renderer(0, sc)], [], []
    for k, r in enumerate(renderers):
        tables.append(Table(r.ctx, 10))
        r.set_materials(tables[-1].materials, tables[-1].dev_images, tables[-1].samplers)
        out = r.render(cam0, want_indices=False)
        if k == 0:
            depth = out["depth"].copy()
            inv_pv = synth.pbr_camera(cam0).inv_projection_view[:]
            pg = r.vsm_update_pages(vsm, fr["clip"], np.float32(inv_pv), cam0["resolution"][0], sun_moved=True, hpb_levels=7)
            r.vsm_draw_shadows(coarse)
            got = r.apply_pbr(cam0, settings, lights, cast_shadows=True, gtao_camera=gcam, gtao_settings=gset)
            no_shadow = r.apply_pbr(cam0, settings, lights, gtao_camera=gcam, gtao_settings=gset)
            gb = r.decode_gbuffer(cam0)
            pt = r.ctx.download(pg.page_tables, np.uint32, 10 * 64 * 64).reshape(10, 64, 64)
            atlas = r.ctx.download(pg.physical_atlas, np.float32, 8192 * 8192).reshape(8192, 8192)
            shadow_r = r.vsm_resolve_shadows(cam0)
            ao_r = r.generate_ambient_occlusion(cam0, gcam, gset)
            again = r.apply_pbr(cam0, settings, lights, cast_shadows=True, gtao_camera=gcam, gtao_settings=gset)
        o = r.render(cam1)
        last.append((o["vis32"].copy(), o["depth"].copy(), np.sort(o["visible"])))
    for a, b in zip(*last):
        np.testing.assert_array_equal(a, b)
    planes = dict(depth=depth, albedo=gb[0], normal=gb[1], emissive=gb[2], metallic_roughness_occlusion=gb[3])
    shadow, _ = vr.vsm_resolve_shadows(vsm, np.float32(inv_pv), cam0["resolution"][0], fr["clip"], depth, gb[1], pt, atlas)
    ao = pyoracle_gtao.generate_ambient_occlusion(gcam, gset, depth, gb[1])["ao"]
    np.testing.assert_array_equal(shadow.view(np.uint32), shadow_r.view(np.uint32))
    np.testing.assert_array_equal(ao.view(np.uint32), ao_r.view(np.uint32))
    want = oracle(po, pcam, settings, lights, dict(planes, ambient_occlusion=ao, shadow=shadow, contact_shadow=None))
    assert_equal(got, want, "renderer chain")
    assert_equal(again, got, "second call")
    assert_equal(no_shadow, oracle(po, pcam, settings, lights, dict(planes, ambient_occlusion=ao, shadow=None, contact_shadow=None)),
                 "without shadows")
    # the same oxc_apply_pbr composed by hand on the renderer's context from its decode, resolve and GTAO outputs
    by_hand = run_device(renderers[0].ctx, pcam, settings, lights, dict(planes, ambient_occlusion=ao_r, shadow=shadow_r), omit=("contact_shadow",))
    assert_equal(by_hand, got, "composed by hand")
    assert (shadow[depth != 0] == 0).sum() > 100 and (np.abs(got - no_shadow).sum(-1) > 0).sum() > 100
    assert np.isfinite(got[depth != 0]).all()
    for t, r in zip(tables, renderers):
        t.free()
        r.close()
