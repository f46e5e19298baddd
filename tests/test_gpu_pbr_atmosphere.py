"""oxc_apply_pbr_atmosphere on the H100 against the oracle (oracle/oxc_oracle_pbr_atmosphere.c), bit for bit: small frames and 1080p
and 4K with 0, 16 and 256 lights over oracle-made LUTs and cube, with cameras at 2 m, 10 km and 200 km and suns above, at and below
the horizon; random and hostile LUTs, cubes, records and planes; every refusal; a captured graph against an eager run."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_pbr import assert_equal, capi, ctx, mixed_lights, random_planes  # noqa: F401
from tests.test_gpu_vsm_pages import Dev
from tests.test_oracle_pbr_atmosphere import random_sky, small_atmosphere

pytestmark = pytest.mark.gpu

EVERY = abi.SCENE_HAS_ATMOSPHERE | abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_CONTACT_SHADOWS


@pytest.fixture(scope="module")
def pa():
    import pyoracle_pbr_atmosphere

    pyoracle_pbr_atmosphere.build()
    return pyoracle_pbr_atmosphere


def run_device(ctx, pcam, s, at, lights, planes, sky):
    h, w = planes["depth"].shape
    d = Dev(ctx)
    inputs = {k: d.put(v) for k, v in planes.items()}
    skyd = dict(zip(abi.PBR_SKY_PLANES, [d.put(p) for p in sky]))
    ldev = d.put(np.frombuffer(bytes(lights), np.uint8)) if lights is not None and len(lights) else None
    out = d.put(np.zeros((h, w, 4), np.float32))
    ctx.apply_pbr_atmosphere(pcam, s, at, ldev, inputs, skyd, w, h, out)
    got = ctx.download(out, np.float32, w * h * 4).reshape(h, w, 4)
    d.free()
    return got


def want(pa, pcam, s, at, lights, planes, sky):
    return pa.apply_pbr_atmosphere(pcam, s, at, lights, *[planes[k] for k in abi.PBR_INPUTS], *sky)


_SKIES = {}


def oracle_sky(camera_y, sun):
    """oracle LUTs at the reference's extents and a cube after two IBL updates, for a camera at camera_y and the sun"""
    import pyoracle_atmosphere
    import pyoracle_sky_ibl

    key = (camera_y, tuple(sun))
    if key not in _SKIES:
        at = abi.atmosphere()
        cam = synth.pbr_camera(synth.make_camera(64, 64, 1))
        cam.position[1] = camera_y
        t = pyoracle_atmosphere.transmittance(at)
        sv, ap = pyoracle_atmosphere.sky_luts(at, cam, sun, 10.0, t)
        cube = None
        for f in range(2):
            cube = pyoracle_sky_ibl.sky_ibl(at, cam, sun, 10.0, abi.SKY_IBL_SUN_AMBIENT_STRENGTH, f, t, sv, cube)
        _SKIES[key] = (at, [t, sv, ap, cube])
    return _SKIES[key]


SUNS = {"high": (0.3, 0.8, 0.52), "horizon": (0.9, 0.0, 0.43), "below": (0.5, -0.3, 0.81)}
# camera y in scene units; get_eye_pos scales by CAMERA_SCALE_UNIT = 0.01 km: 2 m, 10 km, and 200 km above the 100 km atmosphere
HEIGHTS = {"2m": 0.2, "10km": 1000.0, "200km": 20000.0}
# every (extent, light count) of 1080p / 4K x 0 / 16 / 256 and every (height, sun) pair at least once
CASES = [(1920, 1080, 0, "2m", "high"), (1920, 1080, 16, "10km", "horizon"), (1920, 1080, 256, "200km", "below"),
         (3840, 2160, 0, "10km", "below"), (3840, 2160, 16, "200km", "high"), (3840, 2160, 256, "2m", "horizon"),
         (1920, 1080, 16, "2m", "below"), (1920, 1080, 0, "200km", "horizon"), (3840, 2160, 16, "10km", "high")]
SMALL = [(64, 40, 0, "2m", "high"), (96, 54, 16, "10km", "horizon"), (80, 45, 256, "200km", "below")]


def _check(ctx, pa, w, h, n, height, sun):
    at, sky = oracle_sky(HEIGHTS[height], SUNS[sun])
    rng = np.random.default_rng(w * 7 + n)
    pcam, planes = random_planes(rng, w, h, yaw=13.0)
    pcam.position[1] = HEIGHTS[height]
    lights = mixed_lights(rng, n)
    s = abi.pbr_settings(scene_flags=EVERY, sun_direction=SUNS[sun], sun_intensity=10.0, light_count=n)
    assert_equal(run_device(ctx, pcam, s, at, lights, planes, sky), want(pa, pcam, s, at, lights, planes, sky), f"{w}x{h}")


@pytest.mark.parametrize("w,h,n,height,sun", CASES, ids=[f"{w}x{h}_{n}_{c}_{s}" for w, h, n, c, s in CASES])
def test_equals_the_oracle(ctx, pa, w, h, n, height, sun):
    _check(ctx, pa, w, h, n, height, sun)


@pytest.mark.parametrize("w,h,n,height,sun", SMALL, ids=[f"{w}x{h}_{n}_{c}_{s}" for w, h, n, c, s in SMALL])
def test_small_equals_the_oracle(ctx, pa, w, h, n, height, sun):
    _check(ctx, pa, w, h, n, height, sun)


@pytest.mark.parametrize("seed", range(3))
def test_small_hostile(ctx, pa, seed):
    rng = np.random.default_rng(90 + seed)
    at = small_atmosphere((8, 6, 5))
    if seed == 2:
        at.planet_radius, at.aerial_perspective_exposure = float("nan"), float("inf")
    pcam, planes = random_planes(rng, 72, 40, yaw=5.0 * seed, hostile=True)
    sky = random_sky(rng, at, hostile=True)
    lights = mixed_lights(rng, 17, hostile=True)
    s = abi.pbr_settings(scene_flags=EVERY | (abi.SCENE_TRANSPARENT_BACKGROUND if seed == 1 else 0),
                         sun_direction=[float(v) for v in rng.normal(size=3)], sun_intensity=3.0, light_count=17)
    assert_equal(run_device(ctx, pcam, s, at, lights, planes, sky), want(pa, pcam, s, at, lights, planes, sky), f"hostile {seed}")


def test_argument_refusals(capi, ctx):
    d = Dev(ctx)
    buf = d.put(np.zeros(1 << 18, np.uint32))
    pcam = synth.pbr_camera(synth.make_camera(64, 32, 1))
    at = small_atmosphere()
    good = {k: buf for k in abi.PBR_INPUTS}
    sky = {k: buf for k in abi.PBR_SKY_PLANES}
    s = abi.pbr_settings(scene_flags=EVERY, light_count=0)

    def refused(fn, match):
        with pytest.raises(capi.OxcError, match=match):
            fn()

    run = lambda s=s, at=at, inputs=good, sky=sky, w=64, h=32, out=buf: ctx.apply_pbr_atmosphere(pcam, s, at, None, inputs, sky, w, h, out)
    run()
    ctx.sync()
    refused(lambda: run(s=abi.pbr_settings(scene_flags=abi.SCENE_HAS_DIRECTIONAL_LIGHT)), "without HasAtmosphere")
    refused(lambda: run(out=None), "null argument")
    refused(lambda: run(inputs=dict(good, normal=None)), "null input plane")
    refused(lambda: run(s=abi.pbr_settings(scene_flags=EVERY, light_count=257)), "light_count")
    refused(lambda: run(s=abi.pbr_settings(scene_flags=EVERY, light_count=2)), "null lights")
    refused(lambda: run(inputs=dict(good, contact_shadow=None)), "contact_shadow")
    refused(lambda: run(w=0), "empty extent")
    refused(lambda: run(w=40000), "above 32768")
    refused(lambda: run(inputs=dict(good, albedo=buf + 4)), "16-byte")
    refused(lambda: run(inputs=dict(good, depth=buf + 2)), "4-byte")
    for k in abi.PBR_SKY_PLANES:
        refused(lambda k=k: run(sky=dict(sky, **{k: None})), "null sky plane")
        refused(lambda k=k: run(sky=dict(sky, **{k: buf + 4})), "8-byte")
    for field, size, match in (("transmittance_lut_size", (0, 8, 1), "transmittance"), ("sky_view_lut_size", (1, 8, 1), "sky_view"),
                               ("sky_view_lut_size", (4097, 8, 1), "sky_view"), ("aerial_perspective_lut_size", (8, 8, 0), "aerial"),
                               ("aerial_perspective_lut_size", (8, 8, 257), "aerial")):
        bad = small_atmosphere()
        getattr(bad, field)[:] = size
        refused(lambda bad=bad: run(at=bad), match)
    d.free()


def test_graph_capture_equals_eager(capi, ctx, pa):
    """the pass captured into a CUDA graph at its first call and replayed over new planes equals eager runs"""
    import torch

    w, h = 320, 180
    rng = np.random.default_rng(6)
    at = small_atmosphere()
    pcam, p0 = random_planes(rng, w, h)
    _, p1 = random_planes(rng, w, h, yaw=3.0)
    sky = random_sky(rng, at)
    lights = mixed_lights(rng, 16)
    s = abi.pbr_settings(scene_flags=EVERY, sun_direction=(0.3, 0.7, 0.6), light_count=16)
    eager = [run_device(ctx, pcam, s, at, lights, pl, sky) for pl in (p0, p1)]
    d = Dev(ctx)
    inputs = {k: d.put(v) for k, v in p0.items()}
    skyd = dict(zip(abi.PBR_SKY_PLANES, [d.put(p) for p in sky]))
    ldev = d.put(np.frombuffer(bytes(lights), np.uint8))
    out = d.put(np.zeros((h, w, 4), np.float32))
    st = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=st.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st, capture_error_mode="thread_local"):
        gctx.apply_pbr_atmosphere(pcam, s, at, ldev, inputs, skyd, w, h, out)
    for k, pl in enumerate((p0, p1)):
        for name, v in pl.items():
            ctx.upload(inputs[name], v)
        g.replay()
        torch.cuda.synchronize()
        assert_equal(ctx.download(out, np.float32, w * h * 4).reshape(h, w, 4), eager[k], f"replay {k}")
    assert not np.array_equal(eager[0], eager[1])
    assert_equal(eager[1], want(pa, pcam, s, at, lights, p1, sky), "eager vs oracle")
    del g
    d.free()


def test_renderer_sequence(capi, pa):
    """oxr_apply_pbr_atmosphere over three frames of the synthetic scene over a ground plane (camera at 2 m, moving sun): each frame equals
    the oracle run on the G-buffer of oxr_decode_gbuffer and on the LUTs and cube that a second, identical renderer makes with
    oxr_atmosphere_luts / oxr_atmosphere_sky_ibl, so the cube's history and call counter are the same on both; HasAtmosphere without
    HasDirectionalLight is refused before anything runs, and does not advance the counter"""
    from tests.test_gpu_gbuffer import Table, scene_with_materials

    sc = synth.with_ground_caster(scene_with_materials(20000, 48, 10, config_index=2, width=320, height=180, n_unique_meshes=16),
                                  half_size=1200.0, center=(0.0, -2.0, -40.0))
    sc.mesh_instances["material_index"][-1] = 0
    at = abi.atmosphere()
    lights = synth.make_lights(np.random.default_rng(3), 16, eye=(0.0, -1.0, 0.0))
    a, b = capi.Renderer(0, sc), capi.Renderer(0, sc)
    tables = []
    for r in (a, b):
        tables.append(Table(r.ctx, 10))
        r.set_materials(tables[-1].materials, tables[-1].dev_images, tables[-1].samplers)
    try:
        cam = sc.camera(0.0)
        a.render(cam, want_indices=False)
        out = b.render(cam, want_indices=False)
        depth = out["depth"].copy()
        pcam = synth.pbr_camera(cam)
        pcam.position[1] = 0.2
        with pytest.raises(capi.OxcError):
            a.apply_pbr_atmosphere(cam, abi.pbr_settings(scene_flags=abi.SCENE_HAS_ATMOSPHERE), at, pbr_camera=pcam)
        gb = b.decode_gbuffer(cam)
        planes = dict(depth=depth, albedo=gb[0], normal=gb[1], emissive=gb[2], metallic_roughness_occlusion=gb[3])
        lit = 0
        for f, sun in enumerate(((0.3, 0.8, 0.52), (0.5, 0.5, 0.71), (0.9, 0.05, 0.43))):
            s = abi.pbr_settings(scene_flags=abi.SCENE_HAS_ATMOSPHERE | abi.SCENE_HAS_DIRECTIONAL_LIGHT, sun_direction=sun, sun_intensity=10.0,
                                 light_count=len(lights))
            got = a.apply_pbr_atmosphere(cam, s, at, lights, pbr_camera=pcam)
            t, sv, ap = b.atmosphere_luts(at, pcam, sun, 10.0)
            cube = b.atmosphere_sky_ibl(at, pcam, sun, 10.0)
            want_ = pa.apply_pbr_atmosphere(pcam, s, at, lights, planes["depth"], planes["albedo"], planes["normal"], planes["emissive"],
                                            planes["metallic_roughness_occlusion"], None, None, None, t, sv, ap, cube)
            assert_equal(got, want_, f"frame {f}")
            lit += int((got[depth != 0][:, :3].sum(-1) > 0).sum())
        assert lit > 1000
    finally:
        for t in tables:
            t.free()
        a.close()
        b.close()
