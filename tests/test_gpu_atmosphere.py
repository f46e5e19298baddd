"""The atmosphere's lookup tables on the device (oxc_atmosphere_transmittance, oxc_atmosphere_sky_luts, oxr_atmosphere_luts) against the
CPU oracle (oracle/oxc_oracle_atmosphere.c), bit for bit in every case: the reference's sizes and odd and minimum ones, the default and
random atmospheres, the sun at the zenith, on the horizon and below it, cameras at 2 m, 10 km and 150 km, hostile NaN / Inf / denormal
records, the refusals, graph capture, and the renderer's call against the oxc_* calls made by hand."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_vsm_pages import Dev

pytestmark = pytest.mark.gpu

# camera heights in world units: CAMERA_SCALE_UNIT = 0.01 km, so 0.2 is 2 m, 1000 is 10 km and 15000 is 150 km
HEIGHTS = {"2m": 0.2, "10km": 1000.0, "150km": 15000.0}
SUNS = {"zenith": (0.0, 1.0, 0.0), "horizon": (0.8, 0.0, -0.6), "below": (0.3, -0.4, 0.866), "45deg": (0.0, 0.70710677, -0.70710677)}


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def ao():
    """the atmosphere oracle (oracle/pyoracle_atmosphere.py)"""
    import pyoracle_atmosphere

    pyoracle_atmosphere.build()
    return pyoracle_atmosphere


@pytest.fixture(scope="module")
def ctx(capi):
    sc = synth.make_scene(200, config_index=2, width=64, height=64, n_unique_meshes=4)
    hw, hh = sc.hiz_extent()
    c = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
    yield c
    c.close()


def camera_for(height, yaw=0.0, w=32, h=32):
    """abi.PbrCamera of a make_camera camera at (0, height, 0): the binary64 inverse of its projection_view rounded to binary32"""
    proj, view = synth.camera_matrices(w, h, yaw, eye=(0.0, height, 0.0))
    pv = synth.mat_mul_cm(proj, view)
    inv = np.linalg.inv(pv.reshape(4, 4).T.astype(np.float64)).T.astype(np.float32).reshape(16)
    return abi.pbr_camera(inv, (0.0, height, 0.0))


def random_atmosphere(rng, **sizes):
    """fields spread around the defaults: scattering x0.2..5, densities 2..20 km, asymmetry -0.9..3.6, radii with a 20..200 km shell"""
    d = abi.ATMOSPHERE_DEFAULTS
    r = float(rng.uniform(1000.0, 7000.0))
    return abi.atmosphere(rayleigh_scatter=np.float32(d["rayleigh_scatter"]) * rng.uniform(0.2, 5.0, 3), rayleigh_density=rng.uniform(2, 20),
                          mie_scatter=np.float32(d["mie_scatter"]) * rng.uniform(0.2, 5.0, 3), mie_density=rng.uniform(0.5, 5),
                          mie_extinction=rng.uniform(0.001, 0.02), mie_asymmetry=rng.uniform(-0.9, 3.6),
                          ozone_absorption=np.float32(d["ozone_absorption"]) * rng.uniform(0.2, 5.0, 3), ozone_height=rng.uniform(5, 40),
                          ozone_thickness=rng.uniform(2, 30), planet_radius=r, atmos_radius=r + rng.uniform(20.0, 200.0), **sizes)


def hostile_atmospheres(**sizes):
    """NaN, Inf, denormal, zero and inverted fields, one kind per record"""
    nan, inf, den = float("nan"), float("inf"), 1e-40
    return [abi.atmosphere(rayleigh_density=nan, mie_asymmetry=inf, **sizes),
            abi.atmosphere(planet_radius=nan, **sizes),
            abi.atmosphere(atmos_radius=inf, ozone_thickness=0.0, **sizes),
            abi.atmosphere(rayleigh_scatter=(den, inf, -1.0), mie_extinction=-inf, mie_density=den, **sizes),
            abi.atmosphere(atmos_radius=6000.0, **sizes),  # inside the planet: the bake's exit distance is `none`
            abi.atmosphere(mie_asymmetry=1.67154, ozone_height=nan, **sizes)]


def lut_shapes(a):
    t = (a.transmittance_lut_size[1], a.transmittance_lut_size[0], 4)
    sv = (a.sky_view_lut_size[1], a.sky_view_lut_size[0], 4)
    ap = (a.aerial_perspective_lut_size[2], a.aerial_perspective_lut_size[1], a.aerial_perspective_lut_size[0], 4)
    return t, sv, ap


def run_device(ctx, bake, frame, camera, sun, intensity):
    """(transmittance, sky view, aerial perspective) float16 planes: the bake with `bake`, then the per-frame LUTs with `frame`"""
    ts, svs, aps = lut_shapes(frame)
    assert tuple(lut_shapes(bake)[0]) == tuple(ts)
    d = Dev(ctx)
    t, sv, ap = d.put(np.zeros(ts, np.float16)), d.put(np.zeros(svs, np.float16)), d.put(np.zeros(aps, np.float16))
    ctx.atmosphere_transmittance(bake, t)
    ctx.atmosphere_sky_luts(frame, camera, sun, intensity, t, sv, ap)
    out = tuple(d.get(p, np.zeros(s, np.float16)) for p, s in ((t, ts), (sv, svs), (ap, aps)))
    d.free()
    return out


def run_oracle(ao, bake, frame, camera, sun, intensity):
    t = ao.transmittance(bake)
    sv, ap = ao.sky_luts(frame, camera, sun, intensity, t)
    return t, sv, ap


def assert_equal(got, want, label=""):
    for name, g, w in zip(("transmittance", "sky view", "aerial perspective"), got, want):
        bad = np.argwhere(g.view(np.uint16) != w.view(np.uint16))
        assert bad.size == 0, f"{label} {name}: {len(bad)} channels differ, first at {bad[:3].tolist()}"


REFERENCE_SIZES = dict(transmittance_lut_size=(256, 64, 1), sky_view_lut_size=(312, 192, 1), aerial_perspective_lut_size=(32, 32, 32))
SIZES = {"reference": REFERENCE_SIZES,
         "odd": dict(transmittance_lut_size=(37, 11, 1), sky_view_lut_size=(17, 9, 1), aerial_perspective_lut_size=(13, 7, 5)),
         "minimum": dict(transmittance_lut_size=(1, 1, 1), sky_view_lut_size=(2, 2, 1), aerial_perspective_lut_size=(1, 1, 1)),
         "deep": dict(transmittance_lut_size=(64, 16, 1), sky_view_lut_size=(40, 24, 1), aerial_perspective_lut_size=(4, 3, 40))}


@pytest.mark.parametrize("size", list(SIZES))
@pytest.mark.parametrize("height", list(HEIGHTS))
def test_sizes_and_heights(ctx, ao, size, height):
    """the default atmosphere with the sun at 45 degrees at each size and camera height"""
    a = abi.atmosphere(**SIZES[size])
    cam = camera_for(HEIGHTS[height], yaw=13.0)
    want = run_oracle(ao, a, a, cam, SUNS["45deg"], 10.0)
    assert_equal(run_device(ctx, a, a, cam, SUNS["45deg"], 10.0), want, f"{size} {height}")
    if size == "reference":
        sv, ap = want[1].astype(np.float32), want[2].astype(np.float32)
        if height == "150km":  # above the atmosphere: the rays that miss it are exactly 0
            assert (sv == 0).all(-1).sum() > 1000 and (ap == 0).all()
        else:
            assert (sv[..., 3] > 0).all() and np.isfinite(ap).all()


@pytest.mark.parametrize("sun", ["zenith", "horizon", "below"])
def test_suns(ctx, ao, sun):
    a = abi.atmosphere(**SIZES["odd"])
    for height in HEIGHTS.values():
        cam = camera_for(height, yaw=71.0)
        assert_equal(run_device(ctx, a, a, cam, SUNS[sun], 7.5), run_oracle(ao, a, a, cam, SUNS[sun], 7.5), f"{sun} {height}")


@pytest.mark.parametrize("seed", range(4))
def test_random_atmospheres(ctx, ao, seed):
    """random records, cameras and suns; the bake with the default record as the renderer makes it, and with the random one"""
    rng = np.random.default_rng(300 + seed)
    a = random_atmosphere(rng, **SIZES["odd" if seed % 2 else "deep"])
    cam = camera_for(float(rng.choice([0.2, 1000.0, 15000.0, rng.uniform(-100, 30000)])), yaw=float(rng.uniform(0, 360)))
    sun = rng.normal(size=3)
    default = abi.atmosphere(**SIZES["odd" if seed % 2 else "deep"])
    for bake in (default, a):
        si = float(np.float32(rng.uniform(1, 20)))
        assert_equal(run_device(ctx, bake, a, cam, sun, si), run_oracle(ao, bake, a, cam, sun, si), f"seed {seed}")


def test_hostile_records(ctx, ao):
    """NaN, Inf, denormal and inverted records, cameras and suns do not fault and equal the oracle"""
    sizes = SIZES["odd"]
    nan, inf = float("nan"), float("inf")
    cams = [camera_for(0.2), camera_for(15000.0), abi.pbr_camera(np.full(16, nan, np.float32), (nan, nan, nan)),
            abi.pbr_camera(np.eye(4, dtype=np.float32).reshape(16), (0.0, inf, 0.0))]
    suns = [(nan, 1.0, 0.0), (0.0, 0.0, 0.0), (inf, 1e-40, -inf)]
    for k, a in enumerate(hostile_atmospheres(**sizes)):
        cam, sun = cams[k % len(cams)], suns[k % len(suns)]
        assert_equal(run_device(ctx, a, a, cam, sun, 10.0), run_oracle(ao, a, a, cam, sun, 10.0), f"record {k}")
    a = abi.atmosphere(**sizes)
    for k, cam in enumerate(cams):
        for sun in suns:
            assert_equal(run_device(ctx, a, a, cam, sun, nan if k == 3 else 10.0), run_oracle(ao, a, a, cam, sun, nan if k == 3 else 10.0),
                         f"camera {k} sun {sun}")


def test_argument_refusals(capi, ctx):
    d = Dev(ctx)
    buf = d.put(np.zeros(1 << 22, np.uint16))
    a = abi.atmosphere(**SIZES["odd"])
    cam = camera_for(0.2)
    sun = SUNS["45deg"]

    def refused(fn, match):
        with pytest.raises(capi.OxcError, match=match) as e:
            fn()
        assert "(-1)" in str(e.value)

    launches = capi.kernel_launch_count()
    refused(lambda: ctx.atmosphere_transmittance(a, None), "null argument")
    refused(lambda: ctx.atmosphere_transmittance(a, buf + 2), "8-byte")
    for bad in ((0, 4, 1), (4, 0, 1), (4097, 4, 1), (4, 4097, 1)):
        refused(lambda: ctx.atmosphere_transmittance(abi.atmosphere(transmittance_lut_size=bad), buf), "transmittance_lut_size")
        refused(lambda: ctx.atmosphere_sky_luts(abi.atmosphere(**dict(SIZES["odd"], transmittance_lut_size=bad)), cam, sun, 1.0, buf, buf, buf),
                "transmittance_lut_size")
    for bad in ((1, 4, 1), (4, 1, 1), (0, 4, 1), (4097, 4, 1)):
        refused(lambda: ctx.atmosphere_sky_luts(abi.atmosphere(**dict(SIZES["odd"], sky_view_lut_size=bad)), cam, sun, 1.0, buf, buf, buf),
                "sky_view_lut_size")
    for bad in ((0, 4, 4), (4, 0, 4), (4, 4, 0), (4097, 4, 4), (4, 4097, 4), (4, 4, 257)):
        refused(lambda: ctx.atmosphere_sky_luts(abi.atmosphere(**dict(SIZES["odd"], aerial_perspective_lut_size=bad)), cam, sun, 1.0, buf, buf,
                                                buf), "aerial_perspective_lut_size")
    refused(lambda: ctx.atmosphere_sky_luts(a, cam, sun, 1.0, None, buf, buf), "null argument")
    refused(lambda: ctx.atmosphere_sky_luts(a, cam, sun, 1.0, buf, None, buf), "null argument")
    refused(lambda: ctx.atmosphere_sky_luts(a, cam, sun, 1.0, buf, buf, None), "null argument")
    for k in range(3):
        ptrs = [buf, buf, buf]
        ptrs[k] = buf + 4
        refused(lambda: ctx.atmosphere_sky_luts(a, cam, sun, 1.0, *ptrs), "8-byte")
    assert capi.kernel_launch_count() == launches
    # the sizes the calls do not read are not checked
    ok = abi.atmosphere(**dict(SIZES["minimum"], multiscattering_lut_size=(0, 0, 0)))
    ok.transmittance_lut_size[2] = 0
    ok.sky_view_lut_size[2] = 99999
    ctx.atmosphere_transmittance(ok, buf)
    ctx.atmosphere_sky_luts(ok, cam, sun, 1.0, buf, buf + 64, buf + 128)
    ctx.sync()
    d.free()


def test_graph_capture_equals_eager(capi, ctx, ao):
    """both calls captured into a CUDA graph at their first call and replayed with a new camera record upload equal eager runs"""
    import torch

    a = abi.atmosphere(**SIZES["odd"])
    cam = camera_for(1000.0, yaw=30.0)
    eager = run_device(ctx, a, a, cam, SUNS["45deg"], 10.0)
    ts, svs, aps = lut_shapes(a)
    d = Dev(ctx)
    t, sv, ap = d.put(np.zeros(ts, np.float16)), d.put(np.zeros(svs, np.float16)), d.put(np.zeros(aps, np.float16))
    s = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
        gctx.atmosphere_transmittance(a, t)
        gctx.atmosphere_sky_luts(a, cam, SUNS["45deg"], 10.0, t, sv, ap)
    for _ in range(2):
        for p, shape in ((t, ts), (sv, svs), (ap, aps)):
            ctx.upload(p, np.full(shape, np.float16(-7.0)))
        g.replay()
        torch.cuda.synchronize()
        got = tuple(d.get(p, np.zeros(shape, np.float16)) for p, shape in ((t, ts), (sv, svs), (ap, aps)))
        assert_equal(got, eager, "replay")
    assert_equal(eager, run_oracle(ao, a, a, cam, SUNS["45deg"], 10.0), "eager vs oracle")
    del g
    d.free()


def test_renderer_atmosphere_luts(capi, ctx, ao):
    """oxr_atmosphere_luts equals the oxc_* calls made by hand: the bake with the default record even when the caller's record differs,
    the per-frame LUTs with the caller's record at the renderer's sizes whatever sizes it carries; the next camera frame is unchanged"""
    sc = synth.make_scene(2000, config_index=2, width=160, height=96, n_unique_meshes=8)
    cam0, cam1 = sc.camera(0.0), sc.camera(1.5)
    rng = np.random.default_rng(9)
    scene_atmosphere = random_atmosphere(rng, transmittance_lut_size=(3, 3, 1), sky_view_lut_size=(5, 5, 1), aerial_perspective_lut_size=(2, 2, 2))
    pcam = camera_for(1000.0, yaw=40.0)
    sun, intensity = SUNS["45deg"], 12.0
    renderers, last = [capi.Renderer(0, sc), capi.Renderer(0, sc)], []
    for k, r in enumerate(renderers):
        r.render(cam0, want_indices=False)
        if k == 0:
            got = r.atmosphere_luts(scene_atmosphere, pcam, sun, intensity)
            again = r.atmosphere_luts(scene_atmosphere, camera_for(0.2), SUNS["zenith"], intensity)
        o = r.render(cam1)
        last.append((o["vis32"].copy(), o["depth"].copy(), np.sort(o["visible"])))
    for x, y in zip(*last):
        np.testing.assert_array_equal(x, y)
    default = abi.atmosphere()
    sized = abi.Atmosphere.from_buffer_copy(scene_atmosphere)
    for name in ("transmittance_lut_size", "sky_view_lut_size", "aerial_perspective_lut_size"):
        getattr(sized, name)[:] = list(getattr(default, name))
    assert_equal(got, run_device(ctx, default, sized, pcam, sun, intensity), "by hand")
    assert_equal(got, run_oracle(ao, default, sized, pcam, sun, intensity), "oracle")
    assert_equal(again, run_oracle(ao, default, sized, camera_for(0.2), SUNS["zenith"], intensity), "second call")
    assert not np.array_equal(got[0].view(np.uint16), ao.transmittance(abi.Atmosphere.from_buffer_copy(sized)).view(np.uint16))
    for r in renderers:
        r.close()
