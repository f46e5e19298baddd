"""The sky IBL cube on the device (oxc_atmosphere_sky_ibl, oxr_atmosphere_sky_ibl) against the CPU oracle (oracle/oxc_oracle_sky_ibl.c),
bit for bit in every case: the reference's LUT sizes with cameras at 2 m, 10 km and 150 km and four suns, a five-call history sequence
from a zeroed cube, hostile cubes, random and hostile records, the refusals, graph capture, the renderer's call sequence with its
counter, and oxr_atmosphere_luts unchanged beside it.  The LUTs the cube reads are the oracle's, uploaded."""
import functools

import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_atmosphere import HEIGHTS, SUNS, camera_for, hostile_atmospheres, random_atmosphere
from tests.test_gpu_vsm_pages import Dev

pytestmark = pytest.mark.gpu

SMALL = dict(transmittance_lut_size=(48, 12, 1), sky_view_lut_size=(23, 13, 1), aerial_perspective_lut_size=(2, 2, 2))
REFERENCE = dict(transmittance_lut_size=(256, 64, 1), sky_view_lut_size=(312, 192, 1), aerial_perspective_lut_size=(2, 2, 2))
CUBE = abi.SKY_IBL_CUBE_SHAPE
STRENGTH = abi.SKY_IBL_SUN_AMBIENT_STRENGTH


@functools.lru_cache(maxsize=None)
def _transmittance(record_bytes):
    import pyoracle_atmosphere

    return pyoracle_atmosphere.transmittance(abi.Atmosphere.from_buffer_copy(record_bytes))


def luts(a, camera, sun, intensity):
    """the oracle's transmittance and sky-view LUTs of record `a` (the bake with `a` itself)"""
    import pyoracle_atmosphere

    t = _transmittance(bytes(a))
    sv, _ = pyoracle_atmosphere.sky_luts(a, camera, sun, intensity, t)
    return t, sv


def hostile_cubes():
    """cubes whose texels are NaN, +-inf, zero or negative alpha, negative rgb, subnormal, HALF_MAX or valid history, mixed per texel"""
    rng = np.random.default_rng(12)
    kinds = np.float16([np.nan, np.inf, -np.inf, 0.0, -0.0, -1.0, 6e-8, 65504.0, 0.5, 3.0, -65504.0])
    out = []
    for k in range(4):
        c = rng.choice(kinds, size=CUBE).astype(np.float16)
        if k == 1:
            c[..., 3] = 1.0  # every alpha valid: history decided by rgb alone
        if k == 2:
            c[..., :3] = np.abs(rng.normal(size=CUBE[:3] + (3,)) * 100).astype(np.float16)  # finite rgb: decided by alpha alone
        out.append(c)
    return out


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def so():
    import pyoracle_sky_ibl

    pyoracle_sky_ibl.build()
    return pyoracle_sky_ibl


@pytest.fixture(scope="module")
def ctx(capi):
    sc = synth.make_scene(200, config_index=2, width=64, height=64, n_unique_meshes=4)
    hw, hh = sc.hiz_extent()
    c = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
    yield c
    c.close()


def run_device(ctx, a, camera, sun, intensity, strength, frames, t, sv, cube=None):
    """the cube after one call per frame index in `frames`, in place, from `cube` (zeros when None)"""
    d = Dev(ctx)
    tp, svp = d.put(t), d.put(sv)
    cp = d.put(np.zeros(CUBE, np.float16) if cube is None else cube)
    for f in frames:
        ctx.atmosphere_sky_ibl(a, camera, sun, intensity, strength, f, tp, svp, cp)
    out = d.get(cp, np.zeros(CUBE, np.float16))
    d.free()
    return out


def run_oracle(so, a, camera, sun, intensity, strength, frames, t, sv, cube=None):
    for f in frames:
        cube = so.sky_ibl(a, camera, sun, intensity, strength, f, t, sv, cube)
    return cube


def assert_equal(got, want, label=""):
    bad = np.argwhere(got.view(np.uint16) != want.view(np.uint16))
    assert bad.size == 0, f"{label}: {len(bad)} channels differ, first at {bad[:3].tolist()}"


@pytest.mark.parametrize("sun", list(SUNS))
@pytest.mark.parametrize("height", list(HEIGHTS))
def test_reference_sizes(ctx, so, height, sun):
    """the default record at the reference's LUT sizes (312 x 192 sky view, 256 x 64 transmittance)"""
    a = abi.atmosphere(**REFERENCE)
    cam = camera_for(HEIGHTS[height], yaw=23.0)
    t, sv = luts(a, cam, SUNS[sun], 10.0)
    want = run_oracle(so, a, cam, SUNS[sun], 10.0, STRENGTH, [0], t, sv)
    assert_equal(run_device(ctx, a, cam, SUNS[sun], 10.0, STRENGTH, [0], t, sv), want, f"{height} {sun}")
    assert (want[..., 3] == 1).all() and np.isfinite(want).all()
    if height != "150km" and sun != "below":
        assert (want[..., :3].astype(np.float32) > 0).mean() > 0.5


@pytest.mark.parametrize("height", list(HEIGHTS))
def test_small_history_sequence(ctx, so, height):
    """five calls from a zeroed cube with frame_index 0..4: no history at the first, the lerp after"""
    a = abi.atmosphere(**SMALL)
    cam = camera_for(HEIGHTS[height], yaw=5.0)
    t, sv = luts(a, cam, SUNS["45deg"], 10.0)
    got = want = None
    for f in range(5):
        got = run_device(ctx, a, cam, SUNS["45deg"], 10.0, STRENGTH, [f], t, sv, got)
        want = run_oracle(so, a, cam, SUNS["45deg"], 10.0, STRENGTH, [f], t, sv, want)
        assert_equal(got, want, f"call {f}")
    first = run_oracle(so, a, cam, SUNS["45deg"], 10.0, STRENGTH, [0], t, sv)
    assert not np.array_equal(first.view(np.uint16), want.view(np.uint16))


def test_small_hostile_cubes(ctx, so):
    a = abi.atmosphere(**SMALL)
    cam = camera_for(1000.0)
    t, sv = luts(a, cam, SUNS["45deg"], 10.0)
    for k, cube in enumerate(hostile_cubes()):
        for frame in (0, 7, 0xFFFFFFFF):
            got = run_device(ctx, a, cam, SUNS["45deg"], 10.0, STRENGTH, [frame], t, sv, cube)
            assert_equal(got, run_oracle(so, a, cam, SUNS["45deg"], 10.0, STRENGTH, [frame], t, sv, cube), f"cube {k} frame {frame}")
            assert not np.isnan(got[..., :3].astype(np.float32)).any()


@pytest.mark.parametrize("seed", range(3))
def test_small_random_records(ctx, so, seed):
    rng = np.random.default_rng(900 + seed)
    a = random_atmosphere(rng, **SMALL)
    cam = camera_for(float(rng.choice([0.2, 1000.0, 15000.0, rng.uniform(-100, 30000)])), yaw=float(rng.uniform(0, 360)))
    sun = tuple(rng.normal(size=3) * rng.uniform(0.2, 3))
    si, st, frame = float(rng.uniform(1, 20)), float(rng.uniform(0, 1)), int(rng.integers(0, 2 ** 32))
    t, sv = luts(a, cam, sun, si)
    assert_equal(run_device(ctx, a, cam, sun, si, st, [frame, frame + 1], t, sv), run_oracle(so, a, cam, sun, si, st, [frame, frame + 1], t, sv),
                 f"seed {seed}")


def test_small_hostile_records(ctx, so):
    nan, inf = float("nan"), float("inf")
    cams = [camera_for(0.2), camera_for(15000.0), abi.pbr_camera(np.full(16, nan, np.float32), (nan, nan, nan)),
            abi.pbr_camera(np.eye(4, dtype=np.float32).reshape(16), (0.0, inf, 0.0))]
    suns = [(nan, 1.0, 0.0), (0.0, 0.0, 0.0), (inf, 1e-40, -inf), (0.0, 1.0, 0.0)]
    for k, a in enumerate(hostile_atmospheres(**SMALL)):
        cam, sun = cams[k % len(cams)], suns[k % len(suns)]
        t, sv = luts(a, cam, sun, 10.0)
        for si, st in ((10.0, STRENGTH), (nan, inf)):
            assert_equal(run_device(ctx, a, cam, sun, si, st, [k], t, sv), run_oracle(so, a, cam, sun, si, st, [k], t, sv), f"record {k}")


def test_argument_refusals(capi, ctx):
    d = Dev(ctx)
    a = abi.atmosphere(**SMALL)
    nt, nsv = 48 * 12 * 4, 23 * 13 * 4
    buf = d.put(np.zeros(1 << 20, np.uint16))
    t, sv, cube = buf, buf + 131072, buf + 262144  # bytes; every pointer below stays inside the 2 MiB buffer
    cam = camera_for(0.2)
    sun = SUNS["45deg"]

    def refused(fn, match):
        with pytest.raises(capi.OxcError, match=match) as e:
            fn()
        assert "(-1)" in str(e.value)

    def call(rec=a, tp=t, svp=sv, cp=cube, camera=cam, s=sun):
        ctx.atmosphere_sky_ibl(rec, camera, s, 10.0, STRENGTH, 0, tp, svp, cp)

    launches = capi.kernel_launch_count()
    refused(lambda: call(tp=None), "null argument")
    refused(lambda: call(svp=None), "null argument")
    refused(lambda: call(cp=None), "null argument")
    for k in range(3):
        ptrs = [t, sv, cube]
        ptrs[k] += 4
        refused(lambda: call(tp=ptrs[0], svp=ptrs[1], cp=ptrs[2]), "8-byte")
    for bad in ((0, 4, 1), (4, 0, 1), (4097, 4, 1), (4, 4097, 1)):
        refused(lambda: call(rec=abi.atmosphere(**dict(SMALL, transmittance_lut_size=bad))), "transmittance_lut_size")
    for bad in ((1, 4, 1), (4, 1, 1), (0, 4, 1), (4097, 4, 1), (4, 4097, 1)):
        refused(lambda: call(rec=abi.atmosphere(**dict(SMALL, sky_view_lut_size=bad))), "sky_view_lut_size")
    # the cube may not share a byte with either LUT
    refused(lambda: call(cp=t), "overlaps")
    refused(lambda: call(cp=t + nt * 2 - 8), "overlaps")
    refused(lambda: call(cp=sv - abi.SKY_IBL_CUBE_BYTES + 8), "overlaps")
    refused(lambda: call(cp=sv + nsv * 2 - 8), "overlaps")
    assert capi.kernel_launch_count() == launches
    # adjacent planes and the sizes the call does not read are accepted
    ok = abi.atmosphere(**dict(SMALL, aerial_perspective_lut_size=(0, 0, 9999), multiscattering_lut_size=(0, 0, 0)))
    call(rec=ok, cp=sv + nsv * 2)
    call(cp=sv - abi.SKY_IBL_CUBE_BYTES)
    call(cp=t + nt * 2)
    ctx.sync()
    assert capi.kernel_launch_count() == launches + 3
    d.free()


def test_graph_capture_equals_eager(capi, ctx, so):
    """the call captured into a CUDA graph replays the frame_index it was captured with, in place, equal to eager calls"""
    import torch

    a = abi.atmosphere(**SMALL)
    cam = camera_for(1000.0, yaw=30.0)
    t, sv = luts(a, cam, SUNS["45deg"], 10.0)
    eager = run_device(ctx, a, cam, SUNS["45deg"], 10.0, STRENGTH, [6, 6], t, sv)
    d = Dev(ctx)
    tp, svp, cp = d.put(t), d.put(sv), d.put(np.zeros(CUBE, np.float16))
    s = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
        gctx.atmosphere_sky_ibl(a, cam, SUNS["45deg"], 10.0, STRENGTH, 6, tp, svp, cp)
    ctx.upload(cp, np.zeros(CUBE, np.float16))
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert_equal(d.get(cp, np.zeros(CUBE, np.float16)), eager, "replay")
    assert_equal(eager, run_oracle(so, a, cam, SUNS["45deg"], 10.0, STRENGTH, [6, 6], t, sv), "eager vs oracle")
    del g
    d.free()


def test_renderer_sky_ibl_sequence(capi, so):
    """oxr_atmosphere_sky_ibl: the LUTs oxr_atmosphere_luts makes (the bake with the default record, the caller's record at the renderer's
    sizes), then the cube with strength 0.15 and frame_index 0, 1, 2 from a zeroed cube: equal to the oracle's sequence; a second
    renderer's oxr_atmosphere_luts returns what the oracle returns beside it, and the camera frame after the calls is unchanged"""
    import pyoracle_atmosphere as ao

    sc = synth.make_scene(2000, config_index=2, width=160, height=96, n_unique_meshes=8)
    cam0, cam1 = sc.camera(0.0), sc.camera(1.5)
    rng = np.random.default_rng(19)
    scene_atmosphere = random_atmosphere(rng, transmittance_lut_size=(3, 3, 1), sky_view_lut_size=(5, 5, 1), aerial_perspective_lut_size=(2, 2, 2))
    calls = [(camera_for(1000.0, yaw=40.0), SUNS["45deg"], 12.0), (camera_for(0.2), SUNS["zenith"], 12.0), (camera_for(0.2), SUNS["below"], 3.0)]
    default = abi.atmosphere()
    sized = abi.Atmosphere.from_buffer_copy(scene_atmosphere)
    for name in ("transmittance_lut_size", "sky_view_lut_size", "aerial_perspective_lut_size"):
        getattr(sized, name)[:] = list(getattr(default, name))
    t = ao.transmittance(default)
    renderers, last = [capi.Renderer(0, sc), capi.Renderer(0, sc)], []
    for k, r in enumerate(renderers):
        r.render(cam0, want_indices=False)
        if k == 0:
            want = None
            for frame, (pcam, sun, si) in enumerate(calls):
                got = r.atmosphere_sky_ibl(scene_atmosphere, pcam, sun, si)
                sv, _ = ao.sky_luts(sized, pcam, sun, si, t)
                want = so.sky_ibl(sized, pcam, sun, si, STRENGTH, frame, t, sv, want)
                assert_equal(got, want, f"call {frame}")
        else:
            pcam, sun, si = calls[0]
            got = r.atmosphere_luts(scene_atmosphere, pcam, sun, si)
            sv, ap = ao.sky_luts(sized, pcam, sun, si, t)
            for g, w in zip(got, (t, sv, ap)):
                np.testing.assert_array_equal(g.view(np.uint16), w.view(np.uint16))
        o = r.render(cam1)
        last.append((o["vis32"].copy(), o["depth"].copy(), np.sort(o["visible"])))
    for x, y in zip(*last):
        np.testing.assert_array_equal(x, y)
    for r in renderers:
        r.close()
