"""The tonemap on the device (oxc_tonemap, oxr_tonemap) against the CPU oracle (oracle/oxc_oracle_tonemap.c), bit for bit in every case:
every curve with every subset of the six flags it reads, 1920 x 1080 and 3840 x 2160 with every lens effect, tiny and odd extents,
hostile frames, settings and records, the reference behaviour the specification pins (the Repeat wrap of the bloom upscale, chromatic
aberration replacing the colour, the blue tap at the pixel's corner), the refusals, graph capture, and the renderer's post chain
apply_pbr -> eye adaptation -> bloom -> tonemap on a rendered and lit frame."""
import itertools

import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_post import HOSTILE_RECORDS, INF, NAN, hdr_frame, hostile_frame
from tests.test_gpu_vsm_pages import Dev

pytestmark = pytest.mark.gpu

EA, BL = abi.SCENE_HAS_EYE_ADAPTATION, abi.SCENE_HAS_BLOOM
CA, VG, FG, TB = abi.SCENE_HAS_CHROMATIC_ABERRATION, abi.SCENE_HAS_VIGNETTE, abi.SCENE_HAS_FILM_GRAIN, abi.SCENE_TRANSPARENT_BACKGROUND
FLAGS = (EA, BL, CA, VG, FG, TB)
LENS = CA | VG | FG
TYPES = (abi.TONEMAP_NONE, abi.TONEMAP_ACES, abi.TONEMAP_AGX, abi.TONEMAP_GT7)
TYPE_IDS = ("none", "aces", "agx", "gt7")
# hostile settings: (exposure, bloom_intensity, chromatic_aberration_amount, vignette_amount, film_grain_scale, film_grain_amount, seed)
HOSTILE_SETTINGS = [(NAN, 0.1, 0.5, 0.5, 0.7, 0.6, 0), (INF, NAN, INF, -INF, 0.0, INF, 0xFFFFFFFF), (-INF, INF, NAN, NAN, -16.0, NAN, 7),
                    (1e-40, -INF, -3.0, 1e30, NAN, -1.0, 15), (3e38, 1e30, 1e-40, 0.0, 1e30, 0.0, 0xFFFFFFFF),
                    (-2.0, 0.0, 0.0, 2.0, 0.7, 1e30, 3), (1.0, 0.1, 0.5, 0.5, 64.0, 0.6, 12345), (0.5, 1.0, 40.0, -0.5, -0.7, 0.6, 1)]


def hostile_settings(k, scene_flags, tonemap_type):
    e, b, ca, vg, gs, ga, seed = HOSTILE_SETTINGS[k % len(HOSTILE_SETTINGS)]
    return abi.tonemap_settings(scene_flags, tonemap_type, e, b, ca, vg, gs, ga, seed)


def bloom_image(rng, w, h):
    """a bloom image for a w x h frame: (w // 2) x (h // 2) float4, smooth HDR values"""
    return (hdr_frame(rng, max(w // 2, 1), max(h // 2, 1)) * np.float32(0.25)).astype(np.float32)


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def so():
    import pyoracle_tonemap

    pyoracle_tonemap.build()
    return pyoracle_tonemap


@pytest.fixture(scope="module")
def ctx(capi):
    sc = synth.make_scene(200, config_index=2, width=64, height=64, n_unique_meshes=4)
    hw, hh = sc.hiz_extent()
    c = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
    yield c
    c.close()


def run(ctx, frame, settings, record=None, bloom=None):
    """one oxc_tonemap call on device copies; the output plane starts as NaN"""
    h, w = frame.shape[:2]
    d = Dev(ctx)
    fp = d.put(frame)
    rp = d.put(np.frombuffer(bytes(record), np.uint8)) if record is not None else None
    bp = d.put(bloom) if bloom is not None else None
    op = d.put(np.full((h, w, 4), np.nan, np.float32))
    ctx.tonemap(fp, w, h, settings, rp, bp, op)
    out = d.get(op, np.zeros((h, w, 4), np.float32))
    d.free()
    return out


def assert_bits(got, want, label=""):
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, f"{label}: {len(bad)} values differ, first at {bad[:3].tolist()}: {got[tuple(bad[0][:2])]} != {want[tuple(bad[0][:2])]}"


def check(ctx, so, frame, settings, record=None, bloom=None, label=""):
    got = run(ctx, frame, settings, record, bloom)
    want = so.tonemap(frame, settings, record, bloom)
    assert_bits(got, want, label)
    return got


@pytest.mark.parametrize("tonemap_type", TYPES, ids=TYPE_IDS)
def test_small_flag_matrix(ctx, so, tonemap_type):
    """every subset of the six flags read, at 17 x 9 and 64 x 36, with a random record and bloom image"""
    rng = np.random.default_rng(11 + tonemap_type)
    for w, h in ((17, 9), (64, 36)):
        frame, bloom = hdr_frame(rng, w, h), bloom_image(rng, w, h)
        record = abi.Exposure(0.5, float(np.float32(rng.uniform(0.05, 4.0))))
        for n in range(len(FLAGS) + 1):
            for subset in itertools.combinations(FLAGS, n):
                flags = sum(subset)
                s = abi.tonemap_settings(flags, tonemap_type, exposure=1.5, film_grain_seed=int(rng.integers(16)))
                check(ctx, so, frame, s, record, bloom, f"{w}x{h} flags {flags:#x}")


@pytest.mark.parametrize("w,h", [(1920, 1080), (3840, 2160)], ids=["1920x1080", "3840x2160"])
@pytest.mark.parametrize("tonemap_type", TYPES, ids=TYPE_IDS)
def test_full_size(ctx, so, tonemap_type, w, h):
    """the reference defaults with eye adaptation, bloom and every lens effect"""
    rng = np.random.default_rng(w + tonemap_type)
    frame, bloom = hdr_frame(rng, w, h), bloom_image(rng, w, h)
    s = abi.tonemap_settings(EA | BL | LENS, tonemap_type, film_grain_seed=5)
    out = check(ctx, so, frame, s, abi.Exposure(0.3, 0.8), bloom, f"{w}x{h}")
    assert np.isfinite(out).mean() > 0.99


@pytest.mark.parametrize("w,h", [(1, 1), (1, 7), (3, 2)], ids=["1x1", "1x7", "3x2"])
def test_small_extents(ctx, so, w, h):
    """c = 0 on an axis of extent 1: the lens coordinates are inf or NaN and follow the tap's rules; bloom needs 2 x 2"""
    rng = np.random.default_rng(w * 10 + h)
    frame, bloom = hdr_frame(rng, w, h), bloom_image(rng, w, h)
    flags = LENS | EA | TB | (BL if w >= 2 and h >= 2 else 0)
    for t in TYPES:
        for f in (flags, flags & ~CA):
            check(ctx, so, frame, abi.tonemap_settings(f, t), abi.Exposure(1.0, 2.0), bloom if f & BL else None, f"{w}x{h} type {t} flags {f:#x}")


def test_extent_1919x1079(ctx, so):
    """odd extent: 1 / f32(2 c) is not 1 / width, and the bloom image is 959 x 539"""
    rng = np.random.default_rng(1919)
    frame, bloom = hdr_frame(rng, 1919, 1079), bloom_image(rng, 1919, 1079)
    for t in (abi.TONEMAP_AGX, abi.TONEMAP_GT7):
        check(ctx, so, frame, abi.tonemap_settings(EA | BL | LENS, t), abi.Exposure(1.0, 1.25), bloom, f"type {t}")


def test_small_hostile_frames(ctx, so):
    """NaN, +-inf, negative, subnormal and 3e38 pixels in the frame and the bloom image, every curve and every flag"""
    rng = np.random.default_rng(31)
    for k, (w, h) in enumerate(((48, 30), (33, 17), (2, 2))):
        frame, bloom = hostile_frame(rng, w, h), hostile_frame(rng, w // 2, h // 2)
        for t in TYPES:
            for flags in (EA | BL, EA | BL | LENS | TB, BL | VG | FG):
                s = abi.tonemap_settings(flags, t, film_grain_seed=k)
                check(ctx, so, frame, s, abi.Exposure(1.0, 0.75), bloom, f"{w}x{h} type {t} flags {flags:#x}")


def test_small_hostile_settings(ctx, so):
    """NaN and +-inf exposure, intensity and amounts; grain scales 0.7, 0, -16, NaN, 1e30; seed 0xFFFFFFFF; hostile records"""
    rng = np.random.default_rng(41)
    w, h = 40, 26
    frame, bloom = hdr_frame(rng, w, h), bloom_image(rng, w, h)
    for t in TYPES:
        for k in range(len(HOSTILE_SETTINGS)):
            for flags in (BL | VG | FG, EA | BL | LENS | TB):
                check(ctx, so, frame, hostile_settings(k, flags, t), HOSTILE_RECORDS[k % len(HOSTILE_RECORDS)], bloom,
                      f"type {t} settings {k} flags {flags:#x}")


def test_small_repeat_wrap(ctx, so):
    """the sampler's Repeat: a bright last bloom column reaches output column 0 (and no other column but the last three)"""
    w, h = 32, 8
    frame = np.zeros((h, w, 4), np.float32)
    bloom = np.zeros((h // 2, w // 2, 4), np.float32)
    bloom[:, -1, :3] = 8.0
    s = abi.tonemap_settings(BL, abi.TONEMAP_NONE, exposure=1.0, bloom_intensity=1.0)
    out = check(ctx, so, frame, s, None, bloom)
    assert (out[:, 0, :3] == 2.0).all()  # x = 0.25 * 16 - 0.5 = -0.25: weight 0.25 on column -1 = 15
    assert (out[:, 1:w - 3, :3] == 0.0).all() and (out[:, -3:, :3] > 0).all()


def test_small_chromatic_aberration_replaces_the_colour(ctx, so):
    """under CA the output does not depend on the exposure, the record, the bloom image or the curve"""
    rng = np.random.default_rng(51)
    w, h = 36, 20
    frame = hdr_frame(rng, w, h)
    base = None
    for t in TYPES:
        for flags, exposure, record, bloom in ((CA, 1.0, None, None), (CA | BL, 3.0, None, bloom_image(rng, w, h)),
                                               (CA | EA | BL, 0.1, abi.Exposure(2.0, 7.0), bloom_image(rng, w, h))):
            out = check(ctx, so, frame, abi.tonemap_settings(flags, t, exposure=exposure), record, bloom)
            if base is None:
                base = out
            assert_bits(out, base, f"type {t} flags {flags:#x}")
    assert not np.array_equal(base, check(ctx, so, frame, abi.tonemap_settings(0, abi.TONEMAP_NONE)))


def test_small_blue_tap_at_the_pixel_corner(ctx, so):
    """with amount 0 the red and green taps sit at the pixel centre of an even frame and read the pixel; the blue tap at
    f32(x) / W lies on the pixel's corner and averages the 2 x 2 texels up and to the left (wrapping)"""
    rng = np.random.default_rng(61)
    w, h = 32, 16
    frame = rng.uniform(0.0, 1.0, (h, w, 4)).astype(np.float32)
    out = check(ctx, so, frame, abi.tonemap_settings(CA, abi.TONEMAP_NONE, chromatic_aberration_amount=0.0))
    np.testing.assert_array_equal(out[..., :2], frame[..., :2])
    b = frame[..., 2].astype(np.float64)
    corner = (b + np.roll(b, 1, 0) + np.roll(b, 1, 1) + np.roll(np.roll(b, 1, 0), 1, 1)) / 4
    np.testing.assert_allclose(out[..., 2], corner, rtol=1e-5, atol=1e-6)
    assert not np.allclose(out[..., 2], frame[..., 2])


def test_argument_refusals(capi, ctx):
    d = Dev(ctx)
    w, h = 8, 6
    buf = d.put(np.zeros(1 << 16, np.float32))  # 256 KiB; every pointer below stays inside it
    frame, rec, bloom, out = buf, buf + 4096, buf + 8192, buf + 16384
    fb = w * h * 16
    s_all = abi.tonemap_settings(EA | BL | LENS)

    def refused(fn, match):
        with pytest.raises(capi.OxcError, match=match) as e:
            fn()
        assert "(-1)" in str(e.value)

    def tm(fp=frame, ww=w, hh=h, rp=rec, bp=bloom, op=out, s=s_all):
        ctx.tonemap(fp, ww, hh, s, rp, bp, op)

    launches = capi.kernel_launch_count()
    for kw in ("fp", "rp", "bp", "op"):
        refused(lambda: tm(**{kw: None}), "null argument")
    refused(lambda: tm(fp=frame + 8), "16-byte")
    refused(lambda: tm(op=out + 4), "16-byte")
    refused(lambda: tm(bp=bloom + 8), "16-byte")
    refused(lambda: tm(rp=rec + 4), "8-byte")
    for ww, hh in ((0, 4), (4, 0), (32769, 4), (4, 32769)):
        refused(lambda: tm(ww=ww, hh=hh), "extent")
    for t in (4, 5, 0xFFFFFFFF):
        refused(lambda: tm(s=abi.tonemap_settings(EA | BL, t)), "tonemap_type")
    for ww, hh in ((1, 4), (4, 1), (1, 1)):
        refused(lambda: tm(ww=ww, hh=hh), "below 2 x 2")
    refused(lambda: tm(op=frame), "overlap")  # in place
    refused(lambda: tm(op=frame + fb - 16), "overlap")
    refused(lambda: tm(op=frame - fb + 16), "overlap")
    refused(lambda: tm(op=rec - fb + 16), "overlap")
    refused(lambda: tm(op=bloom + (w // 2) * (h // 2) * 16 - 16), "overlap")
    assert capi.kernel_launch_count() == launches
    # adjacent planes are accepted; without HasEyeAdaptation / HasBloom the record / bloom image is not read, so NULL or overlapping is fine
    tm(op=frame + fb)
    tm(rp=None, bp=None, s=abi.tonemap_settings(LENS))
    tm(rp=out, bp=out, s=abi.tonemap_settings(LENS | TB))
    tm(ww=1, hh=1, s=abi.tonemap_settings(EA | LENS))
    ctx.sync()
    assert capi.kernel_launch_count() == launches + 4
    d.free()


def test_graph_capture_equals_eager(capi, ctx, so):
    """two calls (two curves) captured in one CUDA graph from the first call: two replays equal the oracle"""
    import torch

    w, h = 333, 187
    rng = np.random.default_rng(3)
    frame, bloom = hdr_frame(rng, w, h), bloom_image(rng, w, h)
    rec = abi.Exposure(1.0, 0.6)
    s1, s2 = abi.tonemap_settings(EA | BL | LENS, abi.TONEMAP_GT7), abi.tonemap_settings(BL | VG, abi.TONEMAP_ACES)
    d = Dev(ctx)
    fp, rp, bp = d.put(frame), d.put(np.frombuffer(bytes(rec), np.uint8)), d.put(bloom)
    o1, o2 = d.put(np.zeros((h, w, 4), np.float32)), d.put(np.zeros((h, w, 4), np.float32))
    s = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
        gctx.tonemap(fp, w, h, s1, rp, bp, o1)
        gctx.tonemap(fp, w, h, s2, None, bp, o2)
    for _ in range(2):
        ctx.upload(o1, np.zeros((h, w, 4), np.float32))
        g.replay()
        torch.cuda.synchronize()
        assert_bits(d.get(o1, np.zeros((h, w, 4), np.float32)), so.tonemap(frame, s1, rec, bloom), "gt7")
        assert_bits(d.get(o2, np.zeros((h, w, 4), np.float32)), so.tonemap(frame, s2, None, bloom), "aces")
    del g
    d.free()


def test_renderer_chain(capi, ctx, so):
    """oxr_apply_pbr -> oxr_eye_adaptation -> oxr_bloom -> oxr_tonemap on a rendered and lit frame: equal to oxc_tonemap on the same
    planes and to the oracle, for every curve; the lit plane, the record and the bloom image are left as they were; refused before
    apply_pbr (OXC_E_INVALID) and, under HasEyeAdaptation / HasBloom, before eye adaptation / bloom (OXC_E_STATE), in both orders"""
    from tests.test_gpu_gbuffer import Table, scene_with_materials

    sc = synth.with_ground_caster(scene_with_materials(20000, 48, 10, config_index=2, width=320, height=180, n_unique_meshes=16),
                                  half_size=1200.0, center=(0.0, -2.0, -40.0))
    sc.mesh_instances["material_index"][-1] = 0
    lights = synth.make_lights(np.random.default_rng(3), 16, eye=(0.0, -1.0, 0.0))
    orders = []
    for order in (("eye", "bloom"), ("bloom", "eye")):
        r = capi.Renderer(0, sc)
        table = Table(r.ctx, 10)
        r.set_materials(table.materials, table.dev_images, table.samplers)
        try:
            cam = sc.camera(0.0)
            r.render(cam, want_indices=False)
            with pytest.raises(capi.OxcError, match=r"\(-1\)"):
                r.tonemap(abi.tonemap_settings())
            s = abi.pbr_settings(scene_flags=abi.SCENE_HAS_DIRECTIONAL_LIGHT, sun_direction=(0.3, 0.8, 0.52), sun_intensity=10.0,
                                 light_count=len(lights))
            lit = r.apply_pbr(cam, s, lights)
            es, bs = abi.eye_adaptation_settings(), abi.bloom_settings(scene_flags=EA)
            for step in order:
                with pytest.raises(capi.OxcError, match=r"\(-5\)"):
                    r.tonemap(abi.tonemap_settings(EA if step == "eye" else BL))
                if step == "eye":
                    record = r.eye_adaptation(es, 0.016)
                else:
                    r.bloom(abi.bloom_settings())
            assert r.tonemap(abi.tonemap_settings(0)).shape == (sc.height, sc.width, 4)
            image = r.bloom(bs)
            for t in TYPES:
                st = abi.tonemap_settings(EA | BL | LENS | TB, t, film_grain_seed=9)
                got = r.tonemap(st)
                want = so.tonemap(lit, st, record, image)
                assert_bits(got, want, f"renderer type {t}")
                assert_bits(run(r.ctx, lit, st, record, image), want, f"oxc_tonemap type {t}")
                orders.append(got)
            # the record, the bloom image and the lit plane are as they were: bloom reads the last two, and eye adaptation at
            # delta_time 0 returns the record unchanged
            np.testing.assert_array_equal(r.bloom(bs).view(np.uint32), image.view(np.uint32))
            assert np.frombuffer(bytes(r.eye_adaptation(es, 0.0)), np.uint32).tolist() == np.frombuffer(bytes(record), np.uint32).tolist()
            np.testing.assert_array_equal(r.apply_pbr(cam, s, lights).view(np.uint32), lit.view(np.uint32))
        finally:
            r.close()
    for a, b in zip(orders[:4], orders[4:]):
        assert_bits(a, b, "orders")
