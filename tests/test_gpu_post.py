"""Eye adaptation and bloom on the device (oxc_eye_adaptation, oxc_bloom, oxr_eye_adaptation, oxr_bloom) against the CPU oracle
(oracle/oxc_oracle_post.c), bit for bit in every case: 1920 x 1080, 3840 x 2160 and odd and tiny extents, hostile and uniform frames,
the frame whose weighted sum wraps mod 2^32, a ten-call adaptation sequence with bloom under HasEyeAdaptation on and off, NaN and Inf
settings, the refusals, graph capture, and the renderer's sequence on a rendered and lit frame with oxr_apply_pbr's output unchanged."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_vsm_pages import Dev

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
EA = abi.SCENE_HAS_EYE_ADAPTATION


def hdr_frame(rng, w, h):
    """a synthetic HDR frame: log-normal luminance over 2^-14..2^16, random hue, some black pixels; alpha random"""
    lum = np.exp2(rng.normal(1.0, 5.0, (h, w))).astype(np.float32)
    rgb = rng.uniform(0.0, 1.0, (h, w, 3)).astype(np.float32) * lum[..., None]
    rgb[rng.random((h, w)) < 0.05] = 0.0
    return np.concatenate([rgb, rng.uniform(-1, 2, (h, w, 1)).astype(np.float32)], axis=2)


def hostile_frame(rng, w, h):
    """pixels of NaN, +-inf, negative, subnormal, zero, the 0.001 threshold and its neighbours, the exposure bounds' luminances, 3e38"""
    f = hdr_frame(rng, w, h)
    kinds = np.float32([NAN, INF, -INF, -1.0, -0.0, 1e-45, 1e-40, 0.001, np.nextafter(np.float32(0.001), np.float32(0)),
                        np.nextafter(np.float32(0.001), np.float32(1)), 2.0 ** -11.5, 2.0 ** 18, 3e38, 65504.0, 1.0])
    m = rng.random(f.shape) < 0.3
    f[m] = rng.choice(kinds, int(m.sum()))
    return f


def uniform_frame(w, h, value=(2.0, 2.0, 2.0, 1.0)):
    return np.broadcast_to(np.float32(value), (h, w, 4)).copy()


HOSTILE_EYE = [abi.eye_adaptation_settings(), abi.eye_adaptation_settings(NAN, 18.0, 1.1, 1.0),
               abi.eye_adaptation_settings(-11.5, INF, INF, -1.0), abi.eye_adaptation_settings(3.0, 3.0, 1e-40, NAN),
               abi.eye_adaptation_settings(18.0, -11.5, -2.0, 0.0), abi.eye_adaptation_settings(-INF, INF, 1.1, INF)]
HOSTILE_BLOOM = [abi.bloom_settings(), abi.bloom_settings(NAN, 0.125, 4.0, 0.75), abi.bloom_settings(1.0, NAN, INF, NAN),
                 abi.bloom_settings(0.0, 0.0, 0.0, 0.0), abi.bloom_settings(-1.0, 2.0, -INF, INF), abi.bloom_settings(1e-40, 1e30, 1e-40, -1.0)]
HOSTILE_RECORDS = [abi.Exposure(1.0, 1.0), abi.Exposure(NAN, NAN), abi.Exposure(INF, -INF), abi.Exposure(-3.0, 1e-40), abi.Exposure(0.0, 0.0)]


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def so():
    import pyoracle_post

    pyoracle_post.build()
    return pyoracle_post


@pytest.fixture(scope="module")
def ctx(capi):
    sc = synth.make_scene(200, config_index=2, width=64, height=64, n_unique_meshes=4)
    hw, hh = sc.hiz_extent()
    c = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
    yield c
    c.close()


def run_eye(ctx, frame, settings, dts, record):
    """(record, histogram) after one oxc_eye_adaptation call per delta_time in `dts`, the record in place from `record`"""
    h, w = frame.shape[:2]
    d = Dev(ctx)
    fp, rp, hp = d.put(frame), d.put(np.frombuffer(bytes(record), np.uint8)), d.put(np.full(256, 0xDEADBEEF, np.uint32))
    for dt in dts:
        ctx.eye_adaptation(fp, w, h, settings, dt, rp, hp)
    rec = abi.Exposure.from_buffer_copy(d.get(rp, np.zeros(8, np.uint8)).tobytes())
    hist = d.get(hp, np.zeros(256, np.uint32))
    d.free()
    return rec, hist


def oracle_eye(so, frame, settings, dts, record):
    hist = None
    for dt in dts:
        record, hist = so.eye_adaptation(frame, settings, dt, record)
    return record, hist


def run_bloom(ctx, frame, settings, record=None, up_init=None):
    h, w = frame.shape[:2]
    n = abi.bloom_chain_texels(w, h)
    d = Dev(ctx)
    fp = d.put(frame)
    rp = d.put(np.frombuffer(bytes(record), np.uint8)) if record is not None else None
    dp = d.put(np.full((n, 4), np.nan, np.float32))
    up = d.put(np.zeros((n, 4), np.float32) if up_init is None else up_init)
    ctx.bloom(fp, w, h, settings, rp, dp, up)
    out = d.get(dp, np.zeros((n, 4), np.float32)), d.get(up, np.zeros((n, 4), np.float32))
    d.free()
    return out


def assert_record(got, want, label=""):
    g, w = np.frombuffer(bytes(got), np.uint32), np.frombuffer(bytes(want), np.uint32)
    assert (g == w).all(), f"{label}: record {list(g)} != {list(w)}"


def assert_chains(got, want, label=""):
    for name, g, w in zip(("downsampled", "upsampled"), got, want):
        bad = np.argwhere(g.view(np.uint32) != w.view(np.uint32))
        assert bad.size == 0, f"{label} {name}: {len(bad)} values differ, first at {bad[:3].tolist()}"


SIZES = [(1920, 1080), (3840, 2160), (1921, 1079), (2, 2), (3, 2), (2, 1000)]


@pytest.mark.parametrize("w,h", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_sizes(ctx, so, w, h):
    """an HDR frame: the histogram, the record and both chains, with HasEyeAdaptation reading the record eye adaptation left"""
    frame = hdr_frame(np.random.default_rng(w * 7 + h), w, h)
    es = abi.eye_adaptation_settings()
    rec, hist = run_eye(ctx, frame, es, [0.016], abi.Exposure(1.0, 1.0))
    want_rec, want_hist = oracle_eye(so, frame, es, [0.016], abi.Exposure(1.0, 1.0))
    np.testing.assert_array_equal(hist, want_hist)
    assert int(hist.sum()) == w * h
    assert_record(rec, want_rec, f"{w}x{h}")
    bs = abi.bloom_settings(scene_flags=EA)
    got = run_bloom(ctx, frame, bs, rec)
    want = so.bloom(frame, bs, want_rec)
    assert_chains(got, want, f"{w}x{h}")
    lv = abi.bloom_levels(w, h)
    if len(lv) > 1:
        w0, h0, _ = lv[0]
        assert np.isfinite(want[1][: w0 * h0]).all() and (want[1][: w0 * h0, 3] == 1).all()


@pytest.mark.parametrize("w,h", [(1920, 1080), (67, 45)], ids=["1920x1080", "small-67x45"])
def test_uniform_frame(ctx, so, w, h):
    """every pixel in one bin: the adversarial case of the histogram's atomics"""
    frame = uniform_frame(w, h)
    es = abi.eye_adaptation_settings()
    rec, hist = run_eye(ctx, frame, es, [0.1], abi.Exposure(1.0, 1.0))
    want_rec, want_hist = oracle_eye(so, frame, es, [0.1], abi.Exposure(1.0, 1.0))
    np.testing.assert_array_equal(hist, want_hist)
    assert (hist > 0).sum() == 1
    assert_record(rec, want_rec)
    assert_chains(run_bloom(ctx, frame, abi.bloom_settings()), so.bloom(frame, abi.bloom_settings()))


def test_wrapping_frame(ctx, so):
    """4096 x 4352 = 17,825,792 pixels in bin 255: weighted = 255 * 17,825,792 wraps mod 2^32, on both sides alike"""
    w, h = 4096, 4352
    frame = uniform_frame(w, h, (1e30, 1e30, 1e30, 1.0))
    es = abi.eye_adaptation_settings()
    rec, hist = run_eye(ctx, frame, es, [0.5], abi.Exposure(1.0, 1.0))
    want_rec, want_hist = oracle_eye(so, frame, es, [0.5], abi.Exposure(1.0, 1.0))
    assert int(want_hist[255]) == w * h and w * h * 255 >= 2 ** 32
    np.testing.assert_array_equal(hist, want_hist)
    assert_record(rec, want_rec)


def test_small_hostile_frames(ctx, so):
    rng = np.random.default_rng(77)
    for k, (w, h) in enumerate(((96, 70), (2, 2), (3, 3), (1, 1), (33, 2))):  # 96 x 70: level 0 above the tail
        frame = hostile_frame(rng, w, h)
        for j, es in enumerate(HOSTILE_EYE):
            record = HOSTILE_RECORDS[(k + j) % len(HOSTILE_RECORDS)]
            dt = (0.016, 0.0, INF, NAN, -1.0, 1e-40)[j]
            rec, hist = run_eye(ctx, frame, es, [dt], record)
            want_rec, want_hist = oracle_eye(so, frame, es, [dt], record)
            np.testing.assert_array_equal(hist, want_hist, err_msg=f"{w}x{h} settings {j}")
            assert_record(rec, want_rec, f"{w}x{h} settings {j}")
            if w >= 2 and h >= 2:
                bs = HOSTILE_BLOOM[j]
                bs.scene_flags = EA if j % 2 else 0
                assert_chains(run_bloom(ctx, frame, bs, record), so.bloom(frame, bs, record), f"{w}x{h} bloom {j}")


def test_small_adaptation_sequence(ctx, so):
    """ten calls with varying delta_time (0 and inf among them) on changing frames; after each, bloom with HasEyeAdaptation on and off"""
    rng = np.random.default_rng(5)
    es = abi.eye_adaptation_settings()
    rec_dev = rec_or = abi.Exposure(1.0, 1.0)
    dts = [0.016, 0.0, 0.033, 1.0, INF, 0.016, 1e-3, 0.25, 0.0, 0.1]
    exposures = set()
    for k, dt in enumerate(dts):
        frame = hdr_frame(rng, 48, 30) * np.float32(2.0 ** (k - 5))
        rec_dev, _ = run_eye(ctx, frame, es, [dt], rec_dev)
        rec_or, _ = oracle_eye(so, frame, es, [dt], rec_or)
        assert_record(rec_dev, rec_or, f"call {k}")
        exposures.add(rec_or.exposure)
        for flags in (0, EA):
            bs = abi.bloom_settings(scene_flags=flags)
            assert_chains(run_bloom(ctx, frame, bs, rec_dev), so.bloom(frame, bs, rec_or), f"call {k} flags {flags}")
    assert len(exposures) > 5


def test_small_upsampled_last_level_untouched(ctx, so):
    """upsampled level n-1 keeps what the caller left there; a single-level chain is (0, 0, 0, 1)"""
    rng = np.random.default_rng(8)
    for w, h in ((40, 22), (3, 3)):
        frame = hdr_frame(rng, w, h)
        n = abi.bloom_chain_texels(w, h)
        init = rng.normal(size=(n, 4)).astype(np.float32)
        got = run_bloom(ctx, frame, abi.bloom_settings(), None, init)
        want = so.bloom(frame, abi.bloom_settings(), None, init)
        assert_chains(got, want, f"{w}x{h}")
        lw, lh, off = abi.bloom_levels(w, h)[-1]
        if len(abi.bloom_levels(w, h)) > 1:
            np.testing.assert_array_equal(got[1][off:], init[off:])
        else:
            np.testing.assert_array_equal(got[1], np.float32([[0, 0, 0, 1]] * n))


def test_argument_refusals(capi, ctx):
    d = Dev(ctx)
    w, h = 8, 6
    buf = d.put(np.zeros(1 << 16, np.float32))  # 256 KiB; every pointer below stays inside it
    frame, rec, hist = buf, buf + 4096, buf + 8192
    n = abi.bloom_chain_texels(w, h) * 16
    down, up = buf + 16384, buf + 32768
    es, bs = abi.eye_adaptation_settings(), abi.bloom_settings(scene_flags=EA)

    def refused(fn, match):
        with pytest.raises(capi.OxcError, match=match) as e:
            fn()
        assert "(-1)" in str(e.value)

    def eye(fp=frame, ww=w, hh=h, rp=rec, hp=hist, s=es):
        ctx.eye_adaptation(fp, ww, hh, s, 0.016, rp, hp)

    def bloom(fp=frame, ww=w, hh=h, rp=rec, dp=down, upp=up, s=bs):
        ctx.bloom(fp, ww, hh, s, rp, dp, upp)

    launches = capi.kernel_launch_count()
    for kw in ("fp", "rp", "hp"):
        refused(lambda: eye(**{kw: None}), "null argument")
    for kw in ("fp", "rp", "dp", "upp"):
        refused(lambda: bloom(**{kw: None}), "null argument")
    refused(lambda: eye(fp=frame + 4), "16-byte")
    refused(lambda: eye(rp=rec + 4), "8-byte")
    refused(lambda: eye(hp=hist + 2), "4-byte")
    refused(lambda: bloom(fp=frame + 8), "16-byte")
    refused(lambda: bloom(rp=rec + 4), "8-byte")
    refused(lambda: bloom(dp=down + 8), "16-byte")
    refused(lambda: bloom(upp=up + 4), "16-byte")
    for ww, hh in ((0, 4), (4, 0), (32769, 4), (4, 32769)):
        refused(lambda: eye(ww=ww, hh=hh), "extent")
        refused(lambda: bloom(ww=ww, hh=hh), "extent")
    for ww, hh in ((1, 4), (4, 1), (1, 1)):
        refused(lambda: bloom(ww=ww, hh=hh), "below 2 x 2")
    # overlaps: histogram / record / frame, and the chains with the frame, the record and each other
    refused(lambda: eye(hp=frame + w * h * 16 - 4), "overlap")
    refused(lambda: eye(rp=frame), "overlap")
    refused(lambda: eye(rp=hist + 1016), "overlap")
    refused(lambda: eye(hp=rec - 1020), "overlap")
    refused(lambda: bloom(dp=frame + w * h * 16 - 16), "overlap")
    refused(lambda: bloom(upp=frame - n + 16), "overlap")
    refused(lambda: bloom(upp=down + n - 16), "overlap")
    refused(lambda: bloom(rp=down + n - 8), "overlap")
    refused(lambda: bloom(rp=up), "overlap")
    assert capi.kernel_launch_count() == launches
    # adjacent planes are accepted; without HasEyeAdaptation the record is not read, so NULL or overlapping is fine
    eye(hp=frame + w * h * 16, rp=frame + w * h * 16 + 1024)
    bloom(dp=frame + w * h * 16, upp=frame + w * h * 16 + n)
    bloom(rp=None, s=abi.bloom_settings())
    bloom(rp=down, s=abi.bloom_settings())
    ctx.sync()
    assert capi.kernel_launch_count() > launches
    d.free()


def test_graph_capture_equals_eager(capi, ctx, so):
    """both calls captured in one CUDA graph (the histogram's memset is a node): two replays equal two eager frames and the oracle"""
    import torch

    w, h = 333, 187
    frame = hdr_frame(np.random.default_rng(3), w, h)
    es, bs = abi.eye_adaptation_settings(), abi.bloom_settings(scene_flags=EA)
    want_rec, want_hist = oracle_eye(so, frame, es, [0.05, 0.05], abi.Exposure(1.0, 1.0))
    want = so.bloom(frame, bs, want_rec)
    n = abi.bloom_chain_texels(w, h)
    d = Dev(ctx)
    fp, rp, hp = d.put(frame), d.put(np.frombuffer(bytes(abi.Exposure(1.0, 1.0)), np.uint8)), d.put(np.full(256, 7, np.uint32))
    dp, up = d.put(np.zeros((n, 4), np.float32)), d.put(np.zeros((n, 4), np.float32))
    s = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
        gctx.eye_adaptation(fp, w, h, es, 0.05, rp, hp)
        gctx.bloom(fp, w, h, bs, rp, dp, up)
    ctx.upload(rp, np.frombuffer(bytes(abi.Exposure(1.0, 1.0)), np.uint8))
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert_record(abi.Exposure.from_buffer_copy(d.get(rp, np.zeros(8, np.uint8)).tobytes()), want_rec, "replay")
    np.testing.assert_array_equal(d.get(hp, np.zeros(256, np.uint32)), want_hist)
    assert_chains((d.get(dp, np.zeros((n, 4), np.float32)), d.get(up, np.zeros((n, 4), np.float32))), want, "replay")
    del g
    d.free()


def test_renderer_sequence(capi, so):
    """oxr_eye_adaptation and oxr_bloom on the lit plane of oxr_apply_pbr: refused before it; three adaptation calls from the record's
    (1, 1), each equal to the oracle on the lit frame apply_pbr returned; bloom with HasEyeAdaptation on and off; apply_pbr returns the
    same frame afterwards"""
    from tests.test_gpu_gbuffer import Table, scene_with_materials

    sc = synth.with_ground_caster(scene_with_materials(20000, 48, 10, config_index=2, width=320, height=180, n_unique_meshes=16),
                                  half_size=1200.0, center=(0.0, -2.0, -40.0))
    sc.mesh_instances["material_index"][-1] = 0
    lights = synth.make_lights(np.random.default_rng(3), 16, eye=(0.0, -1.0, 0.0))
    r = capi.Renderer(0, sc)
    table = Table(r.ctx, 10)
    r.set_materials(table.materials, table.dev_images, table.samplers)
    try:
        cam = sc.camera(0.0)
        r.render(cam, want_indices=False)
        es = abi.eye_adaptation_settings()
        with pytest.raises(capi.OxcError):
            r.eye_adaptation(es, 0.016)
        with pytest.raises(capi.OxcError):
            r.bloom(abi.bloom_settings())
        s = abi.pbr_settings(scene_flags=abi.SCENE_HAS_DIRECTIONAL_LIGHT, sun_direction=(0.3, 0.8, 0.52), sun_intensity=10.0,
                             light_count=len(lights))
        lit = r.apply_pbr(cam, s, lights)
        with pytest.raises(capi.OxcError):
            r.bloom(abi.bloom_settings(scene_flags=EA))  # no record before an eye adaptation
        want = abi.Exposure(1.0, 1.0)
        for dt in (0.016, 0.5, 0.0):
            got = r.eye_adaptation(es, dt)
            want, _ = so.eye_adaptation(lit, es, dt, want)
            assert_record(got, want, f"dt {dt}")
        w0, h0 = sc.width // 2, sc.height // 2
        for flags in (EA, 0):
            bs = abi.bloom_settings(scene_flags=flags)
            np.testing.assert_array_equal(r.bloom(bs).view(np.uint32), so.bloom(lit, bs, want)[1][: w0 * h0].reshape(h0, w0, 4).view(np.uint32))
        np.testing.assert_array_equal(r.apply_pbr(cam, s, lights).view(np.uint32), lit.view(np.uint32))
    finally:
        r.close()
