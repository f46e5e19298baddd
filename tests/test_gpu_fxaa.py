"""FXAA on the device (oxc_fxaa, oxr_fxaa) against the CPU oracle (oracle/oxc_oracle_fxaa.c), bit for bit in every case: 1920 x 1080,
3840 x 2160, 1919 x 1079 and tiny extents; flat, step-edge, diagonal-edge, bar, high-contrast noise, synthetic HDR and hostile frames
(NaN, +-inf, denormals, negatives), which together reach the early exit, the full walk and every tap count between; the refusals; graph
capture; and the renderer's chain apply_pbr -> fxaa -> eye adaptation -> bloom -> tonemap on a rendered and lit frame, where the FXAA
plane becomes the post chain's source until the next apply_pbr."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_post import hdr_frame, hostile_frame
from tests.test_gpu_vsm_pages import Dev

pytestmark = pytest.mark.gpu

EARLY_EXIT_TAPS, MAX_TAPS = 5, 32


def flat_frame(w, h, value=(0.8, 0.5, 0.3, 1.0)):
    return np.broadcast_to(np.float32(value), (h, w, 4)).copy()


def step_frame(w, h, vertical, at=None, lo=0.05, hi=4.0):
    """a straight step edge across the whole frame: every pixel beside it walks past the walk's reach"""
    f = flat_frame(w, h, (lo, lo, lo, 1.0))
    if vertical:
        f[:, (w // 2 if at is None else at):, :3] = hi
    else:
        f[(h // 2 if at is None else at):, :, :3] = hi
    return f


def diagonal_frame(w, h, slope, lo=0.1, hi=3.0):
    """a straight edge y = slope * x + h / 3: shallow slopes give long stair steps, steep ones short ones"""
    yy, xx = np.mgrid[0:h, 0:w]
    f = flat_frame(w, h, (lo, lo, lo, 0.5))
    f[yy > slope * xx + h / 3.0, :3] = hi
    return f


def bars_frame(w, h):
    """bright horizontal bars of every length 1..40 texels on a dark frame: the walk reaches their ends at every step"""
    f = flat_frame(w, h, (0.02, 0.02, 0.02, 1.0))
    y = 2
    for length in range(1, 41):
        if y + 2 > h:
            break
        x0 = (length * 7) % max(w - length, 1)
        f[y:y + 2, x0:x0 + length, :3] = (1.5, 1.2, 0.9)
        y += 4
    return f


def noise_frame(rng, w, h):
    """high contrast noise: nearly every pixel walks"""
    f = np.where(rng.random((h, w, 1)) < 0.5, np.float32(0.0), rng.uniform(0.5, 8.0, (h, w, 1))).astype(np.float32)
    return np.concatenate([f * rng.uniform(0.5, 1.0, (h, w, 3)).astype(np.float32), rng.uniform(0, 1, (h, w, 1)).astype(np.float32)],
                          axis=2).astype(np.float32)


def small_frames(w, h, seed):
    """(label, frame) of every kind at w x h"""
    rng = np.random.default_rng(seed)
    return [("flat", flat_frame(w, h)), ("step-v", step_frame(w, h, True)), ("step-h", step_frame(w, h, False)),
            ("diag-0.1", diagonal_frame(w, h, 0.1)), ("diag-0.45", diagonal_frame(w, h, 0.45)), ("diag-3", diagonal_frame(w, h, 3.0)),
            ("bars", bars_frame(w, h)), ("noise", noise_frame(rng, w, h)), ("hdr", hdr_frame(rng, w, h)), ("hostile", hostile_frame(rng, w, h))]


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def so():
    import pyoracle_fxaa

    pyoracle_fxaa.build()
    return pyoracle_fxaa


@pytest.fixture(scope="module")
def ctx(capi):
    sc = synth.make_scene(200, config_index=2, width=64, height=64, n_unique_meshes=4)
    hw, hh = sc.hiz_extent()
    c = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh)
    yield c
    c.close()


def run(ctx, frame):
    """one oxc_fxaa call on device copies; the output plane starts as NaN"""
    h, w = frame.shape[:2]
    d = Dev(ctx)
    fp = d.put(frame)
    op = d.put(np.full((h, w, 4), np.nan, np.float32))
    ctx.fxaa(fp, w, h, op)
    out = d.get(op, np.zeros((h, w, 4), np.float32))
    d.free()
    return out


def assert_bits(got, want, label=""):
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, f"{label}: {len(bad)} values differ, first at {bad[:3].tolist()}: {got[tuple(bad[0][:2])]} != {want[tuple(bad[0][:2])]}"


def check(ctx, so, frame, label=""):
    """the device against the oracle; returns the oracle's tap counts"""
    want, taps = so.fxaa(frame, with_taps=True)
    assert_bits(run(ctx, frame), want, label)
    return taps


def test_small_frames_reach_every_path(ctx, so):
    """every frame kind at 64 x 36 and 37 x 23; together they reach the early exit (5 taps), the full walk (32) and every count between
    (12..31: the first ends reached at once, and a break after each step of the walk on one or both sides)"""
    counts = np.zeros(MAX_TAPS + 1, np.int64)
    for w, h, seed in ((64, 36, 1), (37, 23, 2), (96, 170, 3)):
        for label, frame in small_frames(w, h, seed):
            counts += np.bincount(check(ctx, so, frame, f"{label} {w}x{h}").ravel(), minlength=MAX_TAPS + 1)
    assert counts[EARLY_EXIT_TAPS] > 0 and counts[MAX_TAPS] > 0
    missing = [n for n in range(12, MAX_TAPS + 1) if counts[n] == 0]
    assert not missing, f"tap counts never reached: {missing}"
    assert counts[:EARLY_EXIT_TAPS].sum() == 0 and counts[EARLY_EXIT_TAPS + 1:12].sum() == 0


@pytest.mark.parametrize("w,h", [(1, 1), (1, 7), (7, 1), (2, 2), (3, 3)], ids=["1x1", "1x7", "7x1", "2x2", "3x3"])
def test_small_extents(ctx, so, w, h):
    """ClampToEdge on every side of a frame one or a few texels wide"""
    for label, frame in small_frames(w, h, w * 10 + h):
        check(ctx, so, frame, f"{label} {w}x{h}")


def test_small_hostile_frames(ctx, so):
    """NaN, +-inf, negative, subnormal and 3e38 pixels; a negative luma sum gives NaN; every stored NaN is 0x7FFFFFFF"""
    rng = np.random.default_rng(31)
    nonfinite = 0
    for w, h in ((48, 30), (33, 17), (5, 4)):
        frame = hostile_frame(rng, w, h)
        check(ctx, so, frame, f"hostile {w}x{h}")
        nonfinite += int((~np.isfinite(so.fxaa(frame))).sum())
        sparse = hdr_frame(rng, w, h)
        sparse[rng.random((h, w)) < 0.02] = np.float32([np.nan, np.inf, -1.0, 1e-40])
        check(ctx, so, sparse, f"sparse hostile {w}x{h}")
    assert nonfinite > 0


@pytest.mark.parametrize("w,h", [(1920, 1080), (3840, 2160)], ids=["1920x1080", "3840x2160"])
def test_full_size(ctx, so, w, h):
    rng = np.random.default_rng(w)
    for label, frame in (("hdr", hdr_frame(rng, w, h)), ("noise", noise_frame(rng, w, h)), ("diag", diagonal_frame(w, h, 0.2)),
                         ("flat", flat_frame(w, h))):
        taps = check(ctx, so, frame, f"{label} {w}x{h}")
        if label == "flat":
            assert (taps == EARLY_EXIT_TAPS).all()


def test_extent_1919x1079(ctx, so):
    rng = np.random.default_rng(1919)
    for label, frame in (("hdr", hdr_frame(rng, 1919, 1079)), ("noise", noise_frame(rng, 1919, 1079)), ("bars", bars_frame(1919, 1079)),
                         ("hostile", hostile_frame(rng, 1919, 1079))):
        check(ctx, so, frame, label)


def test_argument_refusals(capi, ctx):
    d = Dev(ctx)
    w, h = 8, 6
    buf = d.put(np.zeros(1 << 14, np.float32))  # 64 KiB; every pointer below stays inside it
    frame, out = buf, buf + 8192
    fb = w * h * 16

    def refused(fn, match):
        with pytest.raises(capi.OxcError, match=match) as e:
            fn()
        assert "(-1)" in str(e.value)

    def fx(fp=frame, ww=w, hh=h, op=out):
        ctx.fxaa(fp, ww, hh, op)

    launches = capi.kernel_launch_count()
    for kw in ("fp", "op"):
        refused(lambda: fx(**{kw: None}), "null argument")
    refused(lambda: fx(fp=frame + 8), "16-byte")
    refused(lambda: fx(op=out + 4), "16-byte")
    for ww, hh in ((0, 4), (4, 0), (32769, 4), (4, 32769)):
        refused(lambda: fx(ww=ww, hh=hh), "extent")
    refused(lambda: fx(op=frame), "overlap")  # in place
    refused(lambda: fx(op=frame + fb - 16), "overlap")
    refused(lambda: fx(fp=out + fb - 16), "overlap")
    assert capi.kernel_launch_count() == launches
    # adjacent planes are accepted
    fx(op=frame + fb)
    fx(fp=out + fb)
    fx(ww=1, hh=1)
    ctx.sync()
    assert capi.kernel_launch_count() == launches + 3
    d.free()


def test_graph_capture_equals_eager(capi, ctx, so):
    """two calls captured in one CUDA graph from the first call: two replays equal the oracle"""
    import torch

    w, h = 333, 187
    rng = np.random.default_rng(3)
    f1, f2 = hdr_frame(rng, w, h), noise_frame(rng, w, h)
    d = Dev(ctx)
    p1, p2 = d.put(f1), d.put(f2)
    o1, o2 = d.put(np.zeros((h, w, 4), np.float32)), d.put(np.zeros((h, w, 4), np.float32))
    s = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
        gctx.fxaa(p1, w, h, o1)
        gctx.fxaa(p2, w, h, o2)
    for _ in range(2):
        ctx.upload(o1, np.zeros((h, w, 4), np.float32))
        g.replay()
        torch.cuda.synchronize()
        assert_bits(d.get(o1, np.zeros((h, w, 4), np.float32)), so.fxaa(f1), "hdr")
        assert_bits(d.get(o2, np.zeros((h, w, 4), np.float32)), so.fxaa(f2), "noise")
    del g
    d.free()


def test_renderer_chain(capi, ctx, so):
    """oxr_apply_pbr -> oxr_fxaa -> oxr_eye_adaptation -> oxr_bloom -> oxr_tonemap on a rendered and lit frame equals the same oxc_* calls
    by hand and the oracle chain; a second fxaa gives the same plane; the next apply_pbr makes the lit plane the post chain's source
    again; oxr_fxaa before any apply_pbr is OXC_E_INVALID"""
    import pyoracle_post
    import pyoracle_tonemap

    from tests.test_gpu_gbuffer import Table, scene_with_materials

    sc = synth.with_ground_caster(scene_with_materials(20000, 48, 10, config_index=2, width=320, height=180, n_unique_meshes=16),
                                  half_size=1200.0, center=(0.0, -2.0, -40.0))
    sc.mesh_instances["material_index"][-1] = 0
    lights = synth.make_lights(np.random.default_rng(3), 16, eye=(0.0, -1.0, 0.0))
    EA, BL = abi.SCENE_HAS_EYE_ADAPTATION, abi.SCENE_HAS_BLOOM
    post = abi.SCENE_HAS_CHROMATIC_ABERRATION | abi.SCENE_HAS_VIGNETTE | abi.SCENE_HAS_FILM_GRAIN
    r = capi.Renderer(0, sc)
    table = Table(r.ctx, 10)
    r.set_materials(table.materials, table.dev_images, table.samplers)
    try:
        cam = sc.camera(0.0)
        r.render(cam, want_indices=False)
        with pytest.raises(capi.OxcError, match=r"\(-1\)"):
            r.fxaa()
        s = abi.pbr_settings(scene_flags=abi.SCENE_HAS_DIRECTIONAL_LIGHT | abi.SCENE_HAS_FXAA, sun_direction=(0.3, 0.8, 0.52),
                             sun_intensity=10.0, light_count=len(lights))
        lit = r.apply_pbr(cam, s, lights)
        aa, taps = so.fxaa(lit, with_taps=True)
        assert (taps > EARLY_EXIT_TAPS).mean() > 0.001  # the rendered frame has edges that walk
        assert_bits(r.fxaa(), aa, "oxr_fxaa")
        assert_bits(run(r.ctx, lit), aa, "oxc_fxaa")
        assert_bits(r.fxaa(), aa, "second oxr_fxaa")

        es, bs = abi.eye_adaptation_settings(), abi.bloom_settings(scene_flags=EA)
        ts = abi.tonemap_settings(EA | BL | post | abi.SCENE_TRANSPARENT_BACKGROUND, abi.TONEMAP_AGX, film_grain_seed=4)
        record = r.eye_adaptation(es, 0.016)
        image = r.bloom(bs)
        got = r.tonemap(ts)
        # the oracle chain on the FXAA plane
        want_record, _ = pyoracle_post.eye_adaptation(aa, es, 0.016, abi.Exposure(1.0, 1.0))
        assert bytes(record) == bytes(want_record)
        _, up = pyoracle_post.bloom(aa, bs, want_record)
        want_image = up[: (sc.width // 2) * (sc.height // 2)].reshape(sc.height // 2, sc.width // 2, 4)
        assert_bits(image, want_image, "bloom")
        assert_bits(got, pyoracle_tonemap.tonemap(aa, ts, want_record, want_image), "tonemap")
        # the same oxc_* calls by hand on device copies of the FXAA plane
        d = Dev(r.ctx)
        w, h = sc.width, sc.height
        fp = d.put(lit)
        ap, rp = d.put(np.zeros((h, w, 4), np.float32)), d.put(np.float32([1.0, 1.0]))
        hp = d.put(np.zeros(256, np.uint32))
        texels = abi.bloom_chain_texels(w, h)
        dn, upp = d.put(np.zeros((texels, 4), np.float32)), d.put(np.zeros((texels, 4), np.float32))
        op = d.put(np.zeros((h, w, 4), np.float32))
        r.ctx.fxaa(fp, w, h, ap)
        r.ctx.eye_adaptation(ap, w, h, es, 0.016, rp, hp)
        r.ctx.bloom(ap, w, h, bs, rp, dn, upp)
        r.ctx.tonemap(ap, w, h, ts, rp, upp, op)
        assert_bits(d.get(op, np.zeros((h, w, 4), np.float32)), got, "by hand")
        d.free()

        # the next apply_pbr makes the lit plane the source again: the chain equals the oracle chain on the lit frame
        lit2 = r.apply_pbr(cam, s, lights)
        assert_bits(lit2, lit, "lit again")
        rec2 = r.eye_adaptation(es, 0.016)
        want_rec2, hist_lit = pyoracle_post.eye_adaptation(lit, es, 0.016, record)
        assert bytes(rec2) == bytes(want_rec2)
        assert not np.array_equal(hist_lit, pyoracle_post.eye_adaptation(aa, es, 0.016, record)[1])  # the two planes' histograms differ
        image2 = r.bloom(bs)
        _, up2 = pyoracle_post.bloom(lit, bs, want_rec2)
        assert_bits(image2, up2[: (w // 2) * (h // 2)].reshape(h // 2, w // 2, 4), "bloom of the lit plane")
        lit_tonemapped = r.tonemap(ts)
        assert_bits(lit_tonemapped, pyoracle_tonemap.tonemap(lit, ts, want_rec2, image2), "tonemap of the lit plane")
        assert not np.array_equal(lit_tonemapped, got)  # the FXAA plane and the lit plane give different frames
    finally:
        r.close()
