"""The terrain draw on the device (oxc_draw_terrain) against the CPU oracle (oracle/oxc_oracle_terrain_draw.c), bit for bit in every case:
the reference's default terrain (1024 m, a 2048 x 2048 heightmap, 64 x 64 patches, 16 px, 64) at 1920 x 1080 and 3840 x 2160 from the
three measurement cameras, fed by the real oxc_cull_terrain; grids of 1 x 1, 3 x 7 and 256 x 256; max_tessellation 1, 3 and 64 and
target_edge_pixels 1; early and late passes through the cull; drawing over a meshlet frame with depth ties, and wide_ids; hostile settings,
an out-of-range instance count and bad patch indices; the refusals and graph capture; and the vis-buffer decode's terrain sentinel in
both packings."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests import helpers_terrain as ht
from tests.test_gpu_vsm_pages import Dev

pytestmark = pytest.mark.gpu

CLEAR = np.uint64(0xFFFFFFFF)


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def so():
    import pyoracle_terrain_draw

    pyoracle_terrain_draw.build()
    return pyoracle_terrain_draw


@pytest.fixture(scope="module")
def ctx(capi):
    c = capi.Context(0, 1, 1, 64, 64)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx_wide(capi):
    c = capi.Context(0, 1, 1, 64, 64, wide_ids=True)
    yield c
    c.close()


def draw(ctx, hm, st, visible, count, cam, w, h, start=None):
    """one oxc_draw_terrain call on device copies of everything; returns the vis buffer"""
    d = Dev(ctx)
    vis0 = np.full((h, w), CLEAR, np.uint64) if start is None else np.ascontiguousarray(start, np.uint64)
    hp, vp = d.put(np.ascontiguousarray(hm, np.uint16)), d.put(np.ascontiguousarray(visible, np.uint32), extra=4)
    cp, gp = d.put(np.uint32([4, count, 0, 0])), d.put(vis0)
    ctx.draw_terrain(hp, hm.shape[1], hm.shape[0], st, vp, cp, cam, w, h, gp)
    out = d.get(gp, vis0)
    d.free()
    return out


def oracle(so, hm, st, visible, count, cam, w, h, start=None, prim_bits=8):
    vis = np.full((h, w), CLEAR, np.uint64) if start is None else np.ascontiguousarray(start, np.uint64).copy()
    n = so.draw_terrain(hm, st, visible, count, cam, vis, prim_bits)
    return vis, n


def assert_same(got, want, label):
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{label}: {len(bad)} pixels differ, first at {bad[:3].tolist()}: {hex(int(got[tuple(bad[0])]))} != {hex(int(want[tuple(bad[0])]))}"


def check(ctx, so, hm, st, visible, count, cam, w, h, label, start=None, prim_bits=8):
    want, n = oracle(so, hm, st, visible, count, cam, w, h, start, prim_bits)
    assert_same(draw(ctx, hm, st, visible, count, cam, w, h, start), want, label)
    return want, n


@pytest.fixture(scope="module")
def default_terrain():
    hm = ht.heightmap(2048, 2048, 7, texel_noise=ht.DEFAULT_TEXEL_NOISE)
    t = ht.terrain()
    return hm, t, ht.patch_minmax(hm, (64, 64))


def cull(ctx, t, mm, cam, flags, mask):
    """oxc_cull_terrain on the device: (visible patches, instance count); mask is updated"""
    n = int(t["patch_count"][0].prod())
    d = Dev(ctx)
    mm_dev, vp, mp, cp = d.put(mm), d.put(np.zeros(n, np.uint32)), d.put(mask), d.put(np.zeros(4, np.uint32))
    ctx.cull_terrain(t, mm_dev, cam, flags, vp, mp, cp)
    cmd = d.get(cp, np.zeros(4, np.uint32))
    visible = d.get(vp, np.zeros(n, np.uint32))
    mask[:] = d.get(mp, mask)
    d.free()
    return visible, int(cmd[1])


@pytest.mark.parametrize("extent", [(1920, 1080), (3840, 2160)], ids=["1080p", "4k"])
def test_default_terrain_three_cameras(ctx, so, default_terrain, extent):
    """the reference's default terrain from 2 m above the ground, the air and a grazing angle, the patches chosen by the real frustum
    cull; the near views reach factor 63 and the clip path"""
    hm, t, mm = default_terrain
    w, h = extent
    st = ht.settings(t)
    factors = set()
    ctx.clear_hiz()
    for name, cam in ht.views(hm, t, w, h).items():
        mask = np.zeros(128, np.uint32)
        visible, count = cull(ctx, t, mm, cam, abi.CULL_TEST_FRUSTUM | abi.CULL_LATE_PASS, mask)
        assert 0 < count < 4096, name
        want, n = check(ctx, so, hm, st, visible, count, cam, w, h, f"{name} {w}x{h}")
        assert (want != CLEAR).mean() > 0.3, name
        for i in visible[:count]:
            factors.update(so.patch(hm, st, cam, int(i)).n)
    assert 63 in factors and min(factors) <= 3


@pytest.mark.parametrize("grid", [(1, 1), (3, 7), (256, 256)], ids=lambda g: f"{g[0]}x{g[1]}")
def test_grids(ctx, so, grid):
    """every patch of the grid drawn from the three cameras"""
    hm = ht.heightmap(2 * grid[0] + 5, 3 * grid[1] + 2, grid[0], "noise")
    t = ht.terrain(grid, (200.0, 260.0), (-10.0, 30.0))
    n = grid[0] * grid[1]
    for name, cam in ht.views(hm, t, 320, 200).items():
        want, _ = check(ctx, so, hm, ht.settings(t), np.arange(n, dtype=np.uint32), n, cam, 320, 200, f"{grid} {name}")
        assert (want != CLEAR).any()


@pytest.mark.parametrize("target,max_tess", [(16.0, 1.0), (16.0, 3.0), (16.0, 64.0), (1.0, 64.0)])
def test_tessellation_settings(ctx, so, target, max_tess):
    hm = ht.heightmap(128, 128, 3)
    t = ht.terrain((8, 8), (256.0, 256.0), (0.0, 60.0))
    st = ht.settings(t, target, max_tess)
    cam = ht.views(hm, t, 480, 270)["grazing"]
    want, n = check(ctx, so, hm, st, np.arange(64, dtype=np.uint32), 64, cam, 480, 270, f"{target} {max_tess}")
    expect = {1.0: 2 * 64}.get(max_tess)
    if expect:
        assert n == expect


def test_early_and_late_passes(ctx, so, default_terrain):
    """the two-pass frame's terrain: the early pass draws the patches visible last frame, the late pass the newly visible ones, both
    through the real cull (occlusion against a cleared Hi-Z)"""
    hm, t, mm = default_terrain
    w, h = 640, 360
    st = ht.settings(t)
    cams = [ht.views(hm, t, w, h)["aerial"], ht.views(hm, t, w, h)["grazing"]]
    mask = np.zeros(128, np.uint32)
    ctx.clear_hiz()
    _ = cull(ctx, t, mm, cams[0], abi.CULL_TEST_FRUSTUM | abi.CULL_TEST_OCCLUSION | abi.CULL_LATE_PASS, mask)
    vis = np.full((h, w), CLEAR, np.uint64)
    counts = []
    for flags in (abi.CULL_TEST_FRUSTUM | abi.CULL_TEST_OCCLUSION, abi.CULL_TEST_FRUSTUM | abi.CULL_TEST_OCCLUSION | abi.CULL_LATE_PASS):
        visible, count = cull(ctx, t, mm, cams[1], flags, mask)
        want, _ = oracle(so, hm, st, visible, count, cams[1], w, h, vis)
        assert_same(draw(ctx, hm, st, visible, count, cams[1], w, h, vis), want, f"flags {flags:#x}")
        vis = want
        counts.append(count)
    assert sum(counts) > 0


def test_over_a_meshlet_frame_and_wide_ids(ctx, ctx_wide, so):
    """drawn over a vis buffer of meshlet words: nearer meshlets stay, farther ones are replaced, and at equal depth the terrain wins;
    the word is 0xFFFFFE00, under wide_ids 0xFFFFFF80"""
    hm = ht.heightmap(64, 64, 5)
    t = ht.terrain((8, 8), (128.0, 128.0), (0.0, 20.0))
    st = ht.settings(t, 4.0)
    cam = ht.views(hm, t, 256, 160)["aerial"]
    alone, _ = oracle(so, hm, st, np.arange(64, dtype=np.uint32), 64, cam, 256, 160)
    drawn = alone != CLEAR
    words = {8: 0xFFFFFE00, 6: 0xFFFFFF80}
    for bits, c in ((8, ctx), (6, ctx_wide)):
        rng = np.random.default_rng(bits)
        depth = (alone >> np.uint64(32)).astype(np.uint32)
        meshlet = rng.integers(0, (1 << (32 - bits)) - 2, alone.shape, dtype=np.uint64) << np.uint64(bits)  # ids below the sentinel
        kind = rng.integers(0, 3, alone.shape)
        dz = np.where(kind == 0, 0, np.where(kind == 1, 3, -3)).astype(np.int64)
        zd = np.clip(depth.astype(np.int64) + dz, 0, 0x3F800000).astype(np.uint64)
        start = np.where(drawn, (zd << np.uint64(32)) | meshlet, CLEAR).astype(np.uint64)
        want, _ = oracle(so, hm, st, np.arange(64, dtype=np.uint32), 64, cam, 256, 160, start, bits)
        got = draw(c, hm, st, np.arange(64, dtype=np.uint32), 64, cam, 256, 160, start)
        assert_same(got, want, f"prim_bits {bits}")
        tie = drawn & (kind == 0)
        assert (got[tie] & np.uint64(0xFFFFFFFF) == words[bits]).all()
        assert (got[drawn & (kind == 1)] == start[drawn & (kind == 1)]).all()
        assert set(np.unique(alone[drawn] & np.uint64(0xFFFFFFFF)).tolist()) == {0xFFFFFE00}


def test_hostile_settings_counts_and_indices(ctx, so):
    """NaN, zero and huge fov, inf / NaN inverse sizes and height scales, a camera inside the terrain, an instance count past the
    patch total and patch indices outside the grid: the device equals the oracle in each"""
    hm = ht.heightmap(32, 32, 9, "rough")
    t = ht.terrain((4, 4), (32.0, 32.0), (0.0, 8.0))
    base = ht.views(hm, t, 160, 100)
    cases = []
    for fov in (float("nan"), 0.0, 180.0, -60.0, 1e-30):
        cases.append((f"fov {fov}", ht.settings(t, 2.0, 64.0, fov), base["grazing"]))
    for field, value in (("inv_world_size", np.inf), ("inv_world_size", np.nan)):
        s = ht.settings(t, 2.0)
        s[field][0][0] = value
        cases.append((f"{field} {value}", s, base["aerial"]))
    for hs in (np.nan, np.inf, -1e30):
        tt = t.copy()
        tt["height_scale"] = hs
        cases.append((f"height_scale {hs}", ht.settings(tt, 2.0), base["aerial"]))
    inside = ht.camera(160, 100, (0.0, 4.0, 0.0), (3.0, 3.0, -5.0), near=0.01)
    cases.append(("inside", ht.settings(t, 1.0), inside))
    visible = np.arange(16, dtype=np.uint32)
    for label, st, cam in cases:
        check(ctx, so, hm, st, visible, 16, cam, 160, 100, label)
    bad = np.array([3, 16, 0xFFFFFFFF, 5, 1 << 31, 9] + list(range(10)), np.uint32)
    check(ctx, so, hm, ht.settings(t, 2.0), bad, 16, base["grazing"], 160, 100, "bad indices")
    want, _ = check(ctx, so, hm, ht.settings(t, 2.0), visible, 0xFFFFFFFF, base["grazing"], 160, 100, "count past the total")
    assert_same(want, oracle(so, hm, ht.settings(t, 2.0), visible, 16, base["grazing"], 160, 100)[0], "clamped count")
    empty, _ = check(ctx, so, hm, ht.settings(t, 2.0), visible, 0, base["grazing"], 160, 100, "count 0")
    assert (empty == CLEAR).all()


def test_refusals(capi, ctx):
    hm = ht.heightmap(16, 16, 1)
    t = ht.terrain((2, 2), (16.0, 16.0))
    d = Dev(ctx)
    hp, vp, cp, gp = d.put(hm), d.put(np.arange(4, dtype=np.uint32)), d.put(np.uint32([4, 4, 0, 0])), d.put(np.full(64 * 64, CLEAR))
    cam = ht.camera(64, 64, (0.0, 20.0, 10.0), (0.0, 0.0, 0.0))
    launches = capi.kernel_launch_count()

    def td(**kw):
        a = dict(hp=hp, rx=16, ry=16, st=ht.settings(t), vp=vp, cp=cp, cam=cam, w=64, h=64, gp=gp)
        a.update(kw)
        with pytest.raises(capi.OxcError):
            ctx.draw_terrain(a["hp"], a["rx"], a["ry"], a["st"], a["vp"], a["cp"], a["cam"], a["w"], a["h"], a["gp"])

    td(hp=None)
    td(vp=None)
    td(cp=None)
    td(gp=None)
    td(w=0)
    td(h=0)
    td(w=40000)
    td(rx=0)
    td(ry=0)
    td(rx=70000)
    td(hp=hp + 1)
    td(vp=vp + 2)
    td(cp=cp + 2)
    td(gp=gp + 4)
    for field, v in (("target_edge_pixels", np.nan), ("target_edge_pixels", np.inf), ("target_edge_pixels", 0.5), ("target_edge_pixels", -1.0),
                     ("max_tessellation", np.nan), ("max_tessellation", np.inf), ("max_tessellation", 0.99), ("max_tessellation", 0.0)):
        s = ht.settings(t)
        s[field] = v
        td(st=s)
    tt = t.copy()
    tt["patch_count"] = (0, 4)
    td(st=ht.settings(tt))
    tt["patch_count"] = (65536, 65536)
    td(st=ht.settings(tt))
    ctx.sync()
    assert capi.kernel_launch_count() == launches
    d.free()


def test_graph_capture_equals_eager(capi, ctx, so):
    """two draws captured in one CUDA graph from the first call, the instance count and the patch list changed between replays on
    the device: each replay equals the oracle with that frame's list"""
    import torch

    hm = ht.heightmap(64, 64, 11)
    t = ht.terrain((8, 8), (128.0, 128.0), (0.0, 20.0))
    st = ht.settings(t, 4.0)
    cam = ht.views(hm, t, 320, 180)["grazing"]
    w, h = 320, 180
    d = Dev(ctx)
    hp, vp, cp, gp = d.put(hm), d.put(np.zeros(64, np.uint32)), d.put(np.uint32([4, 0, 0, 0])), d.put(np.full((h, w), CLEAR))
    s = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
        gctx.draw_terrain(hp, 64, 64, st, vp, cp, cam, w, h, gp)
    rng = np.random.default_rng(2)
    for _ in range(3):
        visible = rng.permutation(64).astype(np.uint32)
        count = int(rng.integers(1, 65))
        ctx.upload(vp, visible)
        ctx.upload(cp, np.uint32([4, count, 0, 0]))
        ctx.upload(gp, np.full((h, w), CLEAR))
        g.replay()
        torch.cuda.synchronize()
        want, _ = oracle(so, hm, st, visible, count, cam, w, h)
        assert_same(d.get(gp, np.zeros((h, w), np.uint64)), want, f"count {count}")
    del g
    d.free()


@pytest.mark.parametrize("wide", [False, True], ids=["8bit", "wide"])
def test_decode_skips_terrain_texels(capi, orc, wide):
    """a shard whose id base puts the terrain's id inside its meshlet range: the decode discards the terrain texels (status 0) and
    decodes the meshlet texels beside them"""
    sc = synth.make_scene(2000, config_index=2, width=64, height=48, n_unique_meshes=4)
    hw, hh = sc.hiz_extent()
    ctx = capi.Context(0, sc.mesh_instance_count, sc.max_meshlet_instance_count, hw, hh, wide_ids=wide)
    ctx.set_scene(sc)
    cam = sc.camera(0.0)
    bits = 6 if wide else 8
    sentinel = (0xFFFFFFFF >> bits) - 1
    id_base = sentinel - 3
    base_dev = ctx.alloc(4)
    ctx.upload(base_dev, np.uint32([id_base]))
    ctx.set_shard(0, sc.mesh_instance_count, base_dev)
    ctx.cull_meshes(cam)
    w, h = 64, 48
    v32 = np.full((h, w), (id_base + 1) << bits, np.uint32)
    v32[::2, ::3] = sentinel << bits
    v32[1::4, 1::4] = 0xFFFFFFFF
    d = Dev(ctx)
    vp = d.put(v32)
    lam = d.put(np.full((h, w, 4), np.nan, np.float32))
    ctx.decode_visbuffer(cam, w, h, {"lambda_": lam}, vis32_dev=vp)
    status = d.get(lam, np.zeros((h, w, 4), np.float32))[:, :, 3]
    assert (status[::2, ::3] == 0).all()
    meshlet = (v32 == (id_base + 1) << bits)
    assert (status[meshlet] != 0).all()
    d.free()
    ctx.free(base_dev)
    ctx.close()


@pytest.fixture(scope="module")
def orc():
    import pyoracle

    return pyoracle


def _renderer_scene():
    sc = synth.make_scene(20000, config_index=2, width=640, height=360, n_unique_meshes=32)
    hm = ht.heightmap(128, 128, 13, texel_noise=0.01)
    t = ht.terrain((16, 16), (400.0, 400.0), (-30.0, -10.0))
    return sc, hm, t, ht.patch_minmax(hm, (16, 16)), ht.settings(t)


def oracle_terrain_frame(orc, so, hs, sc, cam, mask, terrain=None, tmask=None):
    """orc.frame with RendererInstance::render's terrain halves (RendererInstance.cpp:864-880): after the early meshlet raster the
    terrain cull (TestFrustum | TestOcclusion against the cleared Hi-Z) and draw, and after the late raster the late cull (| LatePass)
    against the pyramid generate_hiz builds from the early image, and its draw.  Returns (counts, vis32, depth, sorted survivors)."""
    kw = {}
    if terrain is not None:
        hm, t, mm, st = terrain
        hw, hh = abi.hiz_extent(sc.width, sc.height)
        state = {}
        flags = abi.CULL_TEST_FRUSTUM | abi.CULL_TEST_OCCLUSION

        def between(img):
            visible, cmd = orc.cull_terrain(t, mm, cam, flags, orc.Hiz(hw, hh), tmask)
            so.draw_terrain(hm, st, visible, len(visible), cam, img)
            state["hiz"] = orc.build_hiz(orc.resolve(img)[1], orc.Hiz(hw, hh))

        def after(img):
            visible, cmd = orc.cull_terrain(t, mm, cam, flags | abi.CULL_LATE_PASS, state["hiz"], tmask)
            so.draw_terrain(hm, st, visible, len(visible), cam, img)

        kw = dict(between_passes=between, after_frame=after)
    ref = orc.frame(hs, cam, sc.width, sc.height, mask, None, **kw)
    v32, d = orc.resolve(ref["vis64"])
    n = ref["early"] + ref["late"]
    return (int(ref["visibility"]["total"][0]), ref["early"], ref["late"]), v32, d, np.sort(ref["visible"][:n])


def _assert_frame(got, want, label):
    counts, v32, d, ids = want
    assert (got["total"], got["early"], got["late"]) == counts, label
    np.testing.assert_array_equal(got["vis32"], v32, err_msg=label)
    np.testing.assert_array_equal(got["depth"].view(np.uint32), d.view(np.uint32), err_msg=label)
    np.testing.assert_array_equal(np.sort(got["idx"][: got["early"] + got["late"]]), ids, err_msg=label)


def test_renderer_render_and_submit_with_terrain(capi, orc, so):
    """oxr_set_terrain: render() and submit() run the terrain cull and draw in both geometry passes and equal the oracle's two-pass
    frame with the terrain halves, frame after frame (the patch mask persists); the terrain's texels carry 0xFFFFFE00 and some
    meshlets are hidden behind it.  Removing the terrain gives the terrain-less frame bit for bit, in render() and in submit() (whose
    graphs come back); refusals leave no terrain behind."""
    sc, hm, t, mm, st = _renderer_scene()
    hs = orc.HostScene(sc)
    r = capi.Renderer(0, sc)
    mask = np.zeros((sc.max_meshlet_instance_count + 31) // 32, np.uint32)
    tmask = np.zeros(8, np.uint32)
    terrain = (hm, t, mm, st)
    bufs = [dict(vis32=np.zeros((sc.height, sc.width), np.uint32), depth=np.zeros((sc.height, sc.width), np.float32),
                 idx=np.zeros(sc.max_meshlet_instance_count, np.uint32)) for _ in range(2)]

    def submitted(cam, f):
        res = r.wait(r.submit(cam, bufs[f % 2]))
        return dict(res, **bufs[f % 2])

    for f in range(2):  # without a terrain first: the graphs are captured
        cam = sc.camera(1.5 * f)
        _assert_frame(submitted(cam, f), oracle_terrain_frame(orc, so, hs, sc, cam, mask), f"plain submit {f}")
    r.set_terrain(hm, mm, st)
    seen = 0
    for f in range(4):
        cam = sc.camera(2.0 * f)
        want = oracle_terrain_frame(orc, so, hs, sc, cam, mask, terrain, tmask)
        if f % 2 == 0:
            got = r.render(cam)
            got["idx"] = got["visible"]
        else:
            got = submitted(cam, f)
        _assert_frame(got, want, f"terrain frame {f}")
        seen += int((want[1] == 0xFFFFFE00).sum())
    assert seen > 10000
    bad = st.copy()
    bad["max_tessellation"] = np.nan
    with pytest.raises(capi.OxcError):
        r.set_terrain(hm, mm, bad)
    cam = sc.camera(9.0)
    got = r.render(cam)
    got["idx"] = got["visible"]
    _assert_frame(got, oracle_terrain_frame(orc, so, hs, sc, cam, mask), "after a refused terrain")
    r.set_terrain(hm, mm, st)
    r.set_terrain(None)
    for f in range(3):
        cam = sc.camera(3.0 + f)
        _assert_frame(submitted(cam, f), oracle_terrain_frame(orc, so, hs, sc, cam, mask), f"terrain removed {f}")
    r.close()
