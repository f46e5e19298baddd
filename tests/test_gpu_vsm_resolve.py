"""The VSM shadow resolve on the device (oxc_vsm_resolve_shadows, oxr_vsm_resolve_shadows) against the CPU oracle
(oracle/oxc_oracle_vsm_resolve.c orc_vsm_resolve_shadows), the shadow image compared bit for bit in every case."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_vsm_draw import coarse_camera
from tests.test_gpu_vsm_pages import LIGHT, Dev, _sequence_frames, clipmaps, physical_count, vsm_context

pytestmark = pytest.mark.gpu

B, D, V = abi.VSM_PAGE_BACKED, abi.VSM_PAGE_DIRTY, abi.VSM_PAGE_VISIBLE


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def vr():
    """the shadow-resolve oracle (oracle/pyoracle_vsm_resolve.py)"""
    import pyoracle_vsm_resolve

    pyoracle_vsm_resolve.build()
    return pyoracle_vsm_resolve


@pytest.fixture(scope="module")
def scene():
    return synth.make_scene(3000, config_index=2, width=640, height=360, n_unique_meshes=8)


@pytest.fixture(scope="module")
def ctx(capi, scene):
    hw, hh = scene.hiz_extent()
    c = capi.Context(0, scene.mesh_instance_count, scene.max_meshlet_instance_count, hw, hh, max_views=10)
    c.set_scene(scene)
    yield c
    c.close()


def inverse_pv(cam):
    return np.linalg.inv(cam["projection_view"][0].reshape(4, 4).T.astype(np.float64)).T.astype(np.float32).reshape(16)


def random_inputs(rng, scene, vsm, hostile=True):
    """a camera of the synthetic scene, random depth (a third sky, hostile values), random unit normals oct-encoded in .zw (random
    .xy), random tables with Backed entries pointing anywhere in the atlas and beyond it, an atlas of depths, cleared texels and -1"""
    w, h = int(vsm["depth_extent"][0][0]), int(vsm["depth_extent"][0][1])
    layers, size, P = int(vsm["clipmap_count"][0]), int(vsm["page_table_size"][0]), int(vsm["physical_page_table_size"][0])
    cam = scene.camera(1.0)
    depth = (rng.random((h, w)) ** 3).astype(np.float32)
    depth[rng.random((h, w)) < 0.3] = 0.0
    if hostile:
        k = rng.random((h, w))
        depth[k < 0.01] = np.float32(np.nan)
        depth[(k >= 0.01) & (k < 0.02)] = np.float32(np.inf)
        depth[(k >= 0.02) & (k < 0.03)] = np.float32(1e-40)
    n = rng.normal(size=(h, w, 3))
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    p = n[..., :2] / np.abs(n).sum(-1, keepdims=True)
    sgn = np.where(p >= 0, 1.0, -1.0)
    oct_ = np.where(n[..., 2:3] <= 0, (1 - np.abs(p[..., ::-1])) * sgn, p)
    normals = np.zeros((h, w, 4), np.float32)
    normals[..., :2] = rng.random((h, w, 2))
    normals[..., 2:] = oct_
    normals[depth == 0] = 0.0
    if hostile:
        normals[5, :20, 2] = [np.nan, np.inf, -np.inf, 1e-40, 70000.0, -0.0, 1.5, -1.5, 0.0, 2.0] * 2
    state = rng.integers(0, 32, size=(layers, size, size)).astype(np.uint32)
    state[rng.random(state.shape) < 0.7] |= B
    phys = rng.integers(0, physical_count(vsm) + physical_count(vsm) // 16, size=state.shape).astype(np.uint32)
    pt = (state | (phys << 16)).astype(np.uint32)
    atlas = rng.random((P, P)).astype(np.float32)
    atlas[rng.random((P, P)) < 0.3] = 1.0
    atlas[rng.random((P, P)) < 0.01] = -1.0
    return cam, depth, normals, pt, atlas


def run_device(ctx, vsm, inv_pv, res, cm, depth, normals, pt, atlas):
    d = Dev(ctx)
    w, h = int(vsm["depth_extent"][0][0]), int(vsm["depth_extent"][0][1])
    out = d.put(np.zeros((h, w), np.float32))
    ctx.vsm_resolve_shadows(vsm, inv_pv, res, cm, d.put(depth), d.put(normals), d.put(pt), d.put(atlas), out)
    got = ctx.download(out, np.float32, w * h).reshape(h, w)
    d.free()
    return got


@pytest.mark.parametrize("shape", ["reference", "uneven"])
def test_random_cases(ctx, vr, scene, shape):
    """random depth, normals, tables and atlases at 640 x 360 over all ten clipmaps with uneven page offsets; the reference's atlas
    shape (128-px pages, 8192^2) and a smaller non-reference one (64-px pages, 2048^2, 24 x 24 tables) with one clipmap that is not
    orthographic"""
    rng = np.random.default_rng(21 if shape == "reference" else 22)
    if shape == "reference":
        vsm = vsm_context(width=640, height=360)
        cm = clipmaps(10, rng, center=(6.0, -2.0, -115.0))
    else:
        vsm = vsm_context(size=24, page_size=64, physical=2048, width=640, height=360)
        cm = clipmaps(10, rng, center=(6.0, -2.0, -115.0))
        cm["projection_view_mat"][3][3] = np.float32(1.0001)  # row 3 != (0, 0, 0, 1): the divides are taken
        cm["projection_view_mat"][5][7] = np.float32(1e-4)
    cam, depth, normals, pt, atlas = random_inputs(rng, scene, vsm)
    inv_pv, res = inverse_pv(cam), cam["resolution"][0]
    want, pcf = vr.vsm_resolve_shadows(vsm, inv_pv, res, cm, depth, normals, pt, atlas)
    got = run_device(ctx, vsm, inv_pv, res, cm, depth, normals, pt, atlas)
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    inner = (want > 0) & (want < 1)
    assert pcf.sum() > 100 and inner.sum() > 100 and (want == 0).sum() > 100 and (want == 1).sum() > 100
    print(f"{shape}: pcf pixels {int(pcf.sum())}, penumbra {int(inner.sum())}")


def test_argument_refusals(capi, ctx):
    vsm = vsm_context(width=64, height=32)
    d = Dev(ctx)
    buf = d.put(np.zeros(1 << 16, np.uint32))
    cm = clipmaps(10)
    ipv, res = np.eye(4, dtype=np.float32).reshape(16), np.float32([64, 32])

    def refused(fn, match):
        with pytest.raises(capi.OxcError, match=match) as e:
            fn()
        assert "(-1)" in str(e.value)

    def bad(**kw):
        v = vsm.copy()
        for k, x in kw.items():
            v[k] = x
        return v

    for v, match in ((bad(clipmap_count=0), "clipmap_count"), (bad(clipmap_count=11), "clipmap_count"), (bad(page_size=100), "does not divide"),
                     (bad(page_size=16), "65536"), (bad(page_table_size=0), "page_table_size"), (bad(depth_extent=(0, 32)), "depth_extent")):
        refused(lambda: ctx.vsm_resolve_shadows(v, ipv, res, cm, buf, buf, buf, buf, buf), match)
    for k in range(5):
        args = [buf] * 5
        args[k] = None
        refused(lambda: ctx.vsm_resolve_shadows(vsm, ipv, res, cm, *args), "null")
    refused(lambda: ctx.vsm_resolve_shadows(vsm, ipv, res, cm, buf, buf + 4, buf, buf, buf), "aligned")
    d.free()


def test_graph_capture_equals_eager(capi, ctx, scene):
    """the resolve captured into a CUDA graph at its first call and replayed with new depth equals eager runs"""
    import torch

    rng = np.random.default_rng(5)
    vsm = vsm_context(size=32, page_size=64, physical=2048, width=640, height=360)
    cm = clipmaps(10, rng, center=(6.0, -2.0, -115.0))
    cam, depth0, normals, pt, atlas = random_inputs(rng, scene, vsm, hostile=False)
    depth1 = np.roll(depth0, 11, axis=0)
    inv_pv, res = inverse_pv(cam), cam["resolution"][0]
    eager = [run_device(ctx, vsm, inv_pv, res, cm, dep, normals, pt, atlas) for dep in (depth0, depth1)]
    d = Dev(ctx)
    bufs = [d.put(depth0), d.put(normals), d.put(pt), d.put(atlas), d.put(np.zeros((360, 640), np.float32))]
    s = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
        gctx.vsm_resolve_shadows(vsm, inv_pv, res, cm, *bufs)
    for k, dep in enumerate((depth0, depth1)):
        ctx.upload(bufs[0], dep)
        g.replay()
        torch.cuda.synchronize()
        np.testing.assert_array_equal(ctx.download(bufs[4], np.float32, 640 * 360).reshape(360, 640).view(np.uint32), eager[k].view(np.uint32))
    assert not np.array_equal(eager[0], eager[1])
    del g
    d.free()


def test_full_chain_through_renderer_full_size(capi, orc, vr):
    """frames of the VSM sequence at 1920 x 1080 with the reference's shape (64 x 64 pages x 10 clipmaps, 128-px pages, 8192^2 atlas):
    oxr_render, oxr_vsm_update_pages, oxr_vsm_draw_shadows, oxr_vsm_resolve_shadows.  Every frame the shadow image equals the oracle
    resolve over the oracle's decode of the oracle frame (normals), the frame's depth, and the renderer's page table and atlas; the
    resolve leaves the atlas and the page table as they were."""
    sc = synth.make_scene(20000, config_index=2, width=1920, height=1080, n_unique_meshes=32)
    hs = orc.HostScene(sc)
    r = capi.Renderer(0, sc)
    vsm = vsm_context()
    coarse = coarse_camera(sc.mesh_instance_count)
    mask = np.zeros(r.ctx.out.visibility_mask_words, dtype=np.uint32)
    lit_mix = []
    for f, fr in enumerate(_sequence_frames(sc, 4)):
        cam = sc.camera(fr["yaw"])
        out = r.render(cam, want_indices=False)
        ref = orc.frame(hs, cam, 1920, 1080, mask, None)
        v32, depth = orc.resolve(ref["vis64"])
        np.testing.assert_array_equal(out["depth"].view(np.uint32), depth.view(np.uint32))
        inv_pv, res = inverse_pv(cam), cam["resolution"][0]
        pg = r.vsm_update_pages(vsm, fr["clip"], inv_pv, res, sun_moved=fr["sun_moved"], hpb_levels=7)
        r.vsm_draw_shadows(coarse)
        pt = r.ctx.download(pg.page_tables, np.uint32, 10 * 64 * 64).reshape(10, 64, 64)
        atlas = r.ctx.download(pg.physical_atlas, np.float32, 8192 * 8192).reshape(8192, 8192)
        got = r.vsm_resolve_shadows(cam)
        normals = orc.decode_visbuffer(hs, ref["meshlet_instances"], int(ref["visibility"]["total"][0]), cam, v32)["uv_normal"]
        want, pcf = vr.vsm_resolve_shadows(vsm, inv_pv, res, fr["clip"], depth, normals, pt, atlas)
        np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32), err_msg=f"frame {f}")
        np.testing.assert_array_equal(r.ctx.download(pg.page_tables, np.uint32, pt.size).reshape(pt.shape), pt)
        np.testing.assert_array_equal(r.ctx.download(pg.physical_atlas, np.float32, 8192 * 8192).reshape(8192, 8192).view(np.uint32), atlas.view(np.uint32))
        lit_mix.append(((got == 0).sum(), ((got > 0) & (got < 1)).sum(), int(pcf.sum())))
        print(f"frame {f}: shadowed {lit_mix[-1][0]}, penumbra {lit_mix[-1][1]}, pcf pixels {lit_mix[-1][2]}")
    assert sum(m[0] for m in lit_mix) > 1000 and sum(m[1] for m in lit_mix) > 100
    r.close()


def test_next_camera_frame_unchanged(capi):
    """oxr_render after oxr_vsm_resolve_shadows gives bit for bit what it gives without it, and oxr_overdraw still sees the last frame"""
    sc = synth.make_scene(4000, config_index=2, width=640, height=360, n_unique_meshes=8)
    vsm = vsm_context(width=640, height=360)
    coarse = coarse_camera(sc.mesh_instance_count)
    outs = []
    for resolve in (False, True):
        r = capi.Renderer(0, sc)
        with pytest.raises(capi.OxcError, match="(-5)"):
            r.vsm_resolve_shadows(sc.camera(0.0))  # before an update
        r.close()
        r = capi.Renderer(0, sc)
        o = []
        for f, fr in enumerate(_sequence_frames(sc, 3)):
            cam = sc.camera(fr["yaw"])
            out = r.render(cam)
            r.vsm_update_pages(vsm, fr["clip"], inverse_pv(cam), cam["resolution"][0], sun_moved=fr["sun_moved"], hpb_levels=7)
            r.vsm_draw_shadows(coarse)
            if resolve:
                r.vsm_resolve_shadows(cam)
            o.append((out["vis32"].copy(), out["depth"].copy(), np.sort(out["visible"]), r.overdraw(cam)))
        outs.append(o)
        r.close()
    for a, b in zip(*outs):
        for x, y in zip(a, b):
            np.testing.assert_array_equal(x, y)


def _two_sided_grid(n, y):
    """an n x n quad grid over [-1, 1]^2 at height y (x, z), normals +y, both windings (the camera cull keeps one of each pair)"""
    g = np.linspace(-1.0, 1.0, n + 1)
    gx, gz = np.meshgrid(g, g, indexing="ij")
    pos = np.stack([gx.reshape(-1), np.full(gx.size, y), gz.reshape(-1)], 1).astype(np.float32)
    v = (np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]).reshape(-1)
    tri = np.concatenate([np.stack([v, v + 1, v + n + 2], 1), np.stack([v, v + n + 2, v + n + 1], 1)])
    idx = np.concatenate([tri, tri[:, ::-1]]).astype(np.uint32).reshape(-1)
    nrm = np.tile(np.float32([0.0, 1.0, 0.0]), (len(pos), 1))
    return pos, idx, nrm


def test_analytic_square_over_ground(capi):
    """no oracle: a ground plane (y = 0, 200 m square) and a floating 8 m square at height 5 built with oxb_*, light travelling along
    D = (0.8, -1, 0.1) (directional_light_dir = -D, pointing at the light as the reference's; the clipmaps look along D, forward Z), with
    the page offsets of the reference's page-snapped clipmaps, through oxr_render -> oxr_vsm_update_pages -> oxr_vsm_draw_shadows -> oxr_vsm_resolve_shadows.  A ground
    pixel whose world point, moved along -D up to the square's height, lands deeper inside the square than the PCSS radius plus two
    base-clipmap texels (and the normal offset) is 0; one that lands as far outside it is 1.  Catches a y flip, a depth-direction or a
    page-wrap error that the oracle and the kernel would share."""
    W, H, HS, SQ, HY = 640, 360, 8.0, np.float64([0.0, -28.0]), 5.0  # image, square half size 4 -> HS = side, centre (x, z), height
    D = np.float64([0.8, -1.0, 0.1])  # the light travels along D
    gp, gi, gn = _two_sided_grid(32, 0.0)
    sp, si, sn = _two_sided_grid(4, 0.0)
    ground = capi.BuiltMesh(gp, [(gi, 0.0)], normals=gn)
    square = capi.BuiltMesh(sp, [(si, 0.0)], normals=sn)
    xf = np.zeros((2, 16), np.float32)
    xf[0] = np.diag([100.0, 1.0, 100.0, 1.0]).T.reshape(16)
    xf[0, 12:15] = (0.0, 0.0, -30.0)
    xf[1] = np.diag([HS / 2, 1.0, HS / 2, 1.0]).T.reshape(16)
    xf[1, 12:15] = (SQ[0], HY, SQ[1])
    sc = capi.assemble_scene([ground, square], [0, 1], xf, W, H)
    eye = np.float64([0.0, 40.0, -18.0])
    cam = np.zeros(1, dtype=abi.CULL_CAMERA_DT)
    cam["projection_view"][0] = synth.mat_mul_cm(synth.perspective_reverse_z(60.0, W / H, 0.1, 1000.0), synth.look_at(eye, (0.0, 0.0, -30.0), (0.0, 1.0, 0.0)))
    cam["position"][0] = eye
    cam["acceptable_lod_error"], cam["near_clip"], cam["mesh_instance_count"] = 2.0, 0.1, sc.mesh_instance_count
    cam["resolution"][0] = (W, H)
    vsm = vsm_context(width=W, height=H)
    vsm["directional_light_dir"][0] = -D
    cm = synth.make_vsm_clipmaps(-D, eye)  # forward-Z, page offsets from the camera position, as Shadowmaps.cpp:9-60 builds them
    assert len(set(map(tuple, cm["page_offset"]))) > 3
    coarse = np.zeros(1, dtype=abi.CULL_CAMERA_DT)  # clipmap 9's view (Shadowmaps.cpp:433-463)
    coarse["projection_view"][0] = cm["projection_view_mat"][9]
    coarse["position"][0] = -D / np.linalg.norm(D)
    coarse["acceptable_lod_error"], coarse["near_clip"], coarse["mesh_instance_count"] = 2.0, 0.0, sc.mesh_instance_count
    coarse["resolution"][0] = (8192, 8192)
    r = capi.Renderer(0, sc)
    out = r.render(cam)
    inv_pv = inverse_pv(cam)
    r.vsm_update_pages(vsm, cm, inv_pv, cam["resolution"][0], sun_moved=True, hpb_levels=7)
    r.vsm_draw_shadows(coarse)
    shadow = r.vsm_resolve_shadows(cam)
    r.close()
    # world point of every pixel (binary64), and the base clipmap's texel from the pixel footprint (rmvsm.slang:156-188)
    depth = out["depth"].astype(np.float64)
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    ipv = inv_pv.reshape(4, 4).T.astype(np.float64)

    def unproj(u, v):
        p = np.stack([u * 2 - 1, v * 2 - 1, depth, np.ones_like(depth)], -1) @ ipv.T
        return p[..., :3] / p[..., 3:4]

    u, v = (xs + 0.5) / W, (ys + 0.5) / H
    world = unproj(u, v)
    foot = np.linalg.norm(unproj(u - 0.5 / W, v + 0.5 / H) - unproj(u + 0.5 / W, v + 0.5 / H), axis=-1)
    texel = 10.0 * (63.0 / 64.0) * 2.0 / 8192.0
    ci = np.clip(np.ceil(0.25 + np.maximum(np.log2(np.maximum(foot * 1.001, 1e-30) / texel), 0.0)), 0, 9)  # rounded up at a boundary
    cts = 2.0 ** (ci + 1) * texel                               # clipmap_texel_size = two texels of the base clipmap
    ground_px = (depth != 0) & (np.abs(world[..., 1]) < 0.05)
    q = world[..., [0, 2]] + (HY / -D[1]) * -D[[0, 2]]           # along -D (towards the light) up to the square's height
    inside = np.min(HS / 2 - np.abs(q - SQ), axis=-1)            # > 0 inside the square's outline
    # PCSS radius 0.1 + two texels + the normal offset (cts along +y moves the point cts * |D.xz| / |D.y| across the outline) + half a
    # texel for the raster's coverage of the square's edge
    margin = 0.1 + cts + cts * np.linalg.norm(D[[0, 2]]) / -D[1] + 0.25 * cts
    deep = ground_px & (inside > margin)
    far = ground_px & (inside < -margin)
    assert deep.sum() > 500 and far.sum() > 10000, (deep.sum(), far.sum())
    assert (shadow[deep] == 0.0).all(), f"{int((shadow[deep] != 0).sum())} of {int(deep.sum())} pixels deep in the shadow are lit"
    assert (shadow[far] == 1.0).all(), f"{int((shadow[far] != 1).sum())} of {int(far.sum())} pixels outside the shadow are shadowed"
    # values in (0, 1) (the PCF's) appear only near the outline
    band = ground_px & (shadow > 0) & (shadow < 1)
    assert (np.abs(inside[band]) <= margin[band]).all()
    print(f"analytic: deep {int(deep.sum())}, far {int(far.sum())}, penumbra {int(band.sum())}")
