"""The vis-buffer decode into the G-buffer on the device (oxc_decode_gbuffer, oxr_decode_gbuffer) against the CPU oracle
(oracle/oxc_oracle_gbuffer.c orc_decode_gbuffer), all four planes compared bit for bit."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_parity import _assert_planes_equal, _frame_gpu, make_ctx

pytestmark = pytest.mark.gpu

PLANES = abi.GBUFFER_PLANES
IMAGE_FLAGS = (abi.MATERIAL_HAS_ALBEDO_IMAGE, abi.MATERIAL_HAS_NORMAL_IMAGE, abi.MATERIAL_HAS_EMISSIVE_IMAGE,
               abi.MATERIAL_HAS_METALLIC_ROUGHNESS_IMAGE, abi.MATERIAL_HAS_OCCLUSION_IMAGE)
SLOTS = ("albedo_image_index", "normal_image_index", "emissive_image_index", "metallic_roughness_image_index", "occlusion_image_index")


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def gb():
    import pyoracle_gbuffer

    pyoracle_gbuffer.build()
    return pyoracle_gbuffer


def half(x):
    return int(np.float16(x).view(np.uint16))


def random_images(rng, n=10):
    """every format, single levels and full mip chains, square, non-square and odd sizes"""
    import pyoracle as orc

    out = []
    for i in range(n):
        fmt = (abi.IMAGE_RGBA8_UNORM, abi.IMAGE_RGBA8_SRGB, abi.IMAGE_R8_UNORM, abi.IMAGE_RG8_UNORM)[i % 4]
        w, h = [(16, 16), (8, 32), (7, 5), (64, 16), (3, 9), (32, 32), (1, 6), (13, 13), (64, 64), (5, 2)][i % 10]
        ch = {abi.IMAGE_R8_UNORM: (), abi.IMAGE_RG8_UNORM: (2,)}.get(fmt, (4,))
        l0 = rng.integers(0, 256, (h, w) + ch, dtype=np.uint8)
        out.append((orc.mip_chain(l0) if i % 3 != 2 else l0, fmt))
    return out


def random_samplers(rng):
    """every filter, mipmap and address mode"""
    s = np.zeros(12, dtype=abi.SAMPLER_DT)
    for i in range(12):
        s[i] = (i & 1, (i >> 1) & 1, (i >> 2) & 1, i % 3, (i + 1) % 3)
    return s


def random_materials(rng, n, n_images, n_samplers):
    """every subset of the five image flags, with FlipY / TwoComponent, uv_size / uv_offset including negative values"""
    m = np.zeros(n, dtype=abi.MATERIAL_DT)
    for i in range(n):
        flags = i % 32
        if rng.random() < 0.5:
            flags |= abi.MATERIAL_NORMAL_FLIP_Y
        if rng.random() < 0.5:
            flags |= abi.MATERIAL_NORMAL_TWO_COMPONENT
        m[i]["flags"] = flags
        m[i]["albedo_color"] = [half(x) for x in rng.uniform(0.2, 1.5, 4)]
        m[i]["emissive_color"] = [half(x) for x in rng.uniform(0.0, 4.0, 3)]
        m[i]["metallic_factor"], m[i]["roughness_factor"] = half(rng.uniform(0, 1)), half(rng.uniform(0, 1))
        m[i]["sampler_index"] = rng.integers(0, n_samplers + 2)  # beyond the table: linear, linear, repeat
        for s in SLOTS:
            m[i][s] = rng.integers(0, n_images)
        while m[i]["albedo_image_index"] % 4 == 3:  # the alpha test refuses RG8_UNORM (random_images: format = index % 4)
            m[i]["albedo_image_index"] = rng.integers(0, n_images)
        m[i]["uv_size"] = [half(rng.choice([1.0, 2.5, -1.0, 0.25, 3.0])), half(rng.choice([1.0, -2.0, 0.5, 4.0]))]
        m[i]["uv_offset"] = [half(rng.uniform(-2, 2)), half(rng.uniform(-2, 2))]
    return m


class Table:
    """a random material table, as the oracle's host table and on the device"""

    def __init__(self, ctx, seed, n_materials=48):
        import pyoracle as orc

        rng = np.random.default_rng(seed)
        self.images = random_images(rng)
        self.samplers = random_samplers(rng)
        self.materials = random_materials(rng, n_materials, len(self.images), len(self.samplers))
        self.host = orc.MaterialTable(self.materials, self.images, self.samplers)
        self.dev_images, self.ptrs = self.host.device_images(ctx)
        self.ctx = ctx

    def set(self, ctx=None):
        (ctx or self.ctx).set_materials(self.materials, self.dev_images, self.samplers)

    def free(self):
        for p in self.ptrs:
            self.ctx.free(p)


def scene_with_materials(n_instances, n_materials, seed, **kw):
    sc = synth.make_scene(n_instances, **kw)
    sc.mesh_instances["material_index"] = np.random.default_rng(seed).integers(0, n_materials, sc.mesh_instance_count)
    return sc


def decode_gpu(ctx, cam, w, h, planes=PLANES, vis64_dev=None, vis32_dev=None, init=0.0):
    dev = {k: ctx.alloc(w * h * 16) for k in planes}
    for p in dev.values():
        ctx.upload(p, np.full(w * h * 4, init, np.float32))
    ctx.decode_gbuffer(cam, w, h, dev, vis64_dev=vis64_dev, vis32_dev=vis32_dev)
    out = {k: ctx.download(p, np.float32, w * h * 4).reshape(h, w, 4) for k, p in dev.items()}
    for p in dev.values():
        ctx.free(p)
    return out


def gpu_frame(capi, orc, sc, ctx, cam):
    """the two-pass frame on the device; returns (host scene, dict(meshlet_instances, vis64) of that frame, vis64 device buffer,
    total).  The decode is compared on the device's own vis buffer; cull_meshes is the same on both sides."""
    hs = orc.HostScene(sc)
    w, h = sc.width, sc.height
    vis_dev = ctx.alloc(w * h * 8)
    _frame_gpu(capi, ctx, sc, cam, None, vis_dev)
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    np.testing.assert_array_equal(ctx.meshlet_instances(int(vis["total"][0])), mi[: int(vis["total"][0])])
    return hs, dict(meshlet_instances=mi, vis64=ctx.download(vis_dev, np.uint64, w * h).reshape(h, w)), vis_dev, int(vis["total"][0])


def check_frame(capi, orc, gb, sc, seed, vis32_too=True):
    ctx = make_ctx(capi, sc)
    tab = Table(ctx, seed)
    tab.set()
    w, h = sc.width, sc.height
    cam = sc.camera(0.0)
    hs, ref, vis_dev, total = gpu_frame(capi, orc, sc, ctx, cam)
    v32, _ = orc.resolve(ref["vis64"])
    sentinel = np.float32(-7.25)
    want, bad = gb.decode_gbuffer(hs, ref["meshlet_instances"], total, cam, v32, tab.host, init=sentinel)
    assert bad == 0
    got = decode_gpu(ctx, cam, w, h, vis64_dev=vis_dev, init=sentinel)
    for k in PLANES:
        _assert_planes_equal(got[k], want[k], k)
    decoded = (want["albedo"][:, :, 0] != sentinel).sum()
    assert decoded > 1000 and (want["albedo"][:, :, 0] == sentinel).sum() > 0
    if vis32_too:
        v32_dev = ctx.alloc(w * h * 4)
        ctx.upload(v32_dev, v32)
        got = decode_gpu(ctx, cam, w, h, vis32_dev=v32_dev, init=sentinel)
        for k in PLANES:
            _assert_planes_equal(got[k], want[k], k + " (vis32)")
        ctx.free(v32_dev)
    ctx.free(vis_dev)
    tab.free()
    ctx.close()
    return want


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_tables_bit_exact(capi, orc, gb, seed):
    """seeded random tables (every image-flag subset, every format, filter, mipmap and address mode, mip chains, odd sizes, negative
    uv transforms) on a 640 x 360 frame, from the packed vis buffer and from the R32UI attachment"""
    sc = scene_with_materials(200_000, 48, seed, config_index=2, width=640, height=360, n_unique_meshes=16)
    check_frame(capi, orc, gb, sc, seed)


def test_config1_1080p_and_4k(capi, orc, gb):
    """the benchmark's scene (BASELINE.json configs[1]: 1 M meshlet instances) at 1920 x 1080, and one 3840 x 2160 frame"""
    for w, h, vis32 in ((1920, 1080, True), (3840, 2160, False)):
        sc = scene_with_materials(1_000_000, 48, 7, config_index=2, width=w, height=h)
        check_frame(capi, orc, gb, sc, 11, vis32_too=vis32)


def test_null_targets_and_normal_plane(capi, orc, gb):
    """every combination of NULL targets equals the matching planes of the full call; normal.zw equals oxc_decode_visbuffer's
    uv_normal.zw bit for bit, and oxc_vsm_resolve_shadows fed the new plane equals the same call fed the decode's plane"""
    from tests.test_gpu_vsm_pages import clipmaps, vsm_context
    from tests.test_gpu_vsm_resolve import inverse_pv

    sc = scene_with_materials(200_000, 48, 4, config_index=2, width=640, height=360, n_unique_meshes=16)
    ctx = make_ctx(capi, sc, views=10)
    tab = Table(ctx, 4)
    tab.set()
    w, h = sc.width, sc.height
    cam = sc.camera(0.0)
    hs, ref, vis_dev, total = gpu_frame(capi, orc, sc, ctx, cam)
    full = decode_gpu(ctx, cam, w, h, vis64_dev=vis_dev)
    for mask in range(1, 15):
        planes = [k for i, k in enumerate(PLANES) if mask & (1 << i)]
        part = decode_gpu(ctx, cam, w, h, planes=planes, vis64_dev=vis_dev)
        for k in planes:
            _assert_planes_equal(part[k], full[k], f"{k} of {planes}")
    un_dev = ctx.alloc(w * h * 16)
    ctx.decode_visbuffer(cam, w, h, {"uv_normal": un_dev}, vis64_dev=vis_dev)
    un = ctx.download(un_dev, np.float32, w * h * 4).reshape(h, w, 4)
    _assert_planes_equal(full["normal"][:, :, 2:], un[:, :, 2:], "normal.zw")
    assert (full["normal"][:, :, 0] != full["normal"][:, :, 2]).sum() > 1000  # the normal maps move .xy
    # the resolve fed either plane
    rng = np.random.default_rng(8)
    vsm = vsm_context(size=32, page_size=64, physical=2048, width=w, height=h)
    cm = clipmaps(10, rng, center=(6.0, -2.0, -115.0))
    depth_dev, shadow = ctx.alloc(w * h * 4), []
    ctx.resolve_visbuffer(vis_dev, w, h, None, depth_dev)
    pt = (rng.integers(0, 64, (10, 32, 32), dtype=np.uint32) << 16) | np.uint32(abi.VSM_PAGE_BACKED)
    atlas = rng.uniform(0, 1, (2048, 2048)).astype(np.float32)
    pt_dev, atlas_dev, sh_dev, n_dev = ctx.alloc(pt.nbytes), ctx.alloc(atlas.nbytes), ctx.alloc(w * h * 4), ctx.alloc(w * h * 16)
    ctx.upload(pt_dev, pt)
    ctx.upload(atlas_dev, atlas)
    for plane in (un, full["normal"]):
        ctx.upload(n_dev, np.ascontiguousarray(plane))
        ctx.vsm_resolve_shadows(vsm, inverse_pv(cam), cam["resolution"][0], cm, depth_dev, n_dev, pt_dev, atlas_dev, sh_dev)
        shadow.append(ctx.download(sh_dev, np.float32, w * h))
    np.testing.assert_array_equal(shadow[0].view(np.uint32), shadow[1].view(np.uint32))
    for p in (vis_dev, un_dev, depth_dev, pt_dev, atlas_dev, sh_dev, n_dev):
        ctx.free(p)
    tab.free()
    ctx.close()


def test_srgb_albedo_keeps_the_alpha_test(capi, orc):
    """the alpha-tested vis buffer is bit-identical with the albedo image given as RGBA8_SRGB or as RGBA8_UNORM (same texels)"""
    sc = scene_with_materials(200_000, 4, 5, config_index=2, width=640, height=360, n_unique_meshes=16)
    rng = np.random.default_rng(5)
    tex = orc.mip_chain(rng.integers(0, 256, (32, 32, 4), dtype=np.uint8))
    m = np.zeros(4, dtype=abi.MATERIAL_DT)
    for i in range(4):
        m[i]["flags"] = abi.MATERIAL_HAS_ALBEDO_IMAGE if i % 2 == 0 else 0
        m[i]["albedo_color"] = [half(1.0)] * 4
        m[i]["alpha_cutoff"] = half(0.5)
    images = []
    for fmt in (abi.IMAGE_RGBA8_UNORM, abi.IMAGE_RGBA8_SRGB):
        ctx = make_ctx(capi, sc)
        dev, ptrs = orc.MaterialTable(m, [(tex, fmt)]).device_images(ctx)
        ctx.set_materials(m, dev)
        vis_dev = ctx.alloc(sc.width * sc.height * 8)
        _frame_gpu(capi, ctx, sc, sc.camera(0.0), None, vis_dev)
        images.append(ctx.download(vis_dev, np.uint64, sc.width * sc.height))
        for p in ptrs + [vis_dev]:
            ctx.free(p)
        ctx.close()
    assert (images[0] != images[0][0]).any()
    np.testing.assert_array_equal(images[0], images[1])


def test_bad_material_and_refusals(capi, orc, gb):
    """an out-of-range material_index writes zeros and raises OXC_STATUS_BAD_MATERIAL; no table, a flagged image outside the table,
    a misaligned target, a zero extent and both or neither vis input are refused"""
    sc = scene_with_materials(200_000, 48, 6, config_index=2, width=640, height=360, n_unique_meshes=16)
    sc.mesh_instances["material_index"][::3] = 1000
    ctx = make_ctx(capi, sc)
    w, h = sc.width, sc.height
    cam = sc.camera(0.0)
    hs, ref, vis_dev, total = gpu_frame(capi, orc, sc, ctx, cam)
    out = ctx.alloc(w * h * 16 + 16)
    with pytest.raises(capi.OxcError, match="oxc_set_materials first"):
        ctx.decode_gbuffer(cam, w, h, {"albedo": out}, vis64_dev=vis_dev)
    tab = Table(ctx, 6)
    tab.set()
    ctx.status_flags()
    v32, _ = orc.resolve(ref["vis64"])
    want, bad = gb.decode_gbuffer(hs, ref["meshlet_instances"], total, cam, v32, tab.host)
    assert bad > 100
    got = decode_gpu(ctx, cam, w, h, vis64_dev=vis_dev)
    for k in PLANES:
        _assert_planes_equal(got[k], want[k], k)
    assert ctx.status_flags() & abi.STATUS_BAD_MATERIAL
    for kw in ({}, {"vis64_dev": vis_dev, "vis32_dev": vis_dev}):
        with pytest.raises(capi.OxcError, match="exactly one"):
            ctx.decode_gbuffer(cam, w, h, {"albedo": out}, **kw)
    with pytest.raises(capi.OxcError, match="16-byte aligned"):
        ctx.decode_gbuffer(cam, w, h, {"normal": out + 4}, vis64_dev=vis_dev)
    with pytest.raises(capi.OxcError, match="empty extent"):
        ctx.decode_gbuffer(cam, 0, h, {"albedo": out}, vis64_dev=vis_dev)
    bad_mats = tab.materials.copy()
    bad_mats[3]["flags"] |= abi.MATERIAL_HAS_EMISSIVE_IMAGE
    bad_mats[3]["emissive_image_index"] = 99
    ctx.set_materials(bad_mats, tab.dev_images, tab.samplers)  # accepted: the encode reads the albedo slot only
    with pytest.raises(capi.OxcError, match="material 3: emissive image 99"):
        ctx.decode_gbuffer(cam, w, h, {"albedo": out}, vis64_dev=vis_dev)
    ctx.set_materials(None)
    with pytest.raises(capi.OxcError, match="oxc_set_materials first"):
        ctx.decode_gbuffer(cam, w, h, {"albedo": out}, vis64_dev=vis_dev)
    for p in (vis_dev, out):
        ctx.free(p)
    tab.free()
    ctx.close()


def test_graph_capture_equals_eager(capi, orc):
    """the decode captured into a CUDA graph as the context's first decode, then replayed, equals the eager call that follows"""
    import torch

    sc = scene_with_materials(200_000, 48, 9, config_index=2, width=640, height=360, n_unique_meshes=16)
    ctx = make_ctx(capi, sc)
    tab = Table(ctx, 9)
    tab.set()
    w, h = sc.width, sc.height
    cam = sc.camera(0.0)
    hs, ref, vis_dev, total = gpu_frame(capi, orc, sc, ctx, cam)
    dev = {k: ctx.alloc(w * h * 16) for k in PLANES}
    s = torch.cuda.Stream()
    gctx = capi.Context.from_handle(ctx.h.value, stream=s.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
        gctx.decode_gbuffer(cam, w, h, dev, vis64_dev=vis_dev)
    g.replay()
    torch.cuda.synchronize()
    eager = decode_gpu(ctx, cam, w, h, vis64_dev=vis_dev)
    for k in PLANES:
        _assert_planes_equal(ctx.download(dev[k], np.float32, w * h * 4).reshape(h, w, 4), eager[k], k)
    assert (eager["albedo"][:, :, 3] != 0).sum() > 1000
    del g
    for p in list(dev.values()) + [vis_dev]:
        ctx.free(p)
    tab.free()
    ctx.close()


def test_renderer_decode_gbuffer(capi, orc):
    """oxr_decode_gbuffer after oxr_render equals the context call on that frame's vis buffer, and the next camera frame equals the
    one a renderer without the decode produces after the same frames"""
    sc = scene_with_materials(200_000, 48, 10, config_index=2, width=640, height=360, n_unique_meshes=16)
    cam0, cam1 = sc.camera(0.0), sc.camera(1.5)
    renderers, tables = [capi.Renderer(0, sc), capi.Renderer(0, sc)], []
    for r in renderers:
        tables.append(Table(r.ctx, 10))
        r.set_materials(tables[-1].materials, tables[-1].dev_images, tables[-1].samplers)
    last = []
    for k, r in enumerate(renderers):
        r.render(cam0, want_indices=False)
        r.render(cam1, want_indices=False)
        v32 = r.render(cam0, want_indices=False)["vis32"].copy()
        if k == 0:
            got = r.decode_gbuffer(cam0)
        last.append(r.render(cam1, want_indices=False)["vis32"].copy())
    np.testing.assert_array_equal(last[0], last[1])
    ctx = make_ctx(capi, sc)
    tab = Table(ctx, 10)
    tab.set()
    v32_dev = ctx.alloc(sc.width * sc.height * 4)
    ctx.cull_meshes(cam0)
    ctx.upload(v32_dev, v32)
    want = decode_gpu(ctx, cam0, sc.width, sc.height, vis32_dev=v32_dev)
    for k, g in zip(PLANES, got):
        _assert_planes_equal(g, want[k], k)
    assert (got[0][:, :, 3] != 0).sum() > 1000
    ctx.free(v32_dev)
    tab.free()
    ctx.close()
    for t, r in zip(tables, renderers):
        t.free()
        r.close()


def test_checker_quad_at_texel_centres(capi):
    """no oracle: a screen-aligned quad (clip == local, uv = xy + 0.5) covering 32 x 32 pixels of a 64 x 64 target, textured 1:1 with
    a 32 x 32 random RGBA8 checker and a nearest sampler, rasterised by the library.  Every pixel centre is a texel centre, so pixel
    (x, y) reads texel (x - 16, y - 16): albedo = texel / 255 exactly, metallic / roughness = the texel's b / g, occlusion 1, on every
    covered pixel of the quad's 32 x 32 square; pixels away from the quad keep the sentinel."""
    from tests.helpers_scene import quad_scene

    W = H = 64
    sc, cam = quad_scene(W, H, attributes=True)
    ctx = make_ctx(capi, sc)
    rng = np.random.default_rng(12)
    tex = np.ascontiguousarray(rng.integers(0, 256, (32, 32, 4), dtype=np.uint8))
    tex_dev = ctx.alloc(tex.nbytes)
    ctx.upload(tex_dev, tex)
    m = np.zeros(1, dtype=abi.MATERIAL_DT)
    m[0]["flags"] = abi.MATERIAL_HAS_ALBEDO_IMAGE | abi.MATERIAL_HAS_METALLIC_ROUGHNESS_IMAGE
    m[0]["albedo_color"] = [half(1.0)] * 4
    m[0]["metallic_factor"] = m[0]["roughness_factor"] = half(1.0)
    m[0]["uv_size"] = [half(1.0), half(1.0)]
    m[0]["metallic_roughness_image_index"] = 0
    smp = np.array([(abi.FILTER_NEAREST, abi.FILTER_NEAREST, abi.MIPMAP_NEAREST, abi.ADDRESS_CLAMP_TO_EDGE, abi.ADDRESS_CLAMP_TO_EDGE)],
                   dtype=abi.SAMPLER_DT)
    ctx.set_materials(m, [(tex_dev, 32, 32, abi.IMAGE_RGBA8_UNORM)], smp)
    vis_dev = ctx.alloc(W * H * 8)
    ctx.clear_visbuffer(vis_dev, W, H)
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    ctx.cull_meshlets(cam, abi.CULL_TEST_FRUSTUM, False)
    ctx.raster_visbuffer(cam, abi.CULL_TEST_ALL, W, H, vis_dev)
    sentinel = np.float32(-5.0)
    got = decode_gpu(ctx, cam, W, H, vis64_dev=vis_dev, init=sentinel)
    covered = got["albedo"][:, :, 0] != sentinel
    # coverage is the raster's (its own oracle tests pin the fill rule on the quad's edges and diagonal); here: nearly all of the
    # square, nothing away from it
    assert not covered[:15].any() and not covered[49:].any() and not covered[:, :15].any() and not covered[:, 49:].any()
    inside = covered[16:48, 16:48]
    assert inside.sum() > 32 * 32 - 4 * 32
    texel = tex.astype(np.float32) / np.float32(255.0)
    np.testing.assert_array_equal(got["albedo"][16:48, 16:48][inside], texel[inside])
    mro = got["metallic_roughness_occlusion"][16:48, 16:48][inside]
    np.testing.assert_array_equal(mro[:, 0], texel[:, :, 2][inside])
    np.testing.assert_array_equal(mro[:, 1], texel[:, :, 1][inside])
    np.testing.assert_array_equal(mro[:, 2:], np.float32([1.0, 0.0]) + np.zeros((int(inside.sum()), 2), np.float32))
    for p in (tex_dev, vis_dev):
        ctx.free(p)
    ctx.close()


def test_bad_vertex_index_writes_zeros(capi, orc, gb):
    """a mesh whose vertex_count lies below the indices of its triangles (status 2 of the decode) writes zeros to all four planes,
    as the oracle does; discarded pixels keep the sentinel"""
    from tests.helpers_scene import quad_scene

    W = H = 16
    sc, cam = quad_scene(W, H, attributes=True)
    sc.meshes["vertex_count"] = 2
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc)
    tab = Table(ctx, 13, n_materials=1)
    tab.set()
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    v32 = np.full((H, W), 0xFFFFFFFF, dtype=np.uint32)
    v32[4:12, 4:12] = np.arange(64).reshape(8, 8) % 2
    sentinel = np.float32(-7.25)
    want, bad = gb.decode_gbuffer(hs, mi, 1, cam, v32, tab.host, init=sentinel)
    v32_dev = ctx.alloc(v32.nbytes)
    ctx.upload(v32_dev, v32)
    got = decode_gpu(ctx, cam, W, H, vis32_dev=v32_dev, init=sentinel)
    for k in PLANES:
        _assert_planes_equal(got[k], want[k], k)
        assert (got[k][4:12, 4:12] == 0).all() and (got[k][:4] == sentinel).all(), k
    ctx.free(v32_dev)
    tab.free()
    ctx.close()

