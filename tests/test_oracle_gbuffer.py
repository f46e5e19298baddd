"""The G-buffer decode's specification (oracle/oxc_oracle_gbuffer.c) pinned by hand: the sRGB tables, untextured factors, the
tangent frame of a camera-facing quad, normal maps, level selection against the alpha test's sampler, discarded pixels, and the
world-normal half of the normal plane against orc_decode_visbuffer."""
import os
from decimal import Decimal, getcontext

import numpy as np
import pytest

from oxylus_b200 import abi, synth


@pytest.fixture(scope="module")
def gb():
    import pyoracle_gbuffer

    pyoracle_gbuffer.build()
    return pyoracle_gbuffer


def half(x):
    return int(np.float16(x).view(np.uint16))


def nearest_f32_of_eotf(c):
    getcontext().prec = 40
    x = Decimal(c) / Decimal(255)
    e = x / Decimal("12.92") if x <= Decimal("0.04045") else ((x + Decimal("0.055")) / Decimal("1.055")) ** Decimal("2.4")
    f = np.float32(float(e))
    cands = (np.nextafter(f, np.float32(-1)), f, np.nextafter(f, np.float32(2)))
    return min(cands, key=lambda v: abs(Decimal(float(v)) - e))


def test_srgb_tables_are_the_nearest_binary32(gb):
    """the oracle's table and the one compiled into csrc/oxc_gbuffer.cuh both equal the binary32 nearest to the exact EOTF"""
    want = np.array([nearest_f32_of_eotf(c) for c in range(256)], np.float32)
    np.testing.assert_array_equal(gb.srgb_table().view(np.uint32), want.view(np.uint32))
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oxylus_b200", "csrc", "oxc_gbuffer.cuh")).read()
    body = src[src.index("k_srgb_to_linear[256] = {") :].split("{", 1)[1].split("}", 1)[0]
    dev = np.array([float.fromhex(t.strip().rstrip("f")) for t in body.split(",") if t.strip()], np.float32)
    np.testing.assert_array_equal(dev.view(np.uint32), want.view(np.uint32))


def pixel(ddx=(0, 0, 0), ddy=(0, 0, 0), wp=((0, 0, 0),) * 3, uv=(0.5, 0.5), uv_ddx=(0, 0), uv_ddy=(0, 0), n=(0, 0, 1)):
    return np.array(list(ddx) + list(ddy) + [c for p in wp for c in p] + list(uv) + list(uv_ddx) + list(uv_ddy) + list(n), np.float32)


def table(orc, flags=0, images=(), samplers=None, **kw):
    m = np.zeros(1, dtype=abi.MATERIAL_DT)
    m[0]["flags"] = flags
    m[0]["albedo_color"] = [half(v) for v in kw.get("albedo", (0.5, 0.25, 1.0, 0.75))]
    m[0]["emissive_color"] = [half(v) for v in kw.get("emissive", (2.0, 0.0, 0.125))]
    m[0]["metallic_factor"], m[0]["roughness_factor"] = half(0.25), half(0.5)
    m[0]["uv_size"] = [half(1.0), half(1.0)]
    for k, v in kw.get("indices", {}).items():
        m[0][k] = v
    return orc.MaterialTable(m, list(images), samplers)


def quad_pixel(s=4.0, mirror=False, const_uv=False):
    """a camera-facing quad at z = -5: one pixel step right moves along world +x, one step down along world -y (screen rows run
    down); uv = (x / s, -y / s), so v grows down the screen as image rows do"""
    wp = ((0.0, 0.0, -5.0), (1.0, 0.0, -5.0), (0.0, 1.0, -5.0))
    ddx, ddy = (-0.01, 0.01, 0.0), (0.01, 0.0, -0.01)
    uvs = [(x / s * (-1 if mirror else 1), -y / s) for x, y, _ in wp]
    if const_uv:
        uvs = [(0.25, 0.25)] * 3
    uv_ddx = tuple(sum(ddx[i] * uvs[i][j] for i in range(3)) for j in range(2))
    uv_ddy = tuple(sum(ddy[i] * uvs[i][j] for i in range(3)) for j in range(2))
    return pixel(ddx=ddx, ddy=ddy, wp=wp, uv=(0.3, 0.4), uv_ddx=uv_ddx, uv_ddy=uv_ddy, n=(0.0, 0.0, 1.0))


def oct_decode(e):
    x, y = float(e[0]), float(e[1])
    z = 1.0 - abs(x) - abs(y)
    if z < 0:
        x, y = (1 - abs(y)) * np.sign(x), (1 - abs(x)) * np.sign(y)
    v = np.array([x, y, z])
    return v / np.linalg.norm(v)


def test_untextured_material_gives_its_factors(orc, gb):
    out = gb.shade(table(orc), 0, quad_pixel(), (0, 0, 0))
    np.testing.assert_array_equal(out[0:4], np.float32([0.5, 0.25, 1.0, 0.75]))
    np.testing.assert_array_equal(out[8:12], np.float32([2.0, 0.0, 0.125, 0.0]))
    np.testing.assert_array_equal(out[12:16], np.float32([0.25, 0.5, 1.0, 0.0]))
    np.testing.assert_array_equal(out[4:6], out[6:8])  # no normal image: the mapped normal is the world normal
    assert gb.shade(table(orc), 1, quad_pixel(), (0, 0, 0)) is None  # material out of range


def test_tangent_frame_and_normal_maps(orc, gb):
    """a normal map of known tilt on the camera-facing quad: T = +x, B = +y (world up, v down the image); a mirrored uv flips T; FlipY flips B; constant uv gives
    js = 0 and no NaN in .zw; TwoComponent rebuilds z from x and y"""
    tilt = np.zeros((1, 1, 4), np.uint8)
    tilt[0, 0] = (200, 128, 200, 255)  # s = (0.569, 0.004, 0.569)
    s = tilt[0, 0, :3].astype(np.float64) / 255 * 2 - 1
    mk = lambda flags: table(orc, abi.MATERIAL_HAS_NORMAL_IMAGE | flags, [(tilt, abi.IMAGE_RGBA8_UNORM)])
    want = s / np.linalg.norm(s)
    got = oct_decode(gb.shade(mk(0), 0, quad_pixel(), (0, 0, 0))[4:6])
    np.testing.assert_allclose(got, want, atol=1e-3)
    got = oct_decode(gb.shade(mk(0), 0, quad_pixel(mirror=True), (0, 0, 0))[4:6])
    np.testing.assert_allclose(got, want * [-1, 1, 1], atol=1e-3)
    got = oct_decode(gb.shade(mk(abi.MATERIAL_NORMAL_FLIP_Y), 0, quad_pixel(), (0, 0, 0))[4:6])
    np.testing.assert_allclose(got, [want[0], -want[1], want[2]], atol=1e-3)
    two = np.array([s[0], s[1], np.sqrt(max(0.0, 1 - s[0] ** 2 - s[1] ** 2))])
    got = oct_decode(gb.shade(mk(abi.MATERIAL_NORMAL_TWO_COMPONENT), 0, quad_pixel(), (0, 0, 0))[4:6])
    np.testing.assert_allclose(got, two / np.linalg.norm(two), atol=1e-3)
    out = gb.shade(mk(0), 0, quad_pixel(const_uv=True), (0, 0, 0))
    assert not np.isnan(out[6:8]).any()
    np.testing.assert_array_equal(out[6:8], np.float32([0.0, 0.0]))


def test_levels_agree_with_the_alpha_sampler(orc, gb):
    """1:1 and 4:1 texel mappings select levels 0 and 2, and equal orc_alpha_sample's alpha at that uv and level"""
    rng = np.random.default_rng(3)
    lv = orc.mip_chain(rng.integers(0, 256, (16, 16, 4), dtype=np.uint8))
    smp = (abi.FILTER_LINEAR, abi.FILTER_LINEAR, abi.MIPMAP_NEAREST, abi.ADDRESS_REPEAT, abi.ADDRESS_REPEAT)
    for scale, level in ((1.0, 0), (4.0, 2)):
        d = scale / 16
        got = gb.sample_grad(lv, abi.IMAGE_RGBA8_UNORM, 0.37, 0.61, (d, 0.0), (0.0, d), smp)
        np.testing.assert_array_equal(got, gb.sample_level(lv, abi.IMAGE_RGBA8_UNORM, 0.37, 0.61, level, abi.FILTER_LINEAR, smp))
        assert np.float32(got[3]) == np.float32(orc.alpha_sample(lv, abi.IMAGE_RGBA8_UNORM, 0.37, 0.61, smp, level))


def test_formats(orc, gb):
    t = np.array([[[10, 200, 30, 40]]], np.uint8)
    srgb = gb.srgb_table()
    np.testing.assert_array_equal(gb.sample_level(t, abi.IMAGE_RGBA8_UNORM, 0.5, 0.5), np.float32([10, 200, 30, 40]) / np.float32(255))
    np.testing.assert_array_equal(gb.sample_level(t, abi.IMAGE_RGBA8_SRGB, 0.5, 0.5), [srgb[10], srgb[200], srgb[30], np.float32(40) / np.float32(255)])
    np.testing.assert_array_equal(gb.sample_level(t[:, :, 0], abi.IMAGE_R8_UNORM, 0.5, 0.5), np.float32([10 / np.float32(255), 0, 0, 1]))
    np.testing.assert_array_equal(gb.sample_level(t[:, :, :2], abi.IMAGE_RG8_UNORM, 0.5, 0.5),
                                  [np.float32(10) / np.float32(255), np.float32(200) / np.float32(255), 0, 1])


def test_frame_discards_keep_the_sentinel_and_zw_matches_the_decode(orc, gb):
    """over a synth frame: discarded pixels keep the sentinel, decoded pixels are written, and normal.zw equals
    orc_decode_visbuffer's uv_normal.zw"""
    sc = synth.make_scene(60_000, config_index=2, width=160, height=90, n_unique_meshes=8)
    hs = orc.HostScene(sc)
    cam = sc.camera(0.0)
    ref = orc.frame(hs, cam, sc.width, sc.height, np.zeros(1 << 16, np.uint32), None)
    v32, _ = orc.resolve(ref["vis64"])
    total = int(ref["visibility"]["total"][0])
    tab = table(orc)
    out, bad = gb.decode_gbuffer(hs, ref["meshlet_instances"], total, cam, v32, tab, init=np.float32(-3.0))
    dec = orc.decode_visbuffer(hs, ref["meshlet_instances"], total, cam, v32)
    status = dec["lambda_"][:, :, 3]
    assert (status == 1).sum() > 500 and (status == 0).sum() > 100 and bad == 0
    assert (out["albedo"][status == 0] == np.float32(-3.0)).all()
    np.testing.assert_array_equal(out["normal"][status == 1][:, 2:].view(np.uint32), dec["uv_normal"][status == 1][:, 2:].view(np.uint32))
    assert (out["albedo"][status == 1] == np.float32([0.5, 0.25, 1.0, 0.75])).all()


def test_tangent_frame_of_a_camera_facing_quad(gb):
    """T = +x and B = +y on the camera-facing quad, to a few ulps in float64; a mirrored u flips T and keeps B; constant uv gives
    js = 0, so T = B = 0 and no NaN"""
    for mirror, t_want in ((False, 1.0), (True, -1.0)):
        t, b = gb.tangent_frame(quad_pixel(mirror=mirror), (0.0, 0.0, 0.0))
        np.testing.assert_allclose(t.astype(np.float64), [t_want, 0.0, 0.0], rtol=0, atol=4 * np.finfo(np.float32).eps)
        np.testing.assert_allclose(b.astype(np.float64), [0.0, 1.0, 0.0], rtol=0, atol=4 * np.finfo(np.float32).eps)
    t, b = gb.tangent_frame(quad_pixel(const_uv=True), (0.0, 0.0, 0.0))
    assert not np.isnan(t).any() and not np.isnan(b).any()
    np.testing.assert_array_equal(np.abs(np.concatenate([t, b])), 0.0)


def test_bad_vertex_index_writes_zeros(orc, gb):
    """a mesh whose vertex_count lies below an index its meshlets use (status 2 of the decode) writes zeros to all four planes, while
    discarded pixels keep the sentinel and the other pixels are shaded"""
    sc = synth.make_scene(60_000, config_index=2, width=160, height=90, n_unique_meshes=8)
    hs = orc.HostScene(sc)
    cam = sc.camera(0.0)
    ref = orc.frame(hs, cam, sc.width, sc.height, np.zeros(1 << 16, np.uint32), None)
    v32, _ = orc.resolve(ref["vis64"])
    total = int(ref["visibility"]["total"][0])
    hs.meshes["vertex_count"][:4] = 3
    sentinel = np.float32(-3.0)
    out, bad = gb.decode_gbuffer(hs, ref["meshlet_instances"], total, cam, v32, table(orc), init=sentinel)
    status = orc.decode_visbuffer(hs, ref["meshlet_instances"], total, cam, v32)["lambda_"][:, :, 3]
    assert (status == 2).sum() > 20 and (status == 1).sum() > 20 and bad == 0
    for k in gb.PLANES:
        assert (out[k][status == 2] == 0).all() and not np.signbit(out[k][status == 2]).any(), k
        assert (out[k][status == 0] == sentinel).all(), k
    assert (out["albedo"][status == 1] == np.float32([0.5, 0.25, 1.0, 0.75])).all()
