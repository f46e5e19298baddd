"""Known-answer tests of the oracle's VSM shadow raster (oracle/oxc_oracle_vsm_draw.c orc_vsm_draw_pages): hand-built quads drawn
into a 64^2 atlas of 4 x 4 pages of 16 texels, identity world and clipmap matrices (clip == object position, w = 1, so pixel centre
px sits at x = (px + 0.5) / 32 - 1), expected atlases worked out from the shader's text or from an f64 evaluation of the plane."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_oracle_alpha import checker, material

B, D, V = abi.VSM_PAGE_BACKED, abi.VSM_PAGE_DIRTY, abi.VSM_PAGE_VISIBLE


@pytest.fixture(scope="module")
def vd():
    import pyoracle_vsm_draw

    pyoracle_vsm_draw.build()
    return pyoracle_vsm_draw


def quads_scene(quads, uv=False):
    """one mesh, one meshlet: each quad = 4 corner positions (x, y, z) drawn as triangles (0, 1, 2), (0, 2, 3); uv = (x + 1) / 2,
    (y + 1) / 2 when asked"""
    pos = np.concatenate([np.asarray(q, dtype=np.float32) for q in quads])
    n = len(pos)
    tris = np.concatenate([np.array([[0, 1, 2], [0, 2, 3]]) + 4 * k for k in range(len(quads))]).astype(np.uint8)
    chunks, off = [], 0

    def put(a, align=16):
        nonlocal off
        pad = (-off) % align
        if pad:
            chunks.append(np.zeros(pad, dtype=np.uint8))
            off += pad
        start = off
        raw = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        chunks.append(raw)
        off += raw.size
        return start

    pq = np.zeros((n, 4), dtype=np.uint16)
    pq[:, :3] = synth.quantize_half(pos)
    mesh = np.zeros(1, dtype=abi.MESH_DT)
    mesh["vertex_positions"] = put(pq)
    mesh["vertex_count"], mesh["lod_count"] = n, 1
    if uv:
        mesh["texture_coords"] = put(synth.quantize_half((pos[:, :2] + np.float32(1.0)) * np.float32(0.5)))
    meshlet = np.zeros(1, dtype=abi.MESHLET_DT)
    meshlet["vertex_count"], meshlet["triangle_count"] = n, len(tris)
    micro = np.zeros((tris.size + 3) // 4 * 4, dtype=np.uint8)
    micro[: tris.size] = tris.reshape(-1)
    lod = np.zeros(1, dtype=abi.MESH_LOD_DT)
    lod["meshlets"] = put(meshlet)
    lod["meshlet_bounds"] = put(np.zeros(1, dtype=abi.MESHLET_BOUNDS_DT))
    lod["local_triangle_indices"] = put(micro)
    lod["indirect_vertex_indices"] = put(np.arange(n, dtype=np.uint32))
    lod["meshlet_count"] = lod["meshlet_bounds_count"] = 1
    lod["local_triangle_indices_count"], lod["indirect_vertex_indices_count"] = micro.size, n
    mesh["lods"] = put(lod)
    blob = np.concatenate(chunks)
    blob = np.concatenate([blob, np.zeros((-blob.size) % 16, dtype=np.uint8)])
    inst = np.zeros(1, dtype=abi.MESH_INSTANCE_DT)
    xf = np.zeros(1, dtype=abi.TRANSFORM_DT)
    xf["world"][0] = np.eye(4, dtype=np.float32).reshape(16)
    return synth.Scene(mesh, inst, xf, blob, 1, 64, 64, 0)


def coarse():
    """xy scaled by 1e-3 (every triangle's |det| < 1e-4: both windings pass the coarse test), z = 0.5"""
    cam = np.zeros(1, dtype=abi.CULL_CAMERA_DT)
    m = np.diag([1e-3, 1e-3, 0.0, 1.0]).astype(np.float32)
    m[2, 3] = 0.5
    cam["projection_view"][0] = m.T.reshape(16)  # column-major
    cam["mesh_instance_count"] = 1
    return cam


def clipmap(offset=(0, 0), flip_y=False):
    cm = np.zeros(1, dtype=abi.CLIPMAP_DT)
    cm["projection_view_mat"][0] = np.diag([1.0, -1.0 if flip_y else 1.0, 1.0, 1.0]).astype(np.float32).T.reshape(16)
    cm["page_offset"][0] = offset
    return cm


def vsm():
    v = np.zeros(1, dtype=abi.VSM_CONTEXT_DT)
    v["page_size"], v["page_table_size"], v["physical_page_table_size"], v["clipmap_count"] = 16, 4, 64, 1
    return v


def identity_table(bits=B | D):
    """every entry at (x, y) backed on physical page y * 4 + x: the atlas is the virtual image"""
    y, x = np.mgrid[0:4, 0:4]
    return ((bits | ((y * 4 + x) << 16)).astype(np.uint32)).reshape(1, 4, 4)


def draw(vd, orc, quads, table, cm=None, flags=(1,), atlas=None, materials=None, uv=False):
    sc = quads_scene(quads, uv)
    hs = orc.HostScene(sc)
    mi = np.zeros(1, dtype=abi.MESHLET_INSTANCE_DT)
    a = np.ones((64, 64), dtype=np.float32) if atlas is None else atlas.copy()
    n = vd.vsm_draw_pages(hs, mi, [0], coarse(), vsm(), clipmap() if cm is None else cm, list(flags), table, a, materials)
    return a, n


def quad(x0, y0, x1, y1, z=lambda x, y: 0.5):
    return [(x0, y0, z(x0, y0)), (x1, y0, z(x1, y0)), (x1, y1, z(x1, y1)), (x0, y1, z(x0, y1))]


def centres():
    c = (np.arange(64) + 0.5) / 32.0 - 1.0
    return np.meshgrid(c, c, indexing="xy")  # (x, y) of pixel (py, px)


def test_dirty_page_written_clean_page_not(vd, orc):
    t = np.zeros((1, 4, 4), dtype=np.uint32)
    t[0, 0, 0] = B | D | (5 << 16)  # virtual page (0, 0) -> physical page 5 = page coordinates (1, 1)
    t[0, 0, 1] = B | (6 << 16)      # backed, clean
    a, n = draw(vd, orc, [quad(-1.5, -1.5, 1.5, 1.5)], t)
    want = np.ones((64, 64), np.float32)
    want[16:32, 16:32] = 0.5
    np.testing.assert_array_equal(a, want)
    assert n == 256


def test_back_wound_triangle_is_drawn(vd, orc):
    """the clipmap matrix mirrors y: both triangles reach the raster with the other winding and are drawn all the same"""
    front, _ = draw(vd, orc, [quad(-1.5, -1.5, 1.5, 1.5)], identity_table())
    back, n = draw(vd, orc, [quad(-1.5, -1.5, 1.5, 1.5)], identity_table(), cm=clipmap(flip_y=True))
    assert (front == 0.5).all() and n == 4096
    np.testing.assert_array_equal(back, front)


def test_smaller_depth_wins_in_either_order(vd, orc):
    near, far = quad(-1.5, -1.5, 1.5, 0.5, lambda x, y: 0.25), quad(-1.5, -0.5, 1.5, 1.5, lambda x, y: 0.75)
    a, _ = draw(vd, orc, [near, far], identity_table())
    b, _ = draw(vd, orc, [far, near], identity_table())
    np.testing.assert_array_equal(a, b)
    x, y = centres()
    assert (a[y < 0.5] == 0.25).all() and (a[y > 0.5] == 0.75).all()


def test_depth_outside_0_1_is_dropped(vd, orc):
    """z = 0.5 + 2x/3 runs from -0.5 to 1.5 across the viewport: exactly the samples with |x| <= 0.75 are written (no pixel centre is
    near the limits), with the plane's value"""
    a, n = draw(vd, orc, [quad(-1.5, -1.5, 1.5, 1.5, lambda x, y: 0.5 + x * 2.0 / 3.0)], identity_table())
    x, _ = centres()
    inside = np.abs(x) <= 0.75
    assert (a[~inside] == 1.0).all() and n == int(inside.sum())
    np.testing.assert_allclose(a[inside], (0.5 + x * 2.0 / 3.0)[inside], atol=2e-6)


def test_page_offset_wraps(vd, orc):
    """offset (3, 1): virtual page (1, 3) lands on entry ((1 + 3) % 4, (3 + 1) % 4) = (0, 0), the only dirty one, physical page 0"""
    t = np.zeros((1, 4, 4), dtype=np.uint32)
    t[0, 0, 0] = B | D
    z = lambda x, y: 0.5 + x / 8.0 + y / 4.0  # noqa: E731  (corner depths exact in half precision)
    a, n = draw(vd, orc, [quad(-1.5, -1.5, 1.5, 1.5, z)], t, cm=clipmap((3, 1)))
    x, y = centres()
    assert n == 256 and (a[16:, :] == 1.0).all() and (a[:, 16:] == 1.0).all()
    np.testing.assert_allclose(a[:16, :16], z(x, y)[48:64, 16:32], atol=2e-6)


@pytest.mark.parametrize("case", ["not_backed", "backed_clean", "flag_zero"])
def test_untouched(vd, orc, case):
    bits = {"not_backed": V | D, "backed_clean": V | B, "flag_zero": B | D}[case]
    start = np.random.default_rng(1).random((64, 64)).astype(np.float32)
    a, n = draw(vd, orc, [quad(-1.5, -1.5, 1.5, 1.5, lambda x, y: 0.0)], identity_table(bits), flags=(0,) if case == "flag_zero" else (1,), atlas=start)
    assert n == 0
    np.testing.assert_array_equal(a, start)


def test_ground_plane_beyond_the_snap_range(vd, orc):
    """a 4000 x 4000 plane (the corners 64000 pixels out, 4 times the snap range) through the clipper: every texel is written once
    (no crack along the shared diagonal or the cuts) with the f64 plane's depth.  Wound the way the coarse test keeps (its |det| is
    large here)"""
    z = lambda x, y: 0.5 + x / 8192.0 + y / 16384.0  # noqa: E731  (corner depths exact in half precision)
    q = quad(-2000.0, -2000.0, 2000.0, 2000.0, z)
    a, n = draw(vd, orc, [[q[0], q[3], q[2], q[1]]], identity_table())
    x, y = centres()
    assert n == 4096
    np.testing.assert_allclose(a, z(x, y), atol=1e-5)


def test_checker_alpha_removes_exactly_its_discarded_texels(vd, orc):
    """uv = ((x + 1) / 2, (y + 1) / 2) over a 2 x 2 checker (nearest): the quadrants whose texel alpha is 0 stay at the clear value"""
    img = checker(2, 1)
    tab = orc.MaterialTable(np.array([material(image=0, cutoff=0.5, sampler=0)], dtype=abi.MATERIAL_DT), [(img, abi.IMAGE_RGBA8_UNORM)],
                            np.array([abi.sampler(abi.FILTER_NEAREST, abi.FILTER_NEAREST)], dtype=abi.SAMPLER_DT))
    a, n = draw(vd, orc, [quad(-1.0, -1.0, 1.0, 1.0)], identity_table(), materials=tab, uv=True)
    opaque, _ = draw(vd, orc, [quad(-1.0, -1.0, 1.0, 1.0)], identity_table(), uv=True)
    keep = np.kron(img[:, :, 3] >= 128, np.ones((32, 32), dtype=bool))
    assert (a[keep] == opaque[keep]).all() and (a[~keep] == 1.0).all() and keep.sum() == 2048 and n == 2048
