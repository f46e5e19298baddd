"""The shadow-clipmap, multi-view and terrain culls (include/oxcull.h) against the CPU oracle across their shapes, and the oracle's
decisions against an independent float64 restatement of the same maths.

tests/test_gpu_parity.py runs each of these culls at one shape.  This module covers what else the ABI accepts: every page-pyramid
size and level count (the mip clamp and the repeated 1x1 levels), 1 to 16 clipmaps, dirty masks, page offsets far outside the
pyramid, the z_near "projection failed = visible" shortcut, boxes steered onto page edges, shards, the engine's pass order on one
context with and without a bound device camera; 1 to 16 views; terrain grids whose last block and last mask word are partly
filled, every cull-flag subset and Hi-Z state, near-plane and facing-away cameras.  Bar: bit-exact; survivor order is
atomics-ordered, so survivor lists are compared as sorted sets.

The float64 reference (f64_*) evaluates, per meshlet or patch and per view or clipmap, the frustum, the cone and for the shadow cull
the uv box, mip and four page taps, in float64, and flags every decision that lies within a margin of its edge: 1e-4 texel of a tap
edge, 1e-5 relative of a power-of-two mip edge, 1e-5 relative of a plane, cone or depth comparison.  The oracle's binary32
decisions must equal it everywhere else."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests import emulated_torture_check as torture
from tests.helpers_scene import boxes_scene
from tests.test_gpu_parity import SCENES, _assert_planes_equal, make_ctx

pytestmark = pytest.mark.gpu

FRUSTUM, OCC, LATE = abi.CULL_TEST_FRUSTUM, abi.CULL_TEST_OCCLUSION, abi.CULL_LATE_PASS
TAP_MARGIN, REL_MARGIN = 1e-4, 1e-5
EPS_F32 = float(np.float32(1e-7))  # cull.slang:133, an f32 literal


# ------------------------------------------------------------------------------------------------------------------------------
# float64 reference
# ------------------------------------------------------------------------------------------------------------------------------
def _half(h):
    """dequantize_half (common/math.slang:193-201) in float64: denormals flush to signed zero"""
    h = np.asarray(h, dtype=np.uint16)
    v = h.view(np.float16).astype(np.float64)
    return np.where((h & 0x7C00) == 0, np.where(h & 0x8000, -0.0, 0.0), v)


def _mat(m16):
    """column-major 16 floats -> float64 [..., 4, 4] with M[i][j] = row i, column j"""
    m = np.asarray(m16, dtype=np.float64).reshape(-1, 4, 4)
    return np.swapaxes(m, -1, -2)


def meshlet_records(hs, mi, total):
    """per meshlet instance: world matrix [n,4,4], centre, extent, cone axis, cutoff (float64), from the host scene tables"""
    mi = mi[:total]
    inst = hs.mesh_instances[mi["mesh_instance_index"]]
    mesh = hs.meshes[inst["mesh_index"]]
    lod_off = mesh["lods"].astype(np.int64) + inst["lod_index"].astype(np.int64) * abi.MESH_LOD_DT.itemsize
    blob = hs.blob
    u64 = blob[: blob.size // 8 * 8].view(np.uint64)
    bounds_off = u64[(lod_off + abi.MESH_LOD_DT.fields["meshlet_bounds"][1]) // 8].astype(np.int64)
    rec = blob[: blob.size // 16 * 16].view(abi.MESHLET_BOUNDS_DT)[(bounds_off + mi["meshlet_index"].astype(np.int64) * 16) // 16]
    world = _mat(hs.transforms["world"])[inst["transform_index"]]
    c, e = _half(rec["aabb_center"]), _half(rec["aabb_extent"])
    axis = np.stack([rec["cone_axis_xy"][:, 0], rec["cone_axis_xy"][:, 1], rec["cone_axis_z"]], axis=1).astype(np.float64) / 127.0
    return world, c, e, axis, rec["cone_cutoff"].astype(np.float64) / 127.0


def _decided(fail, near):
    """robust decision of an AND of tests: culled if a test clearly fails, kept if every test clearly passes; else excused"""
    clear_fail = (fail & ~near).any(-1)
    clear_pass = (~fail & ~near).all(-1)
    return ~fail.any(-1), ~(clear_fail | clear_pass)


def f64_frustum(M, A, c, he):
    """cull.slang:57-84 on mvp M (abs-product A for the rounding scale): visible, near-edge.  M, A [..., 4, 4]; c, he [..., 3]"""
    rows = lambda X: (X[..., 0, :], X[..., 1, :], X[..., 2, :], X[..., 3, :])
    r0, r1, r2, r3 = rows(M)
    a0, a1, a2, a3 = rows(A)
    P = np.stack([r3 + r0, r3 - r0, r3 + r1, r3 - r1, r2, r3 - r2], axis=-2)
    B = np.stack([a3 + a0, a3 + a0, a3 + a1, a3 + a1, a2, a3 + a2], axis=-2)
    n = P[..., :3]
    p = c[..., None, :] + np.where(np.signbit(n), -1.0, 1.0) * he[..., None, :]
    dist = (n * p).sum(-1) + P[..., 3]
    scale = (B[..., :3] * np.abs(p)).sum(-1) + B[..., 3]
    degenerate = (n == 0).all(-1)  # a zero normal normalises to NaN: that plane never culls
    fail = (dist <= 0) & ~degenerate
    near = (np.abs(dist) <= REL_MARGIN * scale) & ~degenerate
    return _decided(fail, near)


def _cofactor_axis(W, axis):
    """normalize(transform.to_world_normal(axis)) (scene.slang:291-302)"""
    b0, b1, b2 = W[..., :3, 0], W[..., :3, 1], W[..., :3, 2]
    r0, r1, r2 = np.cross(b1, b2), np.cross(b2, b0), np.cross(b0, b1)
    n = r0 * axis[..., 0:1] + r1 * axis[..., 1:2] + r2 * axis[..., 2:3]
    with np.errstate(invalid="ignore", divide="ignore"):
        return n / np.linalg.norm(n, axis=-1, keepdims=True)


def f64_cone_directional(W, axis, cutoff, view_dir):
    """cull.slang:177-179 as cull_meshlets_hpb.slang:53-54 uses it: visible, near-edge"""
    wa = _cofactor_axis(W, axis)
    v = np.asarray(view_dir, dtype=np.float64)
    d = (wa * v).sum(-1)
    with np.errstate(invalid="ignore"):
        culled = (cutoff < 1.0) & (d >= cutoff)
        near = (cutoff < 1.0) & (np.abs(d - cutoff) <= REL_MARGIN * ((np.abs(wa) * np.abs(v)).sum(-1) + np.abs(cutoff)))
    return ~culled, near


def f64_cone_positional(W, c, e, axis, cutoff, cam_pos):
    """cull.slang:173-175 with the world centre / radius of cull_meshlets.slang:42-52: visible, near-edge"""
    wa = _cofactor_axis(W, axis)
    wc = (W[..., :3, :3] @ c[..., None])[..., 0] + W[..., :3, 3]
    radius = np.linalg.norm(e * 0.5, axis=-1) * np.linalg.norm(W[..., :3, :3], axis=-1).max(-1)
    d = wc - np.asarray(cam_pos, dtype=np.float64)
    dl = np.linalg.norm(d, axis=-1)
    lhs, rhs = (d * wa).sum(-1), cutoff * dl + radius
    with np.errstate(invalid="ignore"):
        culled = (cutoff < 1.0) & (lhs >= rhs)
        near = (cutoff < 1.0) & (np.abs(lhs - rhs) <= REL_MARGIN * (dl * (1.0 + np.abs(cutoff)) + radius))
    return ~culled, near


def f64_project(M, A, near_clip, c, e):
    """cull.slang:12-47: (ok, near-edge of the near test, uv min [...,3], uv max [...,3]); corners c +- e/2"""
    sgn = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)])
    corners = c[..., None, :] + sgn * e[..., None, :]
    h = np.concatenate([corners, np.ones(corners.shape[:-1] + (1,))], axis=-1)
    P = np.einsum("...ij,...kj->...ki", M, h)
    Pa = np.einsum("...ij,...kj->...ki", A, np.abs(h))
    depth = P[..., 3].min(-1)
    ok = ~(depth < near_clip)
    near = np.abs(depth - near_clip) <= REL_MARGIN * np.maximum(Pa[..., 3].max(-1), abs(near_clip))
    with np.errstate(invalid="ignore", divide="ignore"):
        ndc = P[..., :3] / P[..., 3:4]
    lo, hi = ndc.min(-2), ndc.max(-2)
    lo[..., :2] = lo[..., :2] * 0.5 + 0.5
    hi[..., :2] = hi[..., :2] * 0.5 + 0.5
    return ok, near, lo, hi


def f64_vsm_page(lo, hi, hpb, size, levels, layers, layer, page_offset):
    """cull.slang:137-166 (test_vsm_page) for boxes lo / hi [n, 3] on one layer: (visible, near-edge, tap texel coordinates [n, 4, 2])"""
    hs = float(size)
    box = np.maximum((hi[:, 0] - lo[:, 0]) * hs, (hi[:, 1] - lo[:, 1]) * hs)
    with np.errstate(invalid="ignore", divide="ignore"):
        lg = np.log2(np.where(box > 0, box, 1.0))
        mip = np.where(box > 1.0, np.ceil(lg), 0.0)
        k = np.round(lg)
        mip_near = (box > 0) & (np.abs(box / np.exp2(k) - 1.0) <= REL_MARGIN) & (k >= 0) & (k <= levels - 2)
    mip = np.minimum(mip, levels - 1).astype(np.int64)
    pox, poy = page_offset[0] / hs, page_offset[1] / hs
    us = np.stack([lo[:, 0], hi[:, 0], lo[:, 0], hi[:, 0]], 1) + pox
    vs = np.stack([lo[:, 1], lo[:, 1], hi[:, 1], hi[:, 1]], 1) + poy
    sz = np.maximum(size >> mip, 1)[:, None]
    offs = np.cumsum([0] + [layers * max(1, size >> l) ** 2 for l in range(levels)])
    tu, tv = (us - np.floor(us)) * sz, (vs - np.floor(vs)) * sz
    x = np.clip(np.floor(tu), 0, sz - 1).astype(np.int64)
    y = np.clip(np.floor(tv), 0, sz - 1).astype(np.int64)
    taps = hpb[offs[mip][:, None] + (layer * sz + y) * sz + x] != 0
    tap_near = ((np.abs(tu - np.round(tu)) <= TAP_MARGIN) | (np.abs(tv - np.round(tv)) <= TAP_MARGIN)).any(1)
    return taps.any(1), mip_near | tap_near, np.stack([tu, tv], -1)


def f64_hpb(hs, mi, total, cam, clipmaps, dirty, hpb, size, levels):
    """cull_meshlets_hpb.slang:27-99: per meshlet instance (visible, near-edge)"""
    W, c, e, axis, cutoff = meshlet_records(hs, mi, total)
    he = e * 0.5
    PV = _mat(cam["projection_view"][0])[0]
    cone_vis, cone_near = f64_cone_directional(W, axis, cutoff, cam["position"][0])
    fr_vis, fr_near = f64_frustum(PV @ W, np.abs(PV) @ np.abs(W), c, he)
    vis = np.zeros(total, dtype=bool)
    near = cone_near | fr_near
    for ci in range(len(clipmaps)):
        if not dirty[ci]:
            continue
        CV = _mat(clipmaps["projection_view_mat"][ci])[0]
        M, A = CV @ W, np.abs(CV) @ np.abs(W)
        cf_vis, cf_near = f64_frustum(M, A, c, he)
        ok, ok_near, lo, hi = f64_project(M, A, float(clipmaps["z_near"][ci]), c, e)
        page, page_near, _ = f64_vsm_page(lo, hi, hpb, size, levels, len(clipmaps), ci, clipmaps["page_offset"][ci])
        vis |= cf_vis & np.where(ok, page, True)
        near |= cf_near | (cf_vis & (ok_near | (ok & page_near)))
    return cone_vis & fr_vis & vis, near


def f64_multiview(hs, mi, total, views, directional):
    """per meshlet instance and view: (visible [n, v], near-edge [n, v])"""
    W, c, e, axis, cutoff = meshlet_records(hs, mi, total)
    vis, near = np.zeros((total, len(views)), bool), np.zeros((total, len(views)), bool)
    for v in range(len(views)):
        PV = _mat(views["projection_view"][v])[0]
        if directional:
            cv, cn = f64_cone_directional(W, axis, cutoff, views["position"][v])
        else:
            cv, cn = f64_cone_positional(W, c, e, axis, cutoff, views["position"][v])
        fv, fn = f64_frustum(PV @ W, np.abs(PV) @ np.abs(W), c, e * 0.5)
        vis[:, v], near[:, v] = cv & fv, cn | fn
    return vis, near


def _f64_occluded(lo, hi, hiz_levels, hw, hh):
    """cull.slang:86-135 (test_occlusion) on the pyramid levels: (occluded, near-edge)"""
    with np.errstate(invalid="ignore", over="ignore"):
        f = [np.maximum(lo[:, 0] * hw, 0.0), np.maximum(lo[:, 1] * hh, 0.0), np.minimum(hi[:, 0] * hw, hw - 1.0), np.minimum(hi[:, 1] * hh, hh - 1.0)]
    occluded, near = _f64_occluded_at(f, hi[:, 2], hiz_levels, hw, hh)
    # a texel coordinate within TAP_MARGIN (or 1e-5 relative, for far-off boxes) of an integer: excused if nudging it changes the answer
    slack = [np.maximum(TAP_MARGIN, REL_MARGIN * np.abs(np.nan_to_num(x))) for x in f]
    close = np.zeros(len(lo), bool)
    for x, s in zip(f, slack):
        close |= (x > 0) & (np.abs(x - np.round(x)) <= s)
    sel = np.nonzero(close)[0]
    for signs in np.ndindex(2, 2, 2, 2):
        if sel.size == 0:
            break
        g = [x[sel] + (2 * sg - 1) * s[sel] for x, s, sg in zip(f, slack, signs)]
        occ2, _ = _f64_occluded_at(g, hi[sel, 2], hiz_levels, hw, hh)
        near[sel] |= occ2 != occluded[sel]
    return occluded, near


def _f64_occluded_at(f, z, hiz_levels, hw, hh):
    n = len(z)
    levels = len(hiz_levels)
    to_u32 = lambda x: np.where(x > 0, np.minimum(np.nan_to_num(x, nan=0.0), 4294967295.0), 0.0).astype(np.uint64).astype(np.uint32)
    tx0, ty0, tx1, ty1 = (to_u32(x) for x in f)
    near = np.zeros(n, bool)
    size = np.maximum(tx1 - tx0, ty1 - ty0).astype(np.uint64)  # u32 wrap, as cull.slang:127
    mip = np.where(size <= 1, 0, np.ceil(np.log2(np.maximum(size, 1).astype(np.float64))).astype(np.int64))
    mip = np.minimum(mip, levels - 1)
    occluded = np.zeros(n, bool)
    for l in np.unique(mip):
        sel = mip == l
        img = hiz_levels[l].astype(np.float64)
        mh, mw = img.shape
        u = ((tx0[sel].astype(np.float64) + tx1[sel]) * 0.5) / hw
        v = ((ty0[sel].astype(np.float64) + ty1[sel]) * 0.5) / hh
        bx, by = np.floor(u * mw - 0.5).astype(np.int64), np.floor(v * mh - 0.5).astype(np.int64)
        x0, x1 = np.clip(bx, 0, mw - 1), np.clip(bx + 1, 0, mw - 1)
        y0, y1 = np.clip(by, 0, mh - 1), np.clip(by + 1, 0, mh - 1)
        d = np.minimum(np.minimum(img[y0, x0], img[y0, x1]), np.minimum(img[y1, x0], img[y1, x1]))
        zs = z[sel]
        occluded[sel] = zs <= d - EPS_F32
        near[sel] |= np.abs(zs - (d - EPS_F32)) <= REL_MARGIN * np.maximum(np.maximum(np.abs(zs), np.abs(d)), EPS_F32)
    return occluded, near


def f64_terrain(terrain, minmax, cam, flags, hiz_levels, hw, hh, mask):
    """terrain_cull.slang:19-83: (emit, visible, near-edge) per patch; `mask` is the mask before the pass"""
    t = terrain[0]
    nx, ny = int(t["patch_count"][0]), int(t["patch_count"][1])
    idx = np.arange(nx * ny)
    px, py = (idx % nx).astype(np.float64), (idx // nx).astype(np.float64)
    wmin, wsize = t["world_min"].astype(np.float64), t["world_size"].astype(np.float64)
    x0, x1 = wmin[0] + px / nx * wsize[0], wmin[0] + (px + 1) / nx * wsize[0]
    z0, z1 = wmin[1] + py / ny * wsize[1], wmin[1] + (py + 1) / ny * wsize[1]
    b = minmax.astype(np.float64)
    hsc = float(t["height_scale"])
    c = np.stack([(x0 + x1) * 0.5, float(t["base_height"]) + (b[:, 0] + b[:, 1]) * 0.5 * hsc, (z0 + z1) * 0.5], 1)
    e = np.stack([x1 - x0, np.maximum(hsc * (b[:, 1] - b[:, 0]), float(np.float32(1e-3))), z1 - z0], 1)
    PV = _mat(cam["projection_view"][0])[0]
    A = np.abs(PV)
    was = ((mask[idx >> 5] >> (idx & 31).astype(np.uint32)) & 1).astype(bool)
    vis = np.ones(len(idx), bool) if flags & LATE else was.copy()
    near = np.zeros(len(idx), bool)
    if flags & FRUSTUM:
        fv, fn = f64_frustum(np.broadcast_to(PV, (len(idx), 4, 4)), np.broadcast_to(A, (len(idx), 4, 4)), c, e * 0.5)
        near |= vis & fn
        vis &= fv
    if flags & (OCC | LATE):
        ok, ok_near, lo, hi = f64_project(np.broadcast_to(PV, (len(idx), 4, 4)), np.broadcast_to(A, (len(idx), 4, 4)),
                                          float(cam["near_clip"][0]), c, e)
        occ, occ_near = _f64_occluded(lo, hi, hiz_levels, hw, hh)
        near |= vis & (ok_near | (ok & occ_near))
        vis &= ~(ok & occ)
    emit = vis & (~was if flags & LATE else True)
    return emit, vis, near


EXCUSED_BOUND = 0.01  # of all decisions a test compares


def assert_f64_agrees(tag, oracle, ref, near):
    """the oracle's decisions equal the float64 ones wherever those are not within the margin of an edge; returns the number of
    decisions excused (the callers bound the total by EXCUSED_BOUND)"""
    oracle, ref, near = (np.asarray(a, bool).reshape(-1) for a in (oracle, ref, near))
    bad = np.nonzero((oracle != ref) & ~near)[0]
    assert len(bad) == 0, f"{tag}: {len(bad)} decisions differ from float64 away from any edge, first {bad[:8]}"
    return int(near.sum())


def mask_bits(mask, n):
    idx = np.arange(n)
    return ((mask[idx >> 5] >> (idx & 31).astype(np.uint32)) & 1).astype(bool)


def survivors_to_mask(ids, n):
    out = np.zeros(n, bool)
    out[np.asarray(ids, dtype=np.int64)] = True
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# scenes, views, pyramids
# ------------------------------------------------------------------------------------------------------------------------------
BOX_SCENE = dict(n_meshlets=3000, width=640, height=360, n_unique_meshes=16, placement="box")
LIGHT = np.float64([0.3, -0.8, -0.5])


def box_scene():
    return synth.make_scene(config_index=4, **BOX_SCENE)


def hostile_scene():
    return torture.mutate(synth.make_scene(config_index=2, **SCENES["small"]), np.random.default_rng(3), "all")


def clipmaps_for(sc, n, offsets, z_near_every=0):
    clip = np.zeros(n, dtype=abi.CLIPMAP_DT)
    for c in range(n):
        v = synth.make_ortho_view(LIGHT, (0.0, 0.0, -200.0), 12.0 * (1.6 ** (c % 10)), 1200.0, sc.mesh_instance_count)
        clip["projection_view_mat"][c] = v["projection_view"][0]
        clip["page_offset"][c] = offsets[c % len(offsets)]
        clip["z_near"][c] = 2.0 if z_near_every and c % z_near_every == 1 else 0.0
    return clip


def coarse_view(sc, half=12.0 * 1.6 ** 9):
    v = synth.make_ortho_view(LIGHT, (0.0, 0.0, -200.0), half, 1200.0, sc.mesh_instance_count)
    v["position"][0] = -LIGHT / np.linalg.norm(LIGHT)
    return v


def offset_patterns(size, rng):
    return [[(0, 0)], [(size, -size)], [(size - 1, -(size - 1))], [(-size, size - 1)], [(1000, -1000)], [(-1000, 1000), (1, -1)],
            [tuple(int(x) for x in rng.integers(-3000, 3000, size=2)) for _ in range(5)]]


DIRTY = {"none": lambda n: [0] * n, "all": lambda n: [1] * n, "only_15": lambda n: [int(c == 15) for c in range(n)],
         "alternating": lambda n: [int(c % 2 == 0) for c in range(n)]}


def random_page_table(rng, size, layers):
    pt = (rng.integers(0, 8, size=(layers, size, size)).astype(np.uint32) | (rng.integers(0, 65536, size=(layers, size, size)).astype(np.uint32) << 16))
    pt[rng.random(pt.shape) < 0.75] &= ~np.uint32(1)  # sparse, like a real frame
    return pt


def device_hpb(ctx, orc, rng, size, layers, levels):
    """a random page table built into a pyramid by oxc_build_hpb, checked against orc.build_hpb first: (device pointer, host bytes)"""
    pt = random_page_table(rng, size, layers)
    want = orc.build_hpb(pt, levels)
    pt_dev, hpb_dev = ctx.alloc(pt.nbytes), ctx.alloc(want.nbytes)
    ctx.upload(pt_dev, pt)
    ctx.upload(hpb_dev, np.full(want.nbytes, 0xAB, dtype=np.uint8))
    ctx.build_hpb(pt_dev, size, layers, hpb_dev, levels)
    np.testing.assert_array_equal(ctx.download(hpb_dev, np.uint8, want.nbytes), want, err_msg=f"build_hpb {size} x {layers} x {levels}")
    ctx.free(pt_dev)
    return hpb_dev, want


def run_hpb_both(ctx, cam, clip, dirty, hpb_dev, size, levels, tag):
    """host flags and device flags: both survivor lists (sorted) and counts; they must agree with each other"""
    ctx.cull_meshlets_hpb(cam, clip, dirty, hpb_dev, size, levels)
    n = int(ctx.cull_triangles_cmd()["x"][0])
    host = np.sort(ctx.visible_indices(n))
    flags_dev = ctx.alloc(4 * len(dirty))
    ctx.upload(flags_dev, np.asarray(dirty, dtype=np.uint32) * np.uint32(0x10001))  # any non-zero word is "dirty"
    ctx.cull_meshlets_hpb_dirty_dev(cam, clip, flags_dev, hpb_dev, size, levels)
    m = int(ctx.cull_triangles_cmd()["x"][0])
    dev = np.sort(ctx.visible_indices(m))
    ctx.free(flags_dev)
    np.testing.assert_array_equal(dev, host, err_msg=f"{tag}: device flags vs host flags")
    return host


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


# ------------------------------------------------------------------------------------------------------------------------------
# shadow-clipmap cull
# ------------------------------------------------------------------------------------------------------------------------------
HPB_SIZES = (1, 16, 48, 64, 128)


def hpb_level_counts(size):
    return sorted({1, 3, int(np.log2(size)) + 1, 16})


@pytest.mark.parametrize("clipmap_count", [1, 5, abi.MAX_VIEWS])
def test_hpb_shapes(capi, orc, clipmap_count):
    """every pyramid size x level count (1, 3, log2(size) + 1, 16) at `clipmap_count` clipmaps; per shape the four dirty masks,
    each with its own page-offset pattern, z_near = 2 on every third clipmap of the alternating mask; host flags, device flags and
    the oracle agree; the oracle agrees with float64"""
    sc = box_scene()
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc, views=abi.MAX_VIEWS)
    cam = sc.camera()
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    total = int(vis["total"][0])
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    coarse = coarse_view(sc)
    rng = np.random.default_rng(100 + clipmap_count)
    survivors, shortcut, excused, decisions = set(), 0, 0, 0
    for size in HPB_SIZES:
        patterns = offset_patterns(size, rng)
        for levels in hpb_level_counts(size):
            hpb_dev, hpb = device_hpb(ctx, orc, rng, size, clipmap_count, levels)
            for k, (name, mk) in enumerate(DIRTY.items()):
                dirty = mk(clipmap_count)
                clip = clipmaps_for(sc, clipmap_count, patterns[(k + levels) % len(patterns)], z_near_every=3 if name == "alternating" else 0)
                tag = f"size {size} levels {levels} clipmaps {clipmap_count} dirty {name}"
                ref, cmd = orc.cull_meshlets_hpb(hs, mi, vis, coarse, clip, dirty, hpb, size, levels)
                got = run_hpb_both(ctx, coarse, clip, dirty, hpb_dev, size, levels, tag)
                assert len(got) == int(cmd["x"][0]), tag
                np.testing.assert_array_equal(got, np.sort(ref), err_msg=tag)
                survivors.add(len(got))
                if not any(dirty):
                    assert len(got) == 0, tag
                f64, near = f64_hpb(hs, mi, total, coarse, clip, dirty, hpb, size, levels)
                excused += assert_f64_agrees(tag, survivors_to_mask(ref, total), f64, near)
                decisions += total
                if name == "alternating" and clipmap_count > 1:
                    shortcut += int((clip["z_near"][np.array(dirty, bool)] > 0).any())
            ctx.free(hpb_dev)
    print(f"hpb, {clipmap_count} clipmaps: {excused} of {decisions} float64 decisions excused")
    assert excused <= EXCUSED_BOUND * decisions
    assert len(survivors) > 3  # the shapes change the answer
    assert shortcut > 0 or clipmap_count == 1
    ctx.close()


def test_hpb_steered_page_edges(capi, orc):
    """boxes whose projected uv box starts or ends exactly on a page edge, with extents of exactly 2^k pages or one half-ulp either
    side; identity transforms, a clipmap of power-of-two scale, and a checkerboard at every pyramid level (a tap one texel off
    flips the answer).  The arithmetic is exact in binary32 here, so the oracle must equal float64 with no margin at all."""
    size, levels, s = 16, 5, 0.125  # world x in [-8, 8] -> u * 16 = x + 8: page edges at integer x
    rng = np.random.default_rng(31)
    n = 900
    # per axis: extent 2^k pages exactly, one half-ulp below (mip k, one texel) or above (mip k + 1); the box starts on the mip-k
    # page edge m * 2^k (exact extents) or half a half-ulp beside it
    k = np.repeat(rng.integers(0, 3, size=(n, 1)), 2, axis=1)
    variant = np.array([1.0, 1.0 - 2.0 ** -11, 1.0 + 2.0 ** -10])[rng.integers(0, 3, size=(n, 2))]
    m = rng.integers(-(8 >> k), np.maximum((8 >> k) - 1, 1))
    e2 = 2.0 ** k * variant
    c2 = m * 2.0 ** k + 2.0 ** (k - 1)
    # and three boxes starting exactly on the edge at 0 whose extent is one half-ulp short of 2^k: their four taps share a texel
    for kk in range(3):
        e2[kk] = c2[kk] = 2.0 ** kk * (1.0 - 2.0 ** -11)
        c2[kk] *= 0.5
    e = np.concatenate([e2, np.ones((n, 1))], 1).astype(np.float32)
    c = np.concatenate([c2, np.full((n, 1), 4.0)], 1).astype(np.float32)
    sc, cdec, edec = boxes_scene(c, e, 64, 64)
    assert np.array_equal(cdec, c) and np.array_equal(edec, e)  # half-exact
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc, views=2)
    cam = np.zeros(1, dtype=abi.CULL_CAMERA_DT)
    pv = np.diag([s, s, s, 1.0]).astype(np.float32)  # symmetric: column-major == row-major
    cam["projection_view"][0] = pv.reshape(16)
    cam["position"][0] = (0.0, 0.0, 1.0)
    cam["resolution"][0] = (64, 64)
    cam["mesh_instance_count"] = n
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    total = int(vis["total"][0])
    assert total == n
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    clip = np.zeros(2, dtype=abi.CLIPMAP_DT)
    clip["projection_view_mat"] = pv.reshape(16)
    clip["page_offset"] = [(0, 0), (3, -5)]
    levels_px = [np.indices((max(1, size >> l),) * 2).sum(0) % 2 == l % 2 for l in range(levels)]
    hpb = np.concatenate([np.stack([lv, ~lv]).astype(np.uint8).reshape(-1) for lv in levels_px])
    hpb_dev = ctx.alloc(hpb.nbytes)
    ctx.upload(hpb_dev, hpb)
    for dirty in ([1, 0], [0, 1]):
        ref, cmd = orc.cull_meshlets_hpb(hs, mi, vis, cam, clip, dirty, hpb, size, levels)
        got = run_hpb_both(ctx, cam, clip, dirty, hpb_dev, size, levels, f"steered, dirty {dirty}")
        np.testing.assert_array_equal(got, np.sort(ref), err_msg=f"steered, dirty {dirty}")
        layer = dirty.index(1)
        W, cc, ee, _, _ = meshlet_records(hs, mi, total)
        P = _mat(pv.reshape(16))[0]
        _, _, lo, hi = f64_project(np.broadcast_to(P, (total, 4, 4)), np.broadcast_to(np.abs(P), (total, 4, 4)), 0.0, cc, ee)
        want, _, taps = f64_vsm_page(lo, hi, hpb, size, levels, 2, layer, clip["page_offset"][layer])
        np.testing.assert_array_equal(survivors_to_mask(ref, total), want, err_msg=f"steered, dirty {dirty}: oracle vs float64")
        on_edge = (taps == np.round(taps)).any(axis=(1, 2))
        # a box on an edge whose four taps fall into one texel decides on that texel alone: those are the ones a tap off by one flips
        one_texel = (np.floor(taps[:, 0]) == np.floor(taps[:, 3])).all(1)
        assert int(on_edge.sum()) >= n // 8 and int((on_edge & one_texel).sum()) >= 1, (int(on_edge.sum()), int((on_edge & one_texel).sum()))
        print(f"steered, dirty {dirty}: {int(on_edge.sum())} of {n} boxes with a tap exactly on a page edge, "
              f"{int((on_edge & one_texel).sum())} of them deciding on one texel")
        assert 0 < len(got) < total
    ctx.free(hpb_dev)
    ctx.close()


def test_hpb_shard_auto(capi, orc):
    """oxc_set_shard_auto at two split points: the shard's survivors plus its automatic id base are the whole-scene oracle's
    survivors of the shard's id range"""
    sc = box_scene()
    hs = orc.HostScene(sc)
    n = sc.mesh_instance_count
    cam = sc.camera()
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    rng = np.random.default_rng(41)
    size, levels, count = 64, 7, 5
    coarse = coarse_view(sc)
    clip = clipmaps_for(sc, count, offset_patterns(size, rng)[-1])
    dirty = [1] * count
    ctx0 = make_ctx(capi, sc, views=count)
    hpb_dev, hpb = device_hpb(ctx0, orc, rng, size, count, levels)
    ref, _ = orc.cull_meshlets_hpb(hs, mi, vis, coarse, clip, dirty, hpb, size, levels)
    ref = np.sort(ref)
    owner = mi["mesh_instance_index"][ref]
    mid = int(np.median(owner))
    assert 0 < mid < n
    for first, cnt in ((1, mid), (mid, n - mid)):  # both shards own survivors, and both have a non-zero id base
        want = ref[(owner >= first) & (owner < first + cnt)]
        ctx = make_ctx(capi, sc, views=count)
        hpb_local = ctx.alloc(hpb.nbytes)
        ctx.upload(hpb_local, hpb)
        ctx.set_shard_auto(first, cnt)
        ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
        got = run_hpb_both(ctx, coarse, clip, dirty, hpb_local, size, levels, f"shard [{first}, +{cnt})")
        assert len(got) == len(want) > 0, (first, cnt)
        np.testing.assert_array_equal(got, want, err_msg=f"shard [{first}, +{cnt})")
        ctx.free(hpb_local)
        ctx.close()
    ctx0.free(hpb_dev)
    ctx0.close()


def test_hpb_refuses_levels_outside_build_range(capi, orc):
    sc = box_scene()
    ctx = make_ctx(capi, sc, views=2)
    cam = sc.camera()
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    clip = clipmaps_for(sc, 2, [(0, 0)])
    hpb_dev = ctx.alloc(2 * 64 * 64 * 2)
    flags_dev = ctx.alloc(8)
    ctx.upload(flags_dev, np.ones(2, np.uint32))
    for levels in (0, 17, 40):
        with pytest.raises(capi.OxcError):
            ctx.cull_meshlets_hpb(cam, clip, [1, 1], hpb_dev, 64, levels)
        with pytest.raises(capi.OxcError):
            ctx.cull_meshlets_hpb_dirty_dev(cam, clip, flags_dev, hpb_dev, 64, levels)
    with pytest.raises(capi.OxcError):
        ctx.build_hpb(hpb_dev, 64, 2, hpb_dev, 17)
    ctx.free(hpb_dev)
    ctx.free(flags_dev)
    ctx.close()


# ------------------------------------------------------------------------------------------------------------------------------
# the engine's pass order on one context, with and without a bound device camera
# ------------------------------------------------------------------------------------------------------------------------------
def _views(sc, n, seed):
    dirs = synth.uniform(sc.seed + seed, 90, 3 * n, -1.0, 1.0).reshape(n, 3)
    dirs[:, 1] = -np.abs(dirs[:, 1]) - 0.2
    return np.concatenate([synth.make_ortho_view(dirs[v], (0.0, 0.0, -200.0), 60.0 * (1 + v % 4), 800.0, sc.mesh_instance_count)
                           for v in range(n)])


@pytest.mark.parametrize("mode", ["unbound", "bound", "renderer"])
def test_engine_order_with_bound_camera(capi, orc, mode):
    """cull_meshes(main) -> cull_meshlets(main, Hi-Z) -> hpb(coarse) -> cull_triangles(main) and multiview -> decode(main) on one
    context: every output equals the oracle.  "bound": a device buffer holding the main camera is bound (oxc_bind_camera_buffer), so
    the main-view passes read it, and the shadow cull must still cull against its coarse argument.  "renderer": the same calls on
    Renderer.ctx after submit / wait; where the frame replayed from a CUDA graph the frame camera is still bound, where capture is
    unavailable submit ran eagerly and unbound.  A replayed graph does not advance oxc_kernel_launch_count; eager launches do."""
    sc = box_scene()
    hs = orc.HostScene(sc)
    w, h = sc.width, sc.height
    main = sc.camera(4.0)
    renderer, cam_dev, graph_path = None, None, None
    if mode == "renderer":
        renderer = capi.Renderer(0, sc, max_views=abi.MAX_VIEWS)
        renderer.set_external_depth(sc.occluder_depth)
        bufs = dict(vis32=np.zeros((h, w), np.uint32), depth=np.zeros((h, w), np.float32), idx=np.zeros(sc.max_meshlet_instance_count, np.uint32))
        for yaw in (1.0, 2.0):  # each of the two slots captures its own graph on its first frame
            renderer.wait(renderer.submit(sc.camera(yaw), bufs))
        before = capi.kernel_launch_count()
        renderer.wait(renderer.submit(main, bufs))
        graph_path = capi.kernel_launch_count() == before
        ctx = renderer.ctx
        print(f"renderer: frame {'replayed from a CUDA graph (camera left bound)' if graph_path else 'ran eagerly (unbound)'}")
    else:
        ctx = make_ctx(capi, sc, reordered=True, views=abi.MAX_VIEWS)
        if mode == "bound":
            cam_dev = ctx.alloc(abi.CULL_CAMERA_DT.itemsize)
            ctx.upload(cam_dev, main)
            ctx.bind_camera_buffer(cam_dev)
    mask0 = np.random.default_rng(7).integers(0, 2**32, size=ctx.out.visibility_mask_words, dtype=np.uint64).astype(np.uint32)
    hiz = orc.build_hiz(sc.occluder_depth, orc.Hiz(*sc.hiz_extent()))
    # 1. mesh pass
    mi, vis, _ = orc.cull_meshes(hs, main, abi.CULL_TEST_ALL)
    total = int(vis["total"][0])
    ctx.cull_meshes(main, abi.CULL_TEST_ALL)
    assert int(ctx.visibility()["total"][0]) == total
    np.testing.assert_array_equal(ctx.meshlet_instances(total), mi[:total])
    # 2. early meshlet pass against a pyramid written from outside
    ctx.upload_hiz(hiz.data)
    ctx.mark_hiz_dirty()
    ctx.set_mask(mask0)
    ctx.cull_meshlets(main, abi.CULL_TEST_ALL, True)
    mask = mask0.copy()
    visible, _ = orc.cull_meshlets_hiz(hs, mi, vis, main, abi.CULL_TEST_ALL, hiz, mask)
    e = int(vis["early"][0])
    assert int(ctx.visibility()["early"][0]) == e > 0
    np.testing.assert_array_equal(np.sort(ctx.visible_indices(e)), np.sort(visible[:e]), err_msg=f"{mode}: meshlet pass")
    np.testing.assert_array_equal(ctx.mask(), mask, err_msg=f"{mode}: mask")
    # 3. shadow-clipmap cull on a narrow coarse view
    rng = np.random.default_rng(9)
    coarse = coarse_view(sc, half=15.0)
    clip = clipmaps_for(sc, 4, offset_patterns(32, rng)[-1])
    hpb = np.ones(orc.hpb_layout(32, 4, 6)[1], dtype=np.uint8)
    hpb_dev = ctx.alloc(hpb.nbytes)
    ctx.upload(hpb_dev, hpb)
    ref_hpb, _ = orc.cull_meshlets_hpb(hs, mi, vis, coarse, clip, [1] * 4, hpb, 32, 6)
    got = run_hpb_both(ctx, coarse, clip, [1] * 4, hpb_dev, 32, 6, f"{mode}: hpb")
    np.testing.assert_array_equal(got, np.sort(ref_hpb), err_msg=f"{mode}: shadow cull on the coarse view")
    # the coarse view decides: culled against the main camera's planes instead, the survivors would differ
    main_planes = coarse.copy()
    main_planes["projection_view"] = main["projection_view"]
    assert not np.array_equal(np.sort(orc.cull_meshlets_hpb(hs, mi, vis, main_planes, clip, [1] * 4, hpb, 32, 6)[0]), got)
    n_hpb = len(got)
    # 4. triangle cull on the main view over the shadow cull's survivor list, and the multi-view cull
    if ctx.out.reordered_indices:
        ref_idx, ref_draw = orc.cull_triangles(hs, mi, np.asarray(ref_hpb, np.uint32), 0, n_hpb, main)
        ctx.cull_triangles(main, abi.CULL_TEST_ALL)
        ic = int(ctx.draw_cmd()["index_count"][0])
        assert ic == int(ref_draw["index_count"][0]) > 0, mode
        g, r = ctx.reordered_indices(ic).reshape(-1, 3), ref_idx.reshape(-1, 3)
        np.testing.assert_array_equal(g[np.lexsort(g.T[::-1])], r[np.lexsort(r.T[::-1])], err_msg=f"{mode}: triangle cull")
    views = _views(sc, 3, 1)
    ref_bits, ref_counts = orc.cull_meshlets_multiview(hs, mi, total, views, 1)
    ctx.cull_meshlets_multiview(views, 1)
    np.testing.assert_array_equal(ctx.view_bits(total), ref_bits, err_msg=f"{mode}: multiview bits")
    np.testing.assert_array_equal(ctx.view_counts(), ref_counts, err_msg=f"{mode}: multiview counts")
    # 5. decode on the main view: a vis buffer of the early survivors' first triangles, with cleared texels
    dw, dh = 64, 48
    ids = np.sort(visible[:e])[np.random.default_rng(5).integers(0, e, size=dw * dh)]
    v32 = ((ids.astype(np.uint32) << np.uint32(8))).reshape(dh, dw)
    v32[::5, ::3] = abi.VIS_CLEAR
    want = orc.decode_visbuffer(hs, mi, total, main, v32)
    v32_dev = ctx.alloc(v32.nbytes)
    ctx.upload(v32_dev, v32)
    dev = {k: ctx.alloc(dw * dh * 16) for k in want}
    ctx.decode_visbuffer(main, dw, dh, dev, vis32_dev=v32_dev)
    for k, p in dev.items():
        _assert_planes_equal(ctx.download(p, np.float32, dw * dh * 4).reshape(dh, dw, 4), want[k], f"{mode}: decode {k}")
        ctx.free(p)
    assert (want["lambda_"][:, :, 3] == 1.0).sum() > 100
    for p in (hpb_dev, v32_dev, cam_dev):
        if p is not None:
            ctx.free(p)
    if renderer is not None:
        renderer.close()
    else:
        ctx.close()


# ------------------------------------------------------------------------------------------------------------------------------
# multi-view cull
# ------------------------------------------------------------------------------------------------------------------------------
def perspective_views(sc, n):
    return np.concatenate([sc.camera(7.0 * v - 20.0) for v in range(n)])


@pytest.mark.parametrize("scene_name", ["box", "hostile", "sharded"])
def test_multiview_view_counts(capi, orc, scene_name):
    """n_views 1, 2, 3, 7, 15, 16, directional and positional, on a max_views = 16 context: bits and all 16 counts.  A 16-view call
    followed by a 3-view call leaves counts[3:] == 0 and no bit above bit 2.  More views than max_views are refused."""
    sc = hostile_scene() if scene_name == "hostile" else box_scene()
    hs = orc.HostScene(sc)
    ctx = make_ctx(capi, sc, views=abi.MAX_VIEWS)
    cam = sc.camera()
    mi, vis, _ = orc.cull_meshes(hs, cam, abi.CULL_TEST_ALL)
    total = int(vis["total"][0])
    n = sc.mesh_instance_count
    first, count, id_lo = 0, n, 0
    if scene_name == "sharded":  # the shard's local meshlet list is the whole list's slice of its mesh instances
        first, count = n // 3, n // 2
        ctx.set_shard_auto(first, count)
        owner = mi["mesh_instance_index"][:total]
        sel = np.nonzero((owner >= first) & (owner < first + count))[0]
        id_lo, total = int(sel[0]), len(sel)
        assert np.array_equal(sel, np.arange(id_lo, id_lo + total))
        mi = np.ascontiguousarray(mi[id_lo:id_lo + total])
    ctx.cull_meshes(cam, abi.CULL_TEST_ALL)
    assert int(ctx.visibility()["total"][0]) == total > 0
    seen = set()
    for directional in (1, 0):
        all_views = _views(sc, abi.MAX_VIEWS, 2) if directional else perspective_views(sc, abi.MAX_VIEWS)
        for nv in (1, 2, 3, 7, 15, 16):
            views = all_views[:nv]
            ref_bits, ref_counts = orc.cull_meshlets_multiview(hs, mi, total, views, directional)
            ctx.cull_meshlets_multiview(views, directional)
            tag = f"{scene_name}: {nv} views, directional {directional}"
            np.testing.assert_array_equal(ctx.view_bits(total), ref_bits, err_msg=tag)
            np.testing.assert_array_equal(ctx.view_counts(), ref_counts, err_msg=tag)
            assert not (ref_bits >> np.uint32(nv)).any() and not ref_counts[nv:].any(), tag
            seen.add(tuple(ref_counts[:nv] > 0))
        ctx.cull_meshlets_multiview(all_views, directional)
        ctx.cull_meshlets_multiview(all_views[:3], directional)
        bits, counts = ctx.view_bits(total), ctx.view_counts()
        assert not counts[3:].any() and not (bits >> np.uint32(3)).any(), f"{scene_name}: 16 views then 3"
        np.testing.assert_array_equal(counts[:3], orc.cull_meshlets_multiview(hs, mi, total, all_views[:3], directional)[1][:3])
    assert any(any(s) for s in seen)
    with pytest.raises(capi.OxcError):
        ctx.cull_meshlets_multiview(np.concatenate([all_views, all_views[:1]]), 1)
    small = make_ctx(capi, sc, views=4)
    small.cull_meshes(cam, abi.CULL_TEST_ALL)
    with pytest.raises(capi.OxcError):
        small.cull_meshlets_multiview(all_views[:5], 1)
    small.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------------------------------------
# terrain cull
# ------------------------------------------------------------------------------------------------------------------------------
TERRAIN_GRIDS = [(1, 1), (7, 5), (33, 31), (256, 1), (1, 300), (512, 512)]
TERRAIN_W, TERRAIN_H = 640, 360


def terrain_record(nx, ny, height_scale=40.0):
    t = np.zeros(1, dtype=abi.TERRAIN_DT)
    t["world_min"][0] = (np.float32(-301.37), np.float32(-503.113))  # not exact in binary32 arithmetic
    t["world_size"][0] = (np.float32(611.3), np.float32(597.7))
    t["patch_count"][0] = (nx, ny)
    t["base_height"] = np.float32(-30.3)
    t["height_scale"] = height_scale
    return t


def terrain_cameras():
    return {"above": synth.make_camera(TERRAIN_W, TERRAIN_H, 0, yaw_deg=8.0, eye=(0.0, 5.0, 60.0)),
            "ground": synth.make_camera(TERRAIN_W, TERRAIN_H, 0, yaw_deg=-30.0, eye=(3.0, -28.0, -100.0)),
            "away": synth.make_camera(TERRAIN_W, TERRAIN_H, 0, yaw_deg=180.0, eye=(0.0, 5.0, 400.0))}


def terrain_minmax(rng, n):
    lo = rng.random(n, dtype=np.float32) * 0.6
    mm = np.stack([lo, lo + rng.random(n, dtype=np.float32) * 0.4], axis=1).astype(np.float32)
    mm[::7, 1] = mm[::7, 0]  # flat patches: the 1e-3 floor of the extent
    return mm


def terrain_pyramids(orc, rng):
    hw, hh = abi.hiz_extent(TERRAIN_W, TERRAIN_H)
    depth = (rng.random((TERRAIN_H, TERRAIN_W), dtype=np.float32) * 0.02).astype(np.float32)
    depth[100:260, 150:500] = 0.01
    return {"cleared": orc.Hiz(hw, hh), "built": orc.build_hiz(depth, orc.Hiz(hw, hh)),
            "external": orc.build_hiz(np.ascontiguousarray(depth[::-1, ::-1]), orc.Hiz(hw, hh))}, depth


SENTINEL = 0xA5A5A5A5


def run_terrain(ctx, orc, t, mm, mm_dev, cam, flags, hiz, mask, dev, tag):
    """one pass on the device from `mask`, checked against the oracle (which updates `mask`): survivors, mask, draw command, and the
    sentinels past the last patch.  Returns the oracle's survivors."""
    n = int(t["patch_count"][0][0]) * int(t["patch_count"][0][1])
    words = (n + 31) // 32
    vis_dev, mask_dev, cmd_dev = dev
    ctx.upload(vis_dev, np.full(n + 64, SENTINEL, np.uint32))
    ctx.upload(mask_dev, np.concatenate([mask, np.full(4, SENTINEL, np.uint32)]))
    ctx.upload(cmd_dev, np.full(4, 0xDEADBEEF, np.uint32))
    ref, ref_cmd = orc.cull_terrain(t, mm, cam, flags, hiz, mask)
    ctx.cull_terrain(t, mm_dev, cam, flags, vis_dev, mask_dev, cmd_dev)
    cmd = ctx.download(cmd_dev, np.uint32, 4)
    k = int(ref_cmd["instance_count"][0])
    assert tuple(int(x) for x in cmd) == (4, k, 0, 0), tag
    got = ctx.download(vis_dev, np.uint32, n + 64)
    np.testing.assert_array_equal(np.sort(got[:k]), np.sort(ref), err_msg=f"{tag}: survivors")
    assert (got[k:] == SENTINEL).all(), f"{tag}: visible_patches written past the count"
    gm = ctx.download(mask_dev, np.uint32, words + 4)
    np.testing.assert_array_equal(gm[:words], mask, err_msg=f"{tag}: mask")
    assert (gm[words:] == SENTINEL).all(), f"{tag}: mask words past the last patch"
    return ref


FLAG_SUBSETS = [f | o | l for f in (0, FRUSTUM) for o in (0, OCC) for l in (0, LATE)]


@pytest.mark.parametrize("grid", TERRAIN_GRIDS, ids=lambda g: f"{g[0]}x{g[1]}")
def test_terrain_shapes(capi, orc, grid):
    """every grid x three cameras x three Hi-Z states x all 8 flag subsets from a random mask (the bits past the last patch set),
    height_scale 40, 0 (the extent floor) and negative; then an early -> late sequence over three frames.  The oracle agrees with
    float64 throughout."""
    nx, ny = grid
    n = nx * ny
    rng = np.random.default_rng(nx * 1000 + ny)
    hw, hh = abi.hiz_extent(TERRAIN_W, TERRAIN_H)
    pyramids, depth = terrain_pyramids(orc, rng)
    ctx = capi.Context(0, 1, 1, hw, hh)
    d_dev = ctx.alloc(depth.nbytes)
    ctx.upload(d_dev, depth)
    mm = terrain_minmax(rng, n)
    mm_dev = ctx.alloc(mm.nbytes)
    ctx.upload(mm_dev, mm)
    words = (n + 31) // 32
    dev = (ctx.alloc((n + 64) * 4), ctx.alloc((words + 4) * 4), ctx.alloc(16))
    emitted, excused, decisions = set(), 0, 0
    for hscale in (40.0, 0.0, -25.0) if n < 100_000 else (40.0,):  # the 512 x 512 grid: one height scale
        t = terrain_record(nx, ny, hscale)
        for cam_name, cam in terrain_cameras().items():
            for state, pyr in pyramids.items():
                if state == "built":
                    ctx.build_hiz(d_dev, TERRAIN_W, TERRAIN_H)
                else:
                    ctx.clear_hiz()
                    if state == "external":
                        ctx.upload_hiz(pyr.data)
                        ctx.mark_hiz_dirty()
                levels = [pyr.level(l) for l in range(pyr.levels)]
                for flags in FLAG_SUBSETS:
                    mask = rng.integers(0, 2**32, size=words, dtype=np.uint64).astype(np.uint32)
                    before = mask.copy()
                    tag = f"{nx}x{ny} scale {hscale} camera {cam_name} pyramid {state} flags {flags:#x}"
                    ref = run_terrain(ctx, orc, t, mm, mm_dev, cam, flags, pyr, mask, dev, tag)
                    emitted.add((cam_name, len(ref) > 0))
                    emit, visible, near = f64_terrain(t, mm, cam, flags, levels, hw, hh, before)
                    excused += assert_f64_agrees(tag, survivors_to_mask(ref, n), emit, near)
                    assert_f64_agrees(tag + ": mask", mask_bits(mask, n), visible if flags & (OCC | LATE) else mask_bits(before, n), near)
                    decisions += n
        # early -> late over three frames from a cleared mask, on the built pyramid, the camera moving
        ctx.build_hiz(d_dev, TERRAIN_W, TERRAIN_H)
        mask = np.zeros(words, np.uint32)
        for f in range(3):
            cam = synth.make_camera(TERRAIN_W, TERRAIN_H, 0, yaw_deg=8.0 + 6.0 * f, eye=(0.0, 5.0, 60.0 - 20.0 * f))
            for flags in (FRUSTUM | OCC, FRUSTUM | OCC | LATE):
                run_terrain(ctx, orc, t, mm, mm_dev, cam, flags, pyramids["built"], mask, dev, f"{nx}x{ny} frame {f} flags {flags:#x}")
    print(f"terrain {nx}x{ny}: {excused} of {decisions} float64 decisions excused")
    assert excused <= EXCUSED_BOUND * decisions
    assert ("above", True) in emitted
    for p in (d_dev, mm_dev) + dev:
        ctx.free(p)
    ctx.close()
