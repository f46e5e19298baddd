"""The VSM shadow-resolve oracle (oracle/oxc_oracle_vsm_resolve.c) and the shadow-raster oracle (oracle/oxc_oracle_vsm_draw.c)
against an independent binary64 restatement of the reference's shaders, over ray-cast analytic frames with unit-length suns and
over random frames.

The restatement is vectorised numpy written from the shader text, not from the oracle.  It does not call the oracle's helpers or
the device header.  Function by function:
- `hash2`: passes/resolve_shadowmaps.slang:27-30;
- `lookup`, `chain`: :32-61 and :63-75, with rmvsm.slang:99-106 (get_physical_coords), :129-138 (the page wrap), :200-206
  (get_virt_coords) and :214-221 (get_clipmap_info), common/math.slang:95-101 (com::mod);
- `basis`: :77-82;
- `pcss`: :84-185, with common/math.slang:189-191 (hammersley2d);
- `restate`: :187-209, with common/encoding.slang:7-15 (oct_to_vec3), rmvsm.slang:147-188 (texel length and clipmap selection)
  and scene.slang:189-193 (unproject_uv).

Everything is binary64 except where the shader's result depends chaotically on the last bits:
- the normal's .zw is rounded to binary16 first: the reference stores it in an R16G16B16A16Sfloat attachment;
- hash2 takes its dot product in binary32 in the shader's order (its argument reaches 1.4e6), sin in binary64 rounded once to
  binary32, and `* 43758.5453` and fract in binary32.  A pixel whose noise still differs from the oracle's is ambiguous.
NaN follows the specification's rules (oracle header, items 6-7), not numpy's: max / min return the other operand, NaN passes
the clip-uv range test, float -> int saturates and NaN converts to 0.

Decision margins.  A pixel's output is 1, 0 or f32(k / n), n <= 24, so a pixel on which no decision is near its threshold equals
the oracle bit for bit.  Each decision records its distance from the jump divided by its epsilon (its ratio):
- per lookup (centre, 16 blocker taps, 24 PCF taps, each with up to three fall-back lookups): cu * size and cv * size from a page
  boundary, cu * P and cv * P from a texel boundary (EPS_UV in uv units; the clip-uv range test at 0 and 1 coincides with the page
  boundaries there, where page -1 and page `size` miss);
- per tap: d + bias_norm - d_recv from 0 (EPS_CMP) and hammersley.x + noise.x from 1, where fract jumps the radius (EPS_XI);
- per pixel: bias + level_f from its ceiling jump (EPS_LEVEL, in log2 units of the raw level) and NoL from 0.99 (EPS_NOL).
A near decision makes a pixel ambiguous only when evaluating both sides changes the result: both candidate pages or texels (and
both together), both comparison outcomes, the pixel again with the clipmap index one lower and one higher, the other bias branch.
A blocker tap whose candidates are all blockers with different depths does not make the pixel ambiguous; it widens the PCF radius
by the spread and the PCF taps' EPS_UV and EPS_CMP by what that moves them.  A pixel whose only ambiguous taps are PCF taps with
unchanged blocker-search outcomes is bounded: |delta| <= k / max(valid - k, 1) for k such taps.  The denominator is valid - k
rather than valid because an ambiguous tap may switch between a hit and a miss, which changes the count the oracle divides by.

Constants and what was measured (oracle against restatement, every scene and frame below):
- EPS_UV = 4e-6, EPS_CMP = 4e-6, EPS_LEVEL = 4e-4, EPS_NOL = 1e-5, EPS_XI = 1e-6.  Every disagreeing pixel is ambiguous at a
  quarter of these epsilons (`MARGIN`: the check runs at 0.25 x and at 1 x); the largest ratio (margin / epsilon) among
  disagreeing pixels is printed per scene as `worst ratio`.  Measured: 3 of the 12 analytic scenes disagree, on 1 or 2 pixels
  each, worst ratio 0.0023; the random frames disagree on 24 and 6 pixels, worst ratio 0.011.  No pixel's noise differs from the
  oracle's on any frame here.
- ambiguous fraction of the non-sky pixels: under AMBIGUOUS_ANALYTIC = 0.10 (measured 0.042 to 0.059) and AMBIGUOUS_RANDOM = 0.5
AMBIGUOUS_CLOSE_UP = 0.6
  (measured 0.37 on the reference shape and 0.12 on the uneven one: random atlases put a depth step at every texel).
- the analytic frames are 96 x 54 (reference atlas shape) and 128 x 72 (uneven shape) pixels; the clipmap selection is given a
  1920 x 1080 camera resolution, so it picks the clipmaps a full-size frame picks for these world points.
- the atlas cast (part 2): tolerance |grad z| * sqrt(2) / 256 + 4 binary32 ulps of 1, grad z per atlas pixel; a texel is in the
  silhouette band when the cast depth at its sample moved by EPS_EDGE = 1/64 px along x or y leaves the plane of its own caster
  (changes by more than 2 * |grad z| * EPS_EDGE plus the tolerance).  The band stays under EDGE_BOUND = 2 % of the cast texels
  (measured at most 0.02 %); outside it the oracle's draw is within 0.39 of the tolerance.

Mutations: each family (`EXPOSED`) names the mutations that make at least MUTATION_MIN unambiguous pixels disagree with the oracle
on one of its scenes.  Measured best counts: analytic reference 4: 66, 5: 1065, 6: 70, 7: 20, 10: 67 (1: 9, 3: 7); analytic
uneven 1: 31, 3: 25, 4: 827, 5: 2758, 6: 949, 7: 106, 8: 423, 10: 181; random reference 1: 358, 3: 332, 4: 82, 5: 1513, 6: 1775,
7: 1353, 10: 24; random uneven 1: 550, 3: 494, 5: 1962, 6: 1917, 7: 956, 8: 75, 10: 20.  Mutations 2 (the lerp reversed) and 9
(the hard shadow at blockers == 0) flip at most 1 and 2 pixels on those frames: the PCF bias term decides a comparison only where
the PCF radius is wide over a receiver at a slant, and the hard shadow differs from 1 only where the centre is shadowed while every
search tap misses.  The two close-ups (192 x 108, every reached entry Backed) are built for them: the high caster's penumbra under
the 20-degree sun flips 55 pixels under mutation 2, and the 1/128 m strip under the 88.5-degree sun flips 42 under mutation 9.
Their ambiguous fractions (0.15 and 0.05) stay under AMBIGUOUS_CLOSE_UP = 0.6: 0.46 was measured on a strip view under the low sun,
where fine clipmaps put the ground's own search taps next to the bias.

Cost: the module takes 69 s on 8 pytest-xdist workers and 3.8 CPU-minutes in all (x86-64 host); most of it is the ten mutated
restatements per scene.
"""
import numpy as np
import pytest

from oxylus_b200 import abi, synth

f32 = np.float32
f64 = np.float64

B, D, V = abi.VSM_PAGE_BACKED, abi.VSM_PAGE_DIRTY, abi.VSM_PAGE_VISIBLE
MISS = -1.0

EPS_UV = 4e-6
EPS_CMP = 4e-6
EPS_LEVEL = 4e-4
EPS_NOL = 1e-5
EPS_XI = 1e-6
MARGIN = 0.25
AMBIGUOUS_ANALYTIC = 0.10
AMBIGUOUS_RANDOM = 0.5
AMBIGUOUS_CLOSE_UP = 0.6
EPS_EDGE = 1.0 / 64.0
EDGE_BOUND = 0.02
MUTATION_MIN = 20
# the mutations each family must expose (at least MUTATION_MIN unambiguous disagreements on one of its scenes)
EXPOSED = {"analytic reference": (4, 5, 6, 7, 10), "analytic uneven": (1, 3, 4, 5, 6, 7, 8, 10), "random reference": (1, 3, 4, 5, 6, 7, 10), "random uneven": (1, 3, 5, 6, 7, 8, 10),
           "close-up penumbra": (2,), "close-up strip": (9,)}

# the shader's binary32 constants, as values (resolve_shadowmaps.slang:19-25, common/math.slang:5, :95-97)
BLOCKER_SAMPLES, PCF_SAMPLES = 16, 24
SEARCH_RADIUS, LIGHT_WIDTH, MAX_PCF_RADIUS = f64(f32(0.1)), f64(f32(0.002)), f64(f32(0.1))
TAU = f64(f32(6.283185307179586))
SQRT2 = f64(f32(1.41421356))
QUANTIZE = 2.0 / (1 << 23)

MUTATIONS = {
    1: "noise.xy in the PCF loop",
    2: "lerp(0, pcf_bias, NoL)",
    3: "bitangent = cross(t, L)",
    4: "fall-back +1 before -1",
    5: "page offset subtracted in the wrap",
    6: "floor in the clipmap selection",
    7: "hammersley2d without reversebits",
    8: "receiver depth from the un-offset position",
    9: "hard shadow when blockers == 0",
    10: "out-of-atlas read taken as a miss",
}


# -- scalar rules of the specification ---------------------------------------------------------------------------------------------
def vmax(a, b):
    return np.where(np.isnan(b) | (a > b), a, b)


def vmin(a, b):
    return np.where(np.isnan(b) | (a < b), a, b)


def sat_i32(x):
    x = np.asarray(x, f64)
    return np.where(np.isnan(x), 0.0, np.clip(x, -2147483648.0, 2147483647.0)).astype(np.int64)


def frac(x):
    return x - np.floor(x)


def dot(a, b):
    return (a * b).sum(-1)


def normalize(v):
    with np.errstate(invalid="ignore", divide="ignore"):
        return v / np.sqrt(dot(v, v))[..., None]


def round_half(x):
    with np.errstate(over="ignore"):
        return np.asarray(x, f32).astype(np.float16).astype(f64)


def hash2(px, py):
    """:27-30.  dot in binary32 in the shader's order, sin in binary64 rounded once, the scale and fract in binary32"""
    px, py = f32(px), f32(py)
    out = []
    for a, b in ((127.1, 311.7), (269.5, 183.3)):
        d = px * f32(a) + py * f32(b)
        s = np.sin(d.astype(f64)).astype(f32)
        t = s * f32(43758.5453)
        out.append((t - np.floor(t)).astype(f64))
    return np.stack(out, -1)


def oct_to_vec3(e):
    """common/encoding.slang:7-15"""
    x, y = e[..., 0], e[..., 1]
    z = 1.0 - np.abs(x) - np.abs(y)
    sx, sy = np.where(x >= 0.0, 1.0, -1.0), np.where(y >= 0.0, 1.0, -1.0)
    neg = z < 0.0
    vx = np.where(neg, (1.0 - np.abs(y)) * sx, x)
    vy = np.where(neg, (1.0 - np.abs(x)) * sy, y)
    return normalize(np.stack([vx, vy, z], -1))


def hammersley(i, n, mutation=0):
    """common/math.slang:189-191"""
    rev = int(f"{i:032b}"[::-1], 2) if mutation != 7 else i
    return f64(i) / f64(n), f64(rev) * 2.3283064365386963e-10


def basis(L, mutation=0):
    """:77-82"""
    axis = np.array([0.0, 1.0, 0.0]) if abs(L[1]) < f64(f32(0.999)) else np.array([1.0, 0.0, 0.0])
    t = normalize(np.cross(axis, L))
    return t, (np.cross(t, L) if mutation == 3 else np.cross(L, t))


# -- the frame ---------------------------------------------------------------------------------------------------------------------
class Frame:
    """the resolve's inputs in binary64: clipmap matrices (row-major), page offsets, page tables, atlas, VSM constants"""

    def __init__(self, vsm, clipmaps, page_tables, atlas):
        v = vsm.reshape(-1)[0]
        self.size, self.P, self.ps = int(v["page_table_size"]), int(v["physical_page_table_size"]), int(v["page_size"])
        self.count = int(v["clipmap_count"])
        self.npp = self.P // self.ps
        self.bias, self.z_length = f64(v["clipmap_selection_bias"]), f64(v["z_length"])
        self.L = np.asarray(v["directional_light_dir"], f64)
        self.texel_length = (f64(v["first_clipmap_width"]) * ((self.size - 1) / self.size) * 2.0) / f64(v["virtual_extent"])
        self.mats = np.stack([np.asarray(clipmaps["projection_view_mat"][k], f64).reshape(4, 4).T for k in range(len(clipmaps))])
        self.off = np.asarray(clipmaps["page_offset"], np.int64)
        self.pt = np.asarray(page_tables, np.uint32)
        self.atlas = np.asarray(atlas, f32).astype(f64)
        # uv per world unit of each clipmap, for the PCF radius' uncertainty
        self.uv_per_m = 0.5 * np.maximum(np.linalg.norm(self.mats[:, 0, :3], axis=1), np.linalg.norm(self.mats[:, 1, :3], axis=1))
        self.ortho = np.all(self.mats[:, 3] == np.array([0.0, 0.0, 0.0, 1.0]), axis=1)


class Stats:
    def __init__(self):
        self.c = {}

    def add(self, k, n):
        self.c[k] = self.c.get(k, 0) + int(n)


def clip_info(fr, ci, pos):
    """rmvsm.slang:214-221"""
    m = fr.mats[np.clip(ci, 0, fr.count - 1)]
    h = np.einsum("nij,nj->ni", m, np.concatenate([pos, np.ones((len(pos), 1))], 1))
    with np.errstate(invalid="ignore", divide="ignore"):
        return (h[:, 0] / h[:, 3] + 1.0) * 0.5, (h[:, 1] / h[:, 3] + 1.0) * 0.5, h[:, 2] / h[:, 3]


def fetch(fr, ci, vx, vy, tx, ty, mutation=0, st=None):
    """:37-60 from the virtual page and the virtual texel: the atlas value, MISS, or 0 beyond the atlas"""
    out = np.full(len(ci), MISS)
    ok = (ci >= 0) & (ci < fr.count) & (vx >= 0) & (vy >= 0) & (vx <= fr.size - 1) & (vy <= fr.size - 1)
    c = np.clip(ci, 0, fr.count - 1)
    sgn = -1 if mutation == 5 else 1
    wx, wy = (vx + sgn * fr.off[c, 0]) % fr.size, (vy + sgn * fr.off[c, 1]) % fr.size
    e = np.where(ok, fr.pt[c, np.where(ok, wy, 0), np.where(ok, wx, 0)], 0).astype(np.int64)
    ok &= (e & B) != 0
    addr = e >> 16
    ax, ay = (addr % fr.npp) * fr.ps + tx % fr.ps, (addr // fr.npp) * fr.ps + ty % fr.ps
    inside = (ax < fr.P) & (ay < fr.P)
    val = fr.atlas[np.where(inside & ok, ay, 0), np.where(inside & ok, ax, 0)]
    out[ok] = np.where(inside, val, MISS if mutation == 10 else 0.0)[ok]
    if st is not None:
        st.add("out_of_atlas_reads", (ok & ~inside).sum())
        st.add("non_ortho_reads", (ok & ~fr.ortho[c]).sum())
    return out


def lookup(fr, ci, pos, mutation=0, eps_uv=None, st=None):
    """one sample_vsm_shadow_depth: (value, alternates, their ratios).  The alternates take the other page and / or texel on each
    axis whose coordinate lies within eps_uv of a boundary."""
    n = len(ci)
    cu, cv, _ = clip_info(fr, ci, pos)
    inr = ~((cu < 0.0) | (cv < 0.0) | (cu > 1.0) | (cv > 1.0))
    with np.errstate(invalid="ignore"):
        vx, vy = sat_i32(np.floor(cu * fr.size)), sat_i32(np.floor(cv * fr.size))
        tx, ty = sat_i32(np.floor(cu * fr.P)), sat_i32(np.floor(cv * fr.P))
    vxm, vym = np.where(inr, vx, -1), np.where(inr, vy, -1)
    val = fetch(fr, ci, vxm, vym, tx, ty, mutation, st)
    if eps_uv is None:
        return val, None, None
    axes = []
    for u, vv, t in ((cu, vx, tx), (cv, vy, ty)):
        with np.errstate(invalid="ignore"):
            kp, kt = np.round(u * fr.size), np.round(u * fr.P)
            rp = np.abs(u * fr.size - kp) / fr.size / eps_uv
            rt = np.abs(u * fr.P - kt) / fr.P / eps_uv
        rp, rt = np.where(np.isnan(rp), np.inf, rp), np.where(np.isnan(rt), np.inf, rt)
        va, ta = 2 * sat_i32(kp) - 1 - vv, 2 * sat_i32(kt) - 1 - t
        axes.append([(vv, t, np.zeros(n)), (va, t, rp), (vv, ta, rt), (va, ta, np.maximum(rp, rt))])
    near = np.zeros(n, bool)
    for _, _, r in axes[0][1:] + axes[1][1:]:
        near |= r < 1.0
    alts, ratios = np.full((n, 15), MISS), np.full((n, 15), np.inf)
    idx = np.nonzero(near)[0]
    if len(idx):
        k = 0
        for ox in range(4):
            for oy in range(4):
                if ox == 0 and oy == 0:
                    continue
                ax_, ay_ = axes[0][ox], axes[1][oy]
                r = np.maximum(ax_[2][idx], ay_[2][idx])
                a = fetch(fr, ci[idx], ax_[0][idx], ay_[0][idx], ax_[1][idx], ay_[1][idx], mutation)
                alts[idx, k], ratios[idx, k] = a, np.where(r < 1.0, r, np.inf)
                k += 1
    return val, alts, ratios


def chain(fr, ci, pos, mutation=0, eps_uv=None, st=None):
    """:63-75: the first of clipmap ci, ci - 1, ci + 1 that does not miss, with the alternates of one lookup at a time"""
    order = (0, 1, -1) if mutation == 4 else (0, -1, 1)
    parts = [lookup(fr, ci + d, pos, mutation, eps_uv, st) for d in order]
    vals = [p[0] for p in parts]

    def pick(v0, v1, v2):
        return np.where(v0 != MISS, v0, np.where(v1 != MISS, v1, v2))

    val = pick(*vals)
    if st is not None and mutation != 4:
        st.add("fallback_minus_hit", ((vals[0] == MISS) & (vals[1] != MISS)).sum())
        st.add("fallback_plus_hit", ((vals[0] == MISS) & (vals[1] == MISS) & (vals[2] != MISS)).sum())
    if eps_uv is None:
        return val, None, None
    alts, ratios = [], []
    for s in range(3):
        a, r = parts[s][1], parts[s][2]
        vs = [np.repeat(v[:, None], a.shape[1], 1) for v in vals]
        vs[s] = a
        alts.append(pick(*vs))
        ratios.append(r)
    return val, np.concatenate(alts, 1), np.concatenate(ratios, 1)


def select_clipmap(fr, inv_pv, res, u, v, d, mutation=0):
    """rmvsm.slang:157-188 (VMS_USE_DIAG_PIXEL_FOOTPRINT): the index, and the raw level's distance from the ceiling's jump"""
    ox, oy = 0.5 / res[0], 0.5 / res[1]
    a, b = unproject(inv_pv, u - ox, v + oy, d), unproject(inv_pv, u + ox, v + oy, d)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.log2(np.linalg.norm(a - b, axis=-1) / fr.texel_length)
    lf = fr.bias + vmax(r, 0.0)
    lv = np.floor(lf) if mutation == 6 else np.ceil(lf)
    ci = np.minimum(np.where(np.isnan(lv), 0, np.clip(np.nan_to_num(lv, nan=0.0), 0, 4294967295.0)), fr.count - 1).astype(np.int64)
    # the jumps of ceil(bias + max(r, 0)) lie at r = k - bias >= 0; the smallest is ceil(bias) - bias
    j0 = np.ceil(fr.bias) - fr.bias
    with np.errstate(invalid="ignore"):
        x = fr.bias + r
        m = np.where(r <= j0, j0 - r, np.minimum(x - np.floor(x), np.ceil(x) - x))
    return ci, np.where(np.isfinite(m), m, np.inf)


def unproject(inv_pv, u, v, d):
    """scene.slang:189-193 in binary64"""
    m = np.asarray(inv_pv, f32).astype(f64).reshape(4, 4).T
    p = np.stack([u * 2.0 - 1.0, v * 2.0 - 1.0, d, np.ones_like(d)], -1) @ m.T
    with np.errstate(invalid="ignore", divide="ignore"):
        return p[:, :3] / p[:, 3:4]


def pcss(fr, ci, W, N, noise, mutation=0, analyse=False, force_branch=None, st=None):
    """:84-185.  Returns the shadow (binary32 values) and, when analysing, (hard ratio, PCF tap ratios, PCF valid counts)"""
    n = len(ci)
    L = fr.L
    nol = vmax(dot(N, L), 0.0)
    cts = 2.0 ** (ci + 1).astype(f64) * fr.texel_length
    b = SQRT2 * cts * 0.5
    branch = nol < 0.99 if force_branch is None else force_branch
    with np.errstate(invalid="ignore", divide="ignore"):
        term = np.where(branch, b * np.linalg.norm(np.cross(N, L), axis=-1) / vmax(nol, 0.1), b)
    base_bias = QUANTIZE + b + term
    inv_z = 1.0 / fr.z_length
    now = cts * (1.0 + 2.0 * (1.0 - nol))
    o = W + N * now[:, None]
    t, bt = basis(L, mutation)
    _, _, d_recv = clip_info(fr, ci, W if mutation == 8 else o)
    d_recv_w = d_recv * fr.z_length
    eps = EPS_UV if analyse else None
    centre, c_alts, c_rat = chain(fr, ci, o, mutation, eps, st)
    hb = inv_z * base_bias
    with np.errstate(invalid="ignore"):
        hard = np.where(centre == MISS, 1.0, np.where(centre + hb < d_recv, 0.0, 1.0))
    accum, blockers, valid = np.zeros(n), np.zeros(n, np.int64), np.zeros(n, np.int64)
    taps = []
    for i in range(BLOCKER_SAMPLES):
        hx, hy = hammersley(i, BLOCKER_SAMPLES, mutation)
        xi_x, xi_y = frac(hx + noise[:, 0]), frac(hy + noise[:, 1])
        r = np.sqrt(xi_x) * SEARCH_RADIUS
        th = xi_y * TAU
        off = r[:, None] * (t * np.cos(th)[:, None] + bt * np.sin(th)[:, None])
        pcf_bias = 2.0 * r
        lerp = nol * pcf_bias if mutation == 2 else pcf_bias + (0.0 - pcf_bias) * nol
        bn = inv_z * (base_bias + lerp)
        d, alts, rat = chain(fr, ci, o + off, mutation, eps, st)
        ok = d != MISS
        with np.errstate(invalid="ignore"):
            blk = ok & (d + bn < d_recv)
        valid += ok
        blockers += blk
        accum += np.where(blk, d * fr.z_length, 0.0)
        if analyse:
            taps.append((d, alts, rat, bn, np.abs(hx + noise[:, 0] - 1.0) / EPS_XI, ok, blk))

    def outcome(vld, blk_n):
        """0 / 1, 2 for the hard shadow, 3 for the PCF loop"""
        if mutation == 9:
            return np.where(vld == 0, 2, np.where(blk_n == 0, 2, np.where(blk_n == vld, 0, 3)))
        return np.where(vld == 0, 2, np.where(blk_n == 0, 1, np.where(blk_n == vld, 0, 3)))

    cls = outcome(valid, blockers)
    out = np.where(cls == 2, hard, np.where(cls == 1, 1.0, 0.0)).astype(f32)
    run = cls == 3
    with np.errstate(invalid="ignore", divide="ignore"):
        radius = vmin(MAX_PCF_RADIUS, (d_recv_w - accum / np.maximum(blockers, 1)) * LIGHT_WIDTH)
    r_hard = np.full(n, np.inf)
    spread = np.zeros(n)
    if analyse:
        # the blocker taps' candidate outcomes
        for d, alts, rat, bn, rx, ok, blk in taps:
            with np.errstate(invalid="ignore"):
                ok_a = alts != MISS
                blk_a = ok_a & (alts + bn[:, None] < d_recv[:, None])
                rc = np.where(ok, np.abs(d + bn - d_recv) / EPS_CMP, np.inf)
            rc = np.where(np.isnan(rc), np.inf, rc)
            cand = [(ok_a[:, k], blk_a[:, k], rat[:, k]) for k in range(alts.shape[1])] + [(ok, ok & ~blk, rc), (ok, blk, rx)]
            for ok_k, blk_k, r_k in cand:
                sel = r_k < 1.0
                if not sel.any():
                    continue
                c2 = outcome(valid + (ok_k.astype(np.int64) - ok), blockers + (blk_k.astype(np.int64) - blk))
                v2 = np.where(c2 == 2, hard, np.where(c2 == 1, 1.0, 0.0))
                changed = (c2 != cls) & ~((c2 != 3) & (cls != 3) & (v2 == out))
                changed |= (cls == 3) & ((ok_k != ok) | (blk_k != blk))
                changed |= rx == r_k  # the fract jump moves the tap by the whole radius
                r_hard = np.where(sel & changed, np.minimum(r_hard, r_k), r_hard)
            for k in range(alts.shape[1]):
                same = (rat[:, k] < 1.0) & blk & blk_a[:, k]
                spread += np.where(same, np.abs(alts[:, k] - d), 0.0)
        # the centre: the hard shadow's candidates
        with np.errstate(invalid="ignore"):
            rc = np.where(centre != MISS, np.abs(centre + hb - d_recv) / EPS_CMP, np.inf)
            hard_alt = np.where(c_alts == MISS, 1.0, np.where(c_alts + hb[:, None] < d_recv[:, None], 0.0, 1.0))
        rc = np.where(np.isnan(rc), np.inf, rc)
        r_centre = np.minimum(np.where(hard_alt != hard[:, None], c_rat, np.inf).min(1), rc)
    # PCF
    lit, vpcf = np.zeros(n), np.zeros(n, np.int64)
    pcf_rat = np.full((n, PCF_SAMPLES), np.inf)
    nz = noise if mutation == 1 else noise[:, ::-1]
    d_rad = LIGHT_WIDTH * spread * fr.z_length / np.maximum(blockers, 1) + 1e-6 * np.abs(radius)
    for i in range(PCF_SAMPLES):
        hx, hy = hammersley(i, PCF_SAMPLES, mutation)
        xi_x, xi_y = frac(hx + nz[:, 0]), frac(hy + nz[:, 1])
        r = np.sqrt(xi_x) * radius
        th = xi_y * TAU
        off = r[:, None] * (t * np.cos(th)[:, None] + bt * np.sin(th)[:, None])
        pcf_bias = 2.0 * r
        lerp = nol * pcf_bias if mutation == 2 else pcf_bias + (0.0 - pcf_bias) * nol
        bn = inv_z * (base_bias + lerp)
        rows = np.nonzero(run)[0]
        if not len(rows):
            break
        e_uv = (EPS_UV + d_rad[rows] * fr.uv_per_m[ci[rows]]) if analyse else None
        d, alts, rat = chain(fr, ci[rows], o[rows] + off[rows], mutation, e_uv, st)
        ok = d != MISS
        with np.errstate(invalid="ignore"):
            isl = ok & (d + bn[rows] >= d_recv[rows])
        vpcf[rows] += ok
        lit[rows] += isl
        if analyse:
            with np.errstate(invalid="ignore"):
                lit_a = (alts != MISS) & (alts + bn[rows, None] >= d_recv[rows, None])
                e_c = EPS_CMP + 2.0 * inv_z * d_rad[rows]
                rc = np.where(ok, np.abs(d + bn[rows] - d_recv[rows]) / e_c, np.inf)
            rc = np.where(np.isnan(rc), np.inf, rc)
            ra = np.where(((alts != MISS) != ok[:, None]) | (lit_a != isl[:, None]), rat, np.inf).min(1)
            rx = np.abs(hx + nz[rows, 0] - 1.0) / EPS_XI
            pcf_rat[rows, i] = np.minimum(np.minimum(ra, rc), rx)
    with np.errstate(invalid="ignore", divide="ignore"):
        frac_lit = (lit.astype(f32) / vpcf.astype(f32)).astype(f32)
    out = np.where(run, np.where(vpcf == 0, hard.astype(f32), frac_lit), out).astype(f32)
    if st is not None:
        st.add("valid_0", (cls == 2).sum())
        st.add("blockers_0", ((cls == 1) | ((mutation == 9) & (valid > 0) & (blockers == 0))).sum())
        st.add("blockers_eq_valid", ((cls == 0) & (valid > 0)).sum())
        st.add("pcf_ratio", (run & (vpcf > 0) & (out > 0) & (out < 1)).sum())
        st.add("bias_branch_lt", branch.sum())
        st.add("bias_branch_ge", (~branch).sum())
    if not analyse:
        return out
    uses_hard = (cls == 2) | (run & (vpcf == 0))
    r_hard = np.where(uses_hard, np.minimum(r_hard, r_centre), r_hard)
    return out, r_hard, np.where(run[:, None], pcf_rat, np.inf), vpcf


def restate(vsm, inv_pv, res, clipmaps, depth, normals, page_tables, atlas, mutation=0, pixels=None, analyse=True, st=None, ref_noise=None):
    """:187-209 over the given pixel indices (all by default): shadow, hard ratio, PCF tap ratios, PCF valid counts"""
    fr = Frame(vsm, clipmaps, page_tables, atlas)
    h, w = depth.shape
    pix = np.arange(h * w) if pixels is None else np.asarray(pixels)
    ys, xs = pix // w, pix % w
    d = depth.reshape(-1)[pix].astype(f64)
    out = np.ones(len(pix), f32)
    r_hard = np.full(len(pix), np.inf)
    pcf_rat = np.full((len(pix), PCF_SAMPLES), np.inf)
    vpcf = np.zeros(len(pix), np.int64)
    live = np.nonzero(d != 0.0)[0]
    if st is not None:
        st.add("sky", len(pix) - len(live))
        st.add("basis_plus_y" if abs(fr.L[1]) < f64(f32(0.999)) else "basis_plus_x", len(live))
    if not len(live):
        return out, r_hard, pcf_rat, vpcf
    nrm = normals.reshape(-1, 4)[pix[live]]
    N = normalize(oct_to_vec3(round_half(nrm[:, 2:4])))
    px, py = xs[live].astype(f64) + 0.5, ys[live].astype(f64) + 0.5
    u, v = px / w, py / h
    W = unproject(inv_pv, u, v, d[live])
    ci, m_level = select_clipmap(fr, inv_pv, res, u, v, d[live], mutation)
    noise = hash2(px, py)
    if not analyse:
        out[live] = pcss(fr, ci, W, N, noise, mutation, st=st)
        return out
    o, rh, pr, vp = pcss(fr, ci, W, N, noise, mutation, analyse=True, st=st)
    # the clipmap selection and the bias branch: the pixel again on the other side
    nol = vmax(dot(N, fr.L), 0.0)
    for ratios, alts in ((m_level / EPS_LEVEL, ("ci", -1, 1)), (np.abs(nol - 0.99) / EPS_NOL, ("branch",))):
        near = np.nonzero(ratios < 1.0)[0]
        if not len(near):
            continue
        if alts[0] == "ci":
            outs = [pcss(fr, np.clip(ci[near] + k, 0, fr.count - 1), W[near], N[near], noise[near], mutation) for k in alts[1:]]
        else:
            outs = [pcss(fr, ci[near], W[near], N[near], noise[near], mutation, force_branch=~(nol[near] < 0.99))]
        diff = np.zeros(len(near), bool)
        for a in outs:
            diff |= a.view(np.uint32) != o[near].view(np.uint32)
        rh[near] = np.where(diff, np.minimum(rh[near], ratios[near]), rh[near])
    if ref_noise is not None:
        rh = np.where(np.any(ref_noise[pix[live]] != noise.astype(f32), axis=1), 0.0, rh)
    out[live], r_hard[live], pcf_rat[live], vpcf[live] = o, rh, pr, vp
    return out, r_hard, pcf_rat, vpcf


def oracle_noise(vr, h, w, pixels=None):
    """the oracle's hash2 per pixel (of the given pixel indices; the others hold 0): only to find the pixels whose noise the
    restatement does not reproduce"""
    out = np.zeros((h * w, 2), f32)
    for k in range(h * w) if pixels is None else pixels:
        out[k] = vr.hash2(k % w + 0.5, k // w + 0.5)
    return out


def classify(r_hard, pcf_rat, vpcf, scale):
    """(ambiguous, bounded, bound) at an epsilon scale"""
    k = (pcf_rat < scale).sum(1)
    full = r_hard < scale
    bounded = ~full & (k > 0)
    return full | bounded, bounded, k / np.maximum(vpcf - k, 1)


def compare(want, res, live, label, ambiguous_bound):
    """asserts the rules of the module docstring; returns (ambiguous fraction, disagreeing pixels)"""
    got, r_hard, pcf_rat, vpcf = res
    want = want.reshape(-1)
    diff = got.view(np.uint32) != want.view(np.uint32)
    amb, bounded, bound = classify(r_hard, pcf_rat, vpcf, 1.0)
    amb_q, bounded_q, bound_q = classify(r_hard, pcf_rat, vpcf, MARGIN)
    delta = np.abs(got.astype(f64) - want.astype(f64))
    bad = diff & ~amb
    over = bounded & ~(r_hard < 1.0) & (delta > bound + 1e-7)
    bad_q = diff & ~(amb_q & ~(bounded_q & (delta > bound_q + 1e-7)))
    worst = np.minimum(r_hard, pcf_rat.min(1))[diff].max() if diff.any() else 0.0
    frac_amb = amb[live].mean() if live.any() else 0.0
    print(f"{label}: pixels {int(live.sum())}, ambiguous {frac_amb:.4f}, disagree {int(diff.sum())}, bounded {int(bounded.sum())}, worst ratio {worst:.3g}")
    assert not bad.any(), f"{label}: {int(bad.sum())} unambiguous pixels differ, e.g. {np.nonzero(bad)[0][:8]}"
    assert not over.any(), f"{label}: {int(over.sum())} PCF-bounded pixels beyond their bound"
    assert not bad_q.any(), f"{label}: {int(bad_q.sum())} disagreeing pixels are not ambiguous at {MARGIN} x epsilon"
    assert frac_amb <= ambiguous_bound, (label, frac_amb)
    return frac_amb, int(diff.sum())


def mutation_flips(want, res):
    """pixels that disagree with the oracle and are unambiguous (at 1 x epsilon)"""
    got, r_hard, pcf_rat, vpcf = res
    diff = got.view(np.uint32) != want.reshape(-1).view(np.uint32)
    amb, bounded, bound = classify(r_hard, pcf_rat, vpcf, 1.0)
    delta = np.abs(got.astype(f64) - want.reshape(-1).astype(f64))
    return int((diff & (~amb | (bounded & (delta > bound + 1e-7)))).sum())


# -- analytic geometry -------------------------------------------------------------------------------------------------------------
def quads():
    """ground, floating squares, a box and a tilted plane; every coordinate is a binary16 value, so the meshes' dequantised positions
    are these exactly"""
    def rect_y(x0, x1, z0, z1, y):
        return [(x0, y, z0), (x1, y, z0), (x1, y, z1), (x0, y, z1)]

    q = [rect_y(-96.0, 96.0, -160.0, 32.0, 0.0), rect_y(-4.0, 4.0, -32.0, -24.0, 5.0), rect_y(6.0, 10.0, -20.0, -16.0, 2.5),
         rect_y(-20.0, -16.0, -12.0, -8.0, 1.5)]
    x0, x1, y0, y1, z0, z1 = -12.0, -6.0, 0.0, 4.0, -40.0, -34.0
    q += [rect_y(x0, x1, z0, z1, y1),
          [(x0, y0, z1), (x1, y0, z1), (x1, y1, z1), (x0, y1, z1)], [(x0, y0, z0), (x1, y0, z0), (x1, y1, z0), (x0, y1, z0)],
          [(x0, y0, z0), (x0, y0, z1), (x0, y1, z1), (x0, y1, z0)], [(x1, y0, z0), (x1, y0, z1), (x1, y1, z1), (x1, y1, z0)]]
    q += [[(14.0, 0.5, -40.0), (22.0, 0.5, -40.0), (22.0, 6.5, -46.0), (14.0, 6.5, -46.0)]]
    # a high caster, whose penumbra is PCF_RADIUS-wide under a low sun, and a strip just above the ground near the camera,
    # (1/128 m wide) whose shadow can hold a tap's centre while every search tap misses it
    q += [rect_y(24.0, 40.0, -8.0, 8.0, 16.0), rect_y(0.5, 0.5078125, -14.0, -6.0, 0.5)]
    return [np.asarray(x, f64) for x in q]


def triangles(qs):
    return np.concatenate([np.stack([q[[0, 1, 2]], q[[0, 2, 3]]]) for q in qs])


def raycast(tris, origin, dirs):
    """nearest hit (t, face normal) of rays origin + t * dirs, binary64"""
    n = len(dirs)
    best, nrm = np.full(n, np.inf), np.zeros((n, 3))
    for a, b, c in tris:
        e1, e2 = b - a, c - a
        p = np.cross(dirs, e2)
        det = p @ e1
        with np.errstate(invalid="ignore", divide="ignore"):
            inv = 1.0 / det
            s = origin - a
            uu = dot(p, s) * inv
            q = np.cross(s, e1)
            vv = dot(dirs, q) * inv
            t = (q @ e2) * inv
        hit = (np.abs(det) > 1e-12) & (uu >= 0) & (vv >= 0) & (uu + vv <= 1) & (t > 1e-9) & (t < best)
        best = np.where(hit, t, best)
        fn = np.cross(e1, e2)
        nrm[hit] = fn / np.linalg.norm(fn)
    return best, nrm


def oct_encode(n):
    p = n[:, :2] / np.abs(n).sum(1, keepdims=True)
    sgn = np.where(p >= 0, 1.0, -1.0)
    return np.where(n[:, 2:3] <= 0, (1 - np.abs(p[:, ::-1])) * sgn, p)


def camera(w, h, eye=(0.0, 14.0, 6.0), target=(0.0, 0.0, -30.0), fov=60.0):
    pv = synth.mat_mul_cm(synth.perspective_reverse_z(fov, w / h, 0.1, 1000.0), synth.look_at(eye, target, (0.0, 1.0, 0.0)))
    cam = np.zeros(1, dtype=abi.CULL_CAMERA_DT)
    cam["projection_view"][0], cam["position"][0], cam["resolution"][0] = pv, eye, (w, h)
    return cam


def inverse_pv(cam):
    return np.linalg.inv(cam["projection_view"][0].reshape(4, 4).T.astype(f64)).T.astype(f32).reshape(16)


def cast_frame(tris, cam, w, h):
    """depth (binary32 of the binary64 hit's NDC z, 0 for sky) and normals (oct of the camera-facing face normal in .zw)"""
    pv = cam["projection_view"][0].reshape(4, 4).T.astype(f64)
    ipv = np.linalg.inv(pv)
    ys, xs = np.mgrid[0:h, 0:w]
    ndc = np.stack([(xs.reshape(-1) + 0.5) / w * 2 - 1, (ys.reshape(-1) + 0.5) / h * 2 - 1], 1)

    def at(z):
        p = np.concatenate([ndc, np.full((len(ndc), 1), z), np.ones((len(ndc), 1))], 1) @ ipv.T
        return p[:, :3] / p[:, 3:4]

    eye = np.asarray(cam["position"][0], f64)
    dirs = at(0.5) - at(1.0)
    t, nrm = raycast(tris, at(1.0), dirs)
    hit = np.isfinite(t)
    X = at(1.0) + t[:, None] * dirs
    c = np.concatenate([X, np.ones((len(X), 1))], 1) @ pv.T
    depth = np.where(hit, c[:, 2] / c[:, 3], 0.0).astype(f32)
    nrm = np.where((dot(nrm, eye - X) < 0)[:, None], -nrm, nrm)
    normals = np.zeros((h * w, 4), f32)
    normals[hit, 2:] = oct_encode(nrm[hit])
    return depth.reshape(h, w), normals.reshape(h, w, 4)


def vsm_ctx(shape, count, bias, light, w, h):
    size, ps, P = (64, 128, 8192) if shape == "reference" else (24, 64, 2048)
    vsm = np.zeros(1, dtype=abi.VSM_CONTEXT_DT)
    vsm["page_size"], vsm["page_table_size"], vsm["physical_page_table_size"], vsm["clipmap_count"] = ps, size, P, count
    vsm["depth_extent"][0] = (w, h)
    vsm["first_clipmap_width"], vsm["clipmap_selection_bias"], vsm["virtual_extent"], vsm["z_length"] = 10.0, bias, float(P), 2000.0
    vsm["directional_light_dir"][0] = light
    return vsm


def cast_atlas_pages(tris, vsm, clipmaps, pt, P, entries=None, sub=1):
    """the expected atlas of every Backed entry (or of the given (clipmap, wrapped y, wrapped x) entries), inverse-mapped: physical
    address -> owning clipmap and wrapped page (unique) -> virtual page (unwrapped by page_offset) -> the virtual texels whose centre
    the draw maps to each physical texel -> clip-space sample -> the nearest caster along the light, binary64.  For the orthographic
    clipmaps the world ray along the light through the sample is the clip-space line of constant (x, y), so the triangles are taken
    to clip space once and intersected there.  sub > 1 casts every sub-th virtual texel per axis only; the other texels of the
    expected page are inf (not checked).  Returns {address: (expected ps x ps, edge-excluded mask, tolerance, clipmap)}."""
    v = vsm.reshape(-1)[0]
    size, ps = int(v["page_table_size"]), int(v["page_size"])
    npp = P // ps
    backed = np.argwhere((pt & B) != 0) if entries is None else np.asarray(entries)
    addrs = (pt[tuple(backed.T)] >> 16).astype(np.int64)
    keep = addrs < npp * npp
    backed, addrs = backed[keep], addrs[keep]
    assert len(np.unique(addrs)) == len(addrs), "a physical address is owned by two entries"
    t = np.arange(P)
    page_of = np.floor((t + 0.5) * size / P).astype(np.int64)
    result = {}
    clip_tris = {}
    for (c, wy, wx), addr in zip(backed, addrs):
        if c not in clip_tris:
            m = np.asarray(clipmaps["projection_view_mat"][c], f64).reshape(4, 4).T
            assert np.all(m[3] == (0, 0, 0, 1))
            hp = np.concatenate([tris, np.ones(tris.shape[:2] + (1,))], 2) @ m.T
            clip_tris[c] = hp[..., :3]
        ct = clip_tris[c]
        off = clipmaps["page_offset"][c]
        vx, vy = (wx - int(off[0])) % size, (wy - int(off[1])) % size
        px, py = t[page_of == vx][::sub], t[page_of == vy][::sub]
        X, Y = np.meshgrid((px + 0.5) / P * 2 - 1, (py + 0.5) / P * 2 - 1)
        grad = np.zeros(X.shape)
        zs = []
        for dx, dy in ((0, 0), (EPS_EDGE, 0), (-EPS_EDGE, 0), (0, EPS_EDGE), (0, -EPS_EDGE)):
            z, g = _cast_points(ct, X + dx * 2.0 / P, Y + dy * 2.0 / P, P)
            zs.append(z)
            if dx == 0 and dy == 0:
                grad = g
        z0 = zs[0]
        tol = grad * np.sqrt(2.0) / 256.0 + 4 * 2.0 ** -24
        edge = np.zeros(z0.shape, bool)
        for z in zs[1:]:  # off the plane of the sample's own caster: a silhouette within EPS_EDGE
            edge |= np.abs(z - z0) > 2.0 * grad * EPS_EDGE + tol
        exp, ex = np.full((ps, ps), np.inf), np.zeros((ps, ps), bool)
        iy, ix = np.meshgrid(py % ps, px % ps, indexing="ij")
        np.minimum.at(exp, (iy, ix), z0)
        np.logical_or.at(ex, (iy, ix), edge)
        tl = np.zeros((ps, ps))
        np.maximum.at(tl, (iy, ix), tol)
        result[int(addr)] = (exp, ex, tl, int(c))
    return result


def _cast_points(ct, X, Y, P):
    """nearest NDC z in [0, 1] of the clip-space triangles at the samples (1.0 where none), and |grad z| per pixel there"""
    best, grad = np.ones(X.shape), np.zeros(X.shape)
    x0, x1, y0, y1 = X.min(), X.max(), Y.min(), Y.max()
    for a, b, c in ct:
        if max(a[0], b[0], c[0]) < x0 or min(a[0], b[0], c[0]) > x1 or max(a[1], b[1], c[1]) < y0 or min(a[1], b[1], c[1]) > y1:
            continue
        det = (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])
        if det == 0:
            continue
        l1 = ((X - a[0]) * (c[1] - a[1]) - (Y - a[1]) * (c[0] - a[0])) / det
        l2 = ((b[0] - a[0]) * (Y - a[1]) - (b[1] - a[1]) * (X - a[0])) / det
        inside = (l1 >= 0) & (l2 >= 0) & (l1 + l2 <= 1)
        z = a[2] + l1 * (b[2] - a[2]) + l2 * (c[2] - a[2])
        ok = inside & (z >= 0) & (z <= 1) & (z < best)
        dzdx = ((b[2] - a[2]) * (c[1] - a[1]) - (c[2] - a[2]) * (b[1] - a[1])) / det
        dzdy = ((c[2] - a[2]) * (b[0] - a[0]) - (b[2] - a[2]) * (c[0] - a[0])) / det
        best = np.where(ok, z, best)
        grad = np.where(ok, np.hypot(dzdx, dzdy) * 2.0 / P, grad)
    return best, grad


def analytic_case(shape, light, bias, count, w, h, seed, unbacked=True, view=None):
    """a cast frame, clipmaps from synth.make_vsm_clipmaps, a page table over the pages the frame's taps can reach (80 % Backed on
    shuffled addresses, some beyond the atlas, one clipmap entirely unbacked), and the cast atlas"""
    rng = np.random.default_rng(seed)
    L = np.asarray(light, f64)
    tris = triangles(quads())
    cam = camera(w, h) if view is None else camera(w, h, *view)
    depth, normals = cast_frame(tris, cam, w, h)
    cam["resolution"][0] = RESOLUTION  # the clipmap selection sees a full-size camera's pixel footprint
    inv_pv, res = inverse_pv(cam), cam["resolution"][0]
    vsm = vsm_ctx(shape, count, bias, L.astype(f32), w, h)
    v = vsm[0]
    size, ps, P = int(v["page_table_size"]), int(v["page_size"]), int(v["physical_page_table_size"])
    cm = synth.make_vsm_clipmaps(L, cam["position"][0], count=count, page_table_size=size)
    # the entries the taps can reach: clipmaps ci - 1 .. ci + 1 around each world point, out to the normal offset and the radius
    fr = Frame(vsm, cm, np.zeros((count, size, size), np.uint32), np.zeros((1, 1)))
    live = np.nonzero(depth.reshape(-1) != 0)[0]
    u, vv = (live % w + 0.5) / w, (live // w + 0.5) / h
    dl = depth.reshape(-1)[live].astype(f64)
    W = unproject(inv_pv, u, vv, dl)
    ci, _ = select_clipmap(fr, inv_pv, res, u, vv, dl)
    touched = np.zeros((count, size, size), bool)
    for dc in (-1, 0, 1):
        c = ci + dc
        ok = (c >= 0) & (c < count)
        cu, cv, _ = clip_info(fr, c[ok], W[ok])
        reach = (0.12 + 3.0 * 2.0 ** (ci[ok] + 1) * fr.texel_length) * fr.uv_per_m[c[ok]]
        for su in (-1, 0, 1):
            for sv in (-1, 0, 1):
                x = np.floor((cu + su * reach) * size).astype(np.int64)
                y = np.floor((cv + sv * reach) * size).astype(np.int64)
                g = (x >= 0) & (y >= 0) & (x < size) & (y < size)
                cc = c[ok][g]
                touched[cc, (y[g] + fr.off[cc, 1]) % size, (x[g] + fr.off[cc, 0]) % size] = True
    if unbacked and count > 1:
        touched[np.bincount(ci, minlength=count).argmax()] = False
    ent = np.argwhere(touched)
    backed = ent[rng.random(len(ent)) < (0.8 if unbacked else 2.0)]
    npp = (P // ps) ** 2
    assert len(backed) <= npp, (len(backed), npp)
    addr = rng.permutation(npp)[: len(backed)].astype(np.uint32)
    beyond = rng.random(len(backed)) < (0.02 if unbacked else 0.0)
    addr[beyond] = npp + rng.integers(0, 65536 - npp, int(beyond.sum()))
    pt = (rng.integers(0, 4, size=(count, size, size)).astype(np.uint32) & (V | D)) | (rng.integers(0, 65536, size=(count, size, size)).astype(np.uint32) << 16)
    pt[tuple(backed.T)] = B | D | (addr << 16)
    atlas = np.ones((P, P), f32)
    for a, (exp, _, _, _) in cast_atlas_pages(tris, vsm, cm, pt, P).items():
        atlas[(a // (P // ps)) * ps:(a // (P // ps) + 1) * ps, (a % (P // ps)) * ps:(a % (P // ps) + 1) * ps] = exp.astype(f32)
    return dict(vsm=vsm, inv_pv=inv_pv, res=res, cm=cm, depth=depth, normals=normals, pt=pt, atlas=atlas, tris=tris)


def unit_sun(elevation_deg, azimuth_deg=35.0):
    e, a = np.radians(elevation_deg), np.radians(azimuth_deg)
    return np.array([np.cos(e) * np.cos(a), np.sin(e), np.cos(e) * np.sin(a)])


# directional_light_dir points towards the light (its y > 0 for a sun above the horizon)
SUNS = {"sun20": unit_sun(20.0), "sun45": unit_sun(45.0), "sun80": unit_sun(80.0), "zenith": unit_sun(88.5, 10.0),
        "unnormalised": np.array([0.3, -1.0, 0.2])}
# (sun, bias, clipmap count) per analytic scene: every sun, every bias and every count at least once per atlas shape
ANALYTIC = [("sun20", 0.25, 10), ("sun45", -1.0, 4), ("sun80", 2.0, 10), ("zenith", 0.0, 10), ("unnormalised", 0.25, 1), ("sun45", 0.0, 10)]
FRAME = {"reference": (96, 54), "uneven": (128, 72)}
RESOLUTION = (1920.0, 1080.0)


@pytest.fixture(scope="module")
def vr():
    import pyoracle_vsm_resolve

    pyoracle_vsm_resolve.build()
    return pyoracle_vsm_resolve


@pytest.fixture(scope="module")
def vd():
    import pyoracle_vsm_draw

    pyoracle_vsm_draw.build()
    return pyoracle_vsm_draw


def oracle(vr, c):
    return vr.vsm_resolve_shadows(c["vsm"], c["inv_pv"], c["res"], c["cm"], c["depth"], c["normals"], c["pt"], c["atlas"])


def run_case(vr, c, label, bound, mutations=False, pixels=None):
    h, w = c["depth"].shape
    want, _ = oracle(vr, c)
    ref_noise = oracle_noise(vr, h, w)
    st = Stats()
    args = (c["vsm"], c["inv_pv"], c["res"], c["cm"], c["depth"], c["normals"], c["pt"], c["atlas"])
    res = restate(*args, st=st, ref_noise=ref_noise)
    live = c["depth"].reshape(-1) != 0
    frac_amb, ndiff = compare(want, res, live, label, bound)
    noise_mismatch = int(np.any(ref_noise[live] != hash2((np.nonzero(live)[0] % w) + 0.5, (np.nonzero(live)[0] // w) + 0.5).astype(f32), 1).sum())
    print(f"  noise mismatches {noise_mismatch}; coverage {st.c}")
    flips = {}
    if mutations:
        for m in MUTATIONS:
            flips[m] = mutation_flips(want, restate(*args, mutation=m, ref_noise=ref_noise))
        print("  mutations: " + ", ".join(f"{m} {flips[m]}" for m in MUTATIONS))
    return st.c, flips


COVERAGE_MIN = {"sky": 100, "valid_0": 20, "blockers_0": 1000, "blockers_eq_valid": 200, "pcf_ratio": 30, "fallback_minus_hit": 100,
                "fallback_plus_hit": 100, "basis_plus_y": 1000, "basis_plus_x": 1000, "bias_branch_lt": 1000, "bias_branch_ge": 1000,
                "out_of_atlas_reads": 20}


@pytest.mark.parametrize("shape", ["reference", "uneven"])
def test_analytic_frames(vr, shape):
    """the cast frames under every sun, bias and clipmap count: the rules of the module docstring, the coverage of every branch
    over the family, and each mutation's unambiguous disagreements on at least one scene"""
    w, h = FRAME[shape]
    total, best = Stats(), {m: 0 for m in MUTATIONS}
    for k, (sun, bias, count) in enumerate(ANALYTIC):
        c = analytic_case(shape, SUNS[sun], bias, count, w, h, seed=100 + k)
        cov, flips = run_case(vr, c, f"{shape} {sun} bias {bias} clipmaps {count}", AMBIGUOUS_ANALYTIC, mutations=True)
        for kk, n in cov.items():
            total.add(kk, n)
        for m, n in flips.items():
            best[m] = max(best[m], n)
    print(f"{shape} coverage {total.c}; mutation best {best}")
    for kk, n in COVERAGE_MIN.items():
        assert total.c.get(kk, 0) >= n, (kk, total.c.get(kk, 0))
    for m in EXPOSED[f"analytic {shape}"]:
        n = best[m]
        assert n >= MUTATION_MIN, f"mutation {m} ({MUTATIONS[m]}) flips only {n} unambiguous pixels"


# close-up views (sun, eye, target, vertical fov): the high caster's penumbra under the 20-degree sun, where the PCF radius reaches
# MAX_PCF_RADIUS over ground at NoL = 0.34, and the strip's shadow under the 88.5-degree sun, where the ground does not shadow its own
# search taps and the strip is narrower than their ring
CLOSE_UPS = {"penumbra": ("sun20", (4.0, 3.0, -16.0), (4.0, 0.0, -24.0), 30.0), "strip": ("zenith", (-1.0, 1.5, -4.0), (0.5, 0.0, -10.0), 8.0)}


@pytest.mark.parametrize("view", list(CLOSE_UPS))
def test_close_ups(vr, view):
    """every entry the taps reach is Backed, on fine clipmaps: the bias term of the PCF taps (mutation 2) decides comparisons in the
    high caster's wide penumbra, and in the strip's shadow the centre lookup is shadowed while no search tap is (mutation 9)"""
    sun, *camera_view = CLOSE_UPS[view]
    c = analytic_case("reference", SUNS[sun], 0.25, 10, 192, 108, seed=300, unbacked=False, view=camera_view)
    _, flips = run_case(vr, c, f"close-up {view}", AMBIGUOUS_CLOSE_UP, mutations=True)
    for m in EXPOSED[f"close-up {view}"]:
        assert flips[m] >= MUTATION_MIN, f"mutation {m} ({MUTATIONS[m]}) flips only {flips[m]} unambiguous pixels"


@pytest.mark.parametrize("shape", ["reference", "uneven"])
def test_random_frames(vr, shape):
    """test_gpu_vsm_resolve.random_inputs (hostile values included) at a small extent, and the uneven shape's non-orthographic
    clipmaps"""
    from tests.test_gpu_vsm_pages import clipmaps, vsm_context
    from tests.test_gpu_vsm_resolve import random_inputs

    rng = np.random.default_rng(31 if shape == "reference" else 32)
    sc = synth.make_scene(500, config_index=2, width=160, height=90, n_unique_meshes=4)
    if shape == "reference":
        vsm = vsm_context(width=160, height=90)
        cm = clipmaps(10, rng, center=(6.0, -2.0, -115.0))
    else:
        vsm = vsm_context(size=24, page_size=64, physical=2048, width=160, height=90)
        cm = clipmaps(10, rng, center=(6.0, -2.0, -115.0))
        cm["projection_view_mat"][3][3] = f32(1.0001)
        cm["projection_view_mat"][5][7] = f32(1e-4)
    cam, depth, normals, pt, atlas = random_inputs(rng, sc, vsm)
    from tests.test_gpu_vsm_resolve import inverse_pv as ipv_of

    c = dict(vsm=vsm, inv_pv=ipv_of(cam), res=cam["resolution"][0], cm=cm, depth=depth, normals=normals, pt=pt, atlas=atlas)
    cov, flips = run_case(vr, c, f"random {shape}", AMBIGUOUS_RANDOM, mutations=True)
    for m in EXPOSED[f"random {shape}"]:
        assert flips[m] >= MUTATION_MIN, f"mutation {m} ({MUTATIONS[m]}) flips only {flips[m]} unambiguous pixels"
    assert cov.get("pcf_ratio", 0) >= 100 and cov.get("valid_0", 0) >= 10 and cov.get("out_of_atlas_reads", 0) >= 10
    if shape == "uneven":
        assert cov.get("non_ortho_reads", 0) >= 100


# -- part 2: the oracle's draw against the cast ------------------------------------------------------------------------------------
def draw_scene(qs):
    """one mesh, one meshlet holding every quad in both windings (the coarse camera keeps one of each pair), identity transform"""
    from tests.test_oracle_vsm_draw import quads_scene

    return quads_scene([q for q in qs] + [q[[0, 3, 2, 1]] for q in qs])


def coarse_all():
    cam = np.zeros(1, dtype=abi.CULL_CAMERA_DT)
    m = np.diag([1e-6, 1e-6, 0.0, 1.0]).astype(f32)
    m[2, 3] = 0.5
    cam["projection_view"][0] = m.T.reshape(16)
    cam["mesh_instance_count"] = 1
    return cam


def check_atlas(atlas, expected, P, ps, label):
    """every cast texel within its tolerance outside the silhouette band, and the band under EDGE_BOUND"""
    npp = P // ps
    n = n_edge = n_bad = 0
    worst = 0.0
    for a, (exp, edge, tol, _) in expected.items():
        got = atlas[(a // npp) * ps:(a // npp + 1) * ps, (a % npp) * ps:(a % npp + 1) * ps].astype(f64)
        cast = np.isfinite(exp)
        edge = edge | ~cast
        err = np.where(cast, np.abs(got - exp), 0.0)
        n += int(cast.sum())
        n_edge += int((edge & cast).sum())
        bad = ~edge & (err > tol)
        n_bad += int(bad.sum())
        if (~edge).any():
            worst = max(worst, float((err / tol)[~edge].max()))
        assert not bad.any(), f"{label}: page {a}: {int(bad.sum())} texels beyond tolerance, max {err[bad].max():.3g}"
    print(f"{label}: texels {n}, edge band {n_edge} ({n_edge / max(n, 1):.4f}), worst error / tolerance {worst:.3g}")
    assert n > 0 and n_edge <= EDGE_BOUND * n


@pytest.mark.parametrize("shape", ["reference", "uneven"])
def test_oracle_draw_equals_cast(orc, vd, shape):
    """orc_vsm_draw_pages of the analytic casters into every Backed, Dirty entry of the analytic page tables equals the inverse-mapped
    binary64 cast of the atlas: page mapping, wrap, address and y direction checked against the opposite direction"""
    w, h = FRAME[shape]
    for k, sun in enumerate(("sun20", "zenith")):
        c = analytic_case(shape, SUNS[sun], 0.25, 10, w, h, seed=200 + k)
        v = c["vsm"][0]
        P, ps = int(v["physical_page_table_size"]), int(v["page_size"])
        sc = draw_scene(quads())
        hs = orc.HostScene(sc)
        mi = np.zeros(1, dtype=abi.MESHLET_INSTANCE_DT)
        atlas = np.ones((P, P), f32)
        flags = [int(((c["pt"][l] & (B | D)) == (B | D)).any()) for l in range(len(c["cm"]))]
        vd.vsm_draw_pages(hs, mi, [0], coarse_all(), c["vsm"], c["cm"], flags, c["pt"], atlas)
        expected = cast_atlas_pages(c["tris"], c["vsm"], c["cm"], c["pt"], P)
        check_atlas(atlas, expected, P, ps, f"draw {shape} {sun}")
        # entries whose address lies beyond the atlas write nothing: every page no in-atlas entry owns still holds the clear value
        npp = P // ps
        beyond = int(((c["pt"] & B) != 0).sum()) - len(expected)
        owned = np.zeros((npp, npp), bool)
        owned.reshape(-1)[list(expected)] = True
        assert beyond > 0 and (atlas.reshape(npp, ps, npp, ps).transpose(0, 2, 1, 3)[~owned] == 1.0).all()


def test_device_source_on_unit_suns(vr, tmp_path):
    """csrc/oxc_vsm_resolve.cuh compiled for the host equals the oracle bit for bit on analytic frames under unit suns on both of
    perpendicular_basis's branches (+y at 20 and 80 degrees, +x at 88.5), NoL <= 1 throughout"""
    from tests.host_harness import compile_harness
    from tests.test_vsm_resolve_source_cpu import _run

    exe = compile_harness(tmp_path, "vsm_resolve_vs_oracle")
    for k, sun in enumerate(("sun20", "sun80", "zenith")):
        c = analytic_case("uneven", SUNS[sun], 0.25, 10, 160, 90, seed=400 + k)
        case = (sun, c["vsm"], c["inv_pv"], c["res"], c["cm"], c["depth"], c["normals"], c["pt"], c["atlas"])
        got, _ = _run(exe, tmp_path, case)
        want, pcf = oracle(vr, c)
        np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32), err_msg=sun)
        assert pcf.sum() > 10 and (want == 0).sum() > 100, sun
