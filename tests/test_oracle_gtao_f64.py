"""The GTAO oracle (oracle/oxc_oracle_gtao.c) against an independent binary64 restatement of the reference's three passes
(passes/gtao/vbgtao_prefilter.slang, vbgtao_main.slang, vbgtao_denoise.slang and common's oct_to_vec3), over ray-cast analytic scenes
and random frames, at every preset and at random settings, with known answers on a single plane.

The restatement is written from the shader text, vectorised over pixels, and evaluates in binary64 everything whose result depends
smoothly on its inputs: the linearization, the weighted average, the edges, sin / cos / log2 / pow, fast_acos's polynomial exactly as
the shader writes it (not acos: its error is the cause of the plane quirk below), the trilinear taps with the textbook weights (no
8-bit quantisation, the deviation DESIGN §4.7 commits to) and the bitmask accumulation.  It keeps binary32 only where the shader's
result depends chaotically on the last bits:
- the R2 noise frac(0.5 + index * c) (an index up to 22 239 times c keeps about 9 fractional bits in binary32);
- the per-sample R1 noise frac(noise.y + k * 0.618...);
- the binary16 store of the noisy plane;
- the round-to-nearest of packUnorm4x8;
- the normals' .zw, read from the reference's R16G16B16A16Sfloat normal attachment (RendererInstance.cpp:709-714), so
  rounded to binary16 before oct_to_vec3.

The shader text leaves NaN open; the restatement follows the GPU's arithmetic, as the oracle's specification (item 7) does: max and
min return the other operand for a NaN, so saturate(NaN) = 0, and sign(NaN) = 0.  A rendered frame needs it: the decode leaves NaN
normals on its ground, where n comes out 0 and the occlusion still counts.

Gather layout, worked out from GatherRed's definition (the 2 x 2 footprint of a bilinear fetch at uv, components x = (i0, j1),
y = (i1, j1), z = (i1, j0), w = (i0, j0), the offset added to the texel coordinates, point-clamp clamping each texel into the extent):
at the texel corner uv = p / size the footprint is {p - 1, p}, so with offset o the quad is {p - 1 + o, p + o} and x, y, z, w are
(p.x - 1 + o.x, p.y + o.y), (p.x + o.x, p.y + o.y), (p.x + o.x, p.y - 1 + o.y), (p.x - 1 + o.x, p.y - 1 + o.y).  That makes the
prefilter's Gather(2t, (1, 1)) the quad 2t .. 2t + 1 with w = 2t, z = 2t + (1, 0), x = 2t + (0, 1), y = 2t + (1, 1); the edges read
left, centre, top from offset 0 and bottom, right from (1, 1); the denoise reads the left, centre, top edges from offset 0, the right
from (2, 0).x, the bottom from (1, 2).w, and its nine visibilities from the x, y, z, w of offsets (0, 0), (2, 0), (0, 2), (2, 2).

Every thread of the prefilter's 8 x 8 groups runs, so a level k texel averages level k - 1 texels 2t .. 2t + 1 of a pyramid whose
level 0 continues past the extent by clamping; only the texels inside level k's extent max(1, size >> k) are stored.

Each noisy texel comes with a slack: how far the binary32 rounding of the oracle or the device can move it by flipping a discrete
decision.  A decision is near when the quantity it truncates or ceils lies within err sectors of a jump, with
err = DELTA + POLE_ERR [a cosine within POLE of +-1 went through fast_acos's square root] + TAP_ERR * (depth range of the tap's
texels * texels per uv unit) / |delta| (a tap across a depth step, where the binary32 uv moves the depth):
- the width * 32 of a sample's arc (ceil jumps at every integer; an arc whose two ends both clamp to one bound is an exact 0 until
  the nearer end crosses that bound, a negative one until it crosses 0);
- the start * 32 of a non-empty arc (the truncation jumps at 1..31; below 0 and at 32 the clamps hold it).
A near width toggles one end bit of the arc and a near start two; a toggled bit moves its slice's occlusion by at most 1 / 32 (it is
counted at some sample's falloff in [0, 1] or not at all), so the slack adds 1 / (32 * slice_count) per toggled bit.  The slack is
infinite where a linear depth lies within FAR_MARGIN (relative) of far_clip * 0.999, the sky test, or where the normal projected into
a slice is shorter than EPS, where its direction (and so n) is chaotic.  A pixel with a slack above 0 is ambiguous; a denoised pixel
takes the largest slack of its 3 x 3 neighbourhood.

The constants, chosen from the measured distribution over the cases below (oracle against restatement):
- DELTA = 1e-3 sectors, POLE = 1e-4, POLE_ERR = 0.02, TAP_ERR = 2e-6: on the 211 x 97 scenes at every preset, every noisy texel
  that disagrees by more than one binary16 ulp has a near decision at under 0.17 of its err, a margin of 6 (the worst pole cases sit
  2.7e-3 sectors from a jump).  At preset 3 they make 15 to 18 % of the pixels of those scenes ambiguous, 1.5 to 4 % at preset 0.
- FAR_MARGIN = 1e-5 relative, 100 times the binary32 rounding of the linearization; EPS = 1e-3: binary32 rounding moves a projected
  normal of that length by ~1e-4 rad.
- mips: 32 binary32 ulps relative.  The measured worst is 3.6 on the analytic scenes and 9.8 on the random frames, where a tap lies
  in the weighted average's linear falloff range and its weight (d - min) * mul + add cancels in binary32.
- edges: every byte within +-1 (binary32 moves a value across a rounding half only); the measured worst is 1, on the random frames
  and the ramp scene.
- noisy: within one binary16 ulp plus 1e-6 (the falloff's binary32 rounding, ~1e-7 per sample) plus the slack, on every pixel.
  Pixels that differ by more than one binary16 ulp (a decision really flipped) stay under FLIPPED_BOUND = 3 % of the pixels holding
  depth: the measured worst is 1.5 % on the camera-facing plane at 2 m and preset 3, whose tangent-plane horizons all sit next to the
  bottom sector's edge, and 0.6 % everywhere else.
- ambiguous pixels: under AMBIGUOUS_BOUND = 0.25 of the pixels holding depth on the 211 x 97 scenes at the presets (measured at most
  0.18); under AMBIGUOUS_BOUND_RANDOM = 0.7 on the random frames and on the scenes at random settings (measured at most 0.59 and
  0.42: the random frames' depth steps every few pixels put most taps across one, and random settings reach 15 x 8 samples); under
  AMBIGUOUS_BOUND_CROP = 0.9 on the 153-pixel 17 x 9 crops (measured at most 0.55 at the presets and 0.85 at 14 slices), which are
  there for the border clamp and the virtual pyramid.  The flipped bound above holds on all of them.
- ao: with a 3 x 3 slack of 0 within AO_TIGHT * max(1, final_power) = 1e-3 * max(1, p) (one binary16 ulp of a neighbour moves the
  blend by at most 2^-11 before the power; the measured worst is 2.4e-4); elsewhere within p * (slack + 2^-10), or
  (slack + 2^-10)^p for p < 1.  Over all pixels holding depth the mean |difference| stays under AO_MEAN = 1e-4 (measured at most
  4.7e-5): a systematic error (a mirrored sample, a lost nudge, a wrong mip) moves whole planes by 1e-2 and more.
"""
import math

import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_gtao import oct_encode, random_frame, random_settings

f32 = np.float32
f64 = np.float64

DELTA = 1e-3
POLE = 1e-4
POLE_ERR = 0.02
TAP_ERR = 2e-6
FAR_MARGIN = 1e-5
EPS = 1e-3
MIP_ULPS = 32
AMBIGUOUS_BOUND = 0.25
AMBIGUOUS_BOUND_RANDOM = 0.7
AMBIGUOUS_BOUND_CROP = 0.9
FLIPPED_BOUND = 0.03
UNBOUNDED_BOUND = 0.01
AO_TIGHT = 1e-3
AO_MEAN = 1e-4

HALF_PI = math.pi / 2
SECTORS = 32
LEVELS = 5


# -- vbgtao_prefilter.slang --------------------------------------------------------------------------------------------------------

def linearize(projection, device_depth):
    """linearize_depth with mul_add = (projection[3][2], projection[2][2]) of the column-major glm matrix (PBR.cpp:186)"""
    p = np.asarray(projection, f32).reshape(16).astype(f64)
    return p[14] / (np.asarray(device_depth, f32).astype(f64) + p[10])


def weighted_average(d0, d1, d2, d3):
    effect_radius = 0.75 * 0.5 * 1.457
    falloff_range = 0.615 * effect_radius
    falloff_from = effect_radius * (1.0 - 0.615)
    falloff_mul = -1.0 / falloff_range
    falloff_add = falloff_from / falloff_range + 1.0
    m = np.minimum(np.minimum(d0, d1), np.minimum(d2, d3))
    w = [np.clip((d - m) * falloff_mul + falloff_add, 0.0, 1.0) for d in (d0, d1, d2, d3)]
    return (w[0] * d0 + w[1] * d1 + w[2] * d2 + w[3] * d3) / (w[0] + w[1] + w[2] + w[3])


def depth_pyramid(projection, depth):
    """levels 0..4 as float64 arrays of their stored extents max(1, size >> k)"""
    h, w = depth.shape
    vw, vh = 16 * -(-w // 16), 16 * -(-h // 16)  # the texels the prefilter's threads cover
    lin = linearize(projection, depth)
    level = lin[np.minimum(np.arange(vh), h - 1)][:, np.minimum(np.arange(vw), w - 1)]
    out = [lin]
    for k in range(1, LEVELS):
        level = weighted_average(level[0::2, 0::2], level[0::2, 1::2], level[1::2, 0::2], level[1::2, 1::2])
        out.append(level[:max(1, h >> k), :max(1, w >> k)])
    return out


def pack_mips(levels):
    return np.concatenate([lv.reshape(-1) for lv in levels])


# -- vbgtao_main.slang ---------------------------------------------------------------------------------------------------------------

def sat(x):
    """saturate as the GPU evaluates it: max / min return the other operand for a NaN, so saturate(NaN) = 0"""
    return np.fmin(np.fmax(x, 0.0), 1.0)


def sign(x):
    """sign with sign(NaN) = 0, as (x > 0) - (x < 0)"""
    return np.where(x > 0, 1.0, np.where(x < 0, -1.0, 0.0))


def fast_acos(x):
    a = np.abs(x)
    res = (-0.156583 * a + HALF_PI) * np.sqrt(sat(1.0 - a))
    return np.where(x >= 0, res, math.pi - res)


def hilbert_table():
    """RendererInstance.cpp:151-177: the 64 x 64 table the main pass Loads, indexed [y, x]"""
    out = np.zeros((64, 64), np.int64)
    for y0 in range(64):
        for x0 in range(64):
            x, y, index, level = x0, y0, 0, 32
            while level > 0:
                rx, ry = int((x & level) > 0), int((y & level) > 0)
                index += level * level * ((3 * rx) ^ ry)
                if ry == 0:
                    if rx == 1:
                        x, y = 63 - x, 63 - y
                    x, y = y, x
                level //= 2
            out[y0, x0] = index
    return out


_HILBERT = hilbert_table()


def frac32(x):
    x = f32(x) if np.isscalar(x) else x.astype(f32)
    return (x - np.floor(x)).astype(f32)


def r2_noise(xs, ys, noise_index):
    """load_noise in binary32"""
    index = (_HILBERT[ys % 64, xs % 64] + 288 * (int(noise_index) % 64)).astype(f32)
    nx = frac32(f32(0.5) + index * f32(0.75487766624669276005))
    ny = frac32(f32(0.5) + index * f32(0.5698402909980532659114))
    return nx, ny


def oct_to_vec3(e):
    """common/encoding.slang oct_to_vec3 of [..., 2]"""
    x, y = e[..., 0].astype(f64), e[..., 1].astype(f64)
    z = 1.0 - np.abs(x) - np.abs(y)
    sx, sy = np.where(x >= 0.0, 1.0, -1.0), np.where(y >= 0.0, 1.0, -1.0)
    neg = z < 0.0
    x, y = np.where(neg, (1.0 - np.abs(y)) * sx, x), np.where(neg, (1.0 - np.abs(e[..., 0].astype(f64))) * sy, y)
    v = np.stack([x, y, z], -1)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def sample_level(levels, u, v, lam):
    """SampleLevel with a linear clamp sampler: trilinear, the textbook weights; also returns the depth range of the taps times the
    texels per uv unit, which scales how far binary32 rounding of uv moves the result"""
    lo = np.floor(lam).astype(np.int64)
    f = lam - lo
    hi = np.minimum(lo + 1, LEVELS - 1)
    out, spread = np.zeros_like(u), np.zeros_like(u)
    for k, lv in enumerate(levels):
        wk = np.where(lo == k, 1.0 - f, 0.0) + np.where(hi == k, f, 0.0)
        sel = wk != 0.0
        if not sel.any():
            continue
        lh, lw = lv.shape
        x, y = u[sel] * lw - 0.5, v[sel] * lh - 0.5
        x0, y0 = np.floor(x), np.floor(y)
        a, b = x - x0, y - y0
        x0, y0 = x0.astype(np.int64), y0.astype(np.int64)
        xa, xb = np.clip(x0, 0, lw - 1), np.clip(x0 + 1, 0, lw - 1)
        ya, yb = np.clip(y0, 0, lh - 1), np.clip(y0 + 1, 0, lh - 1)
        q = [lv[ya, xa], lv[ya, xb], lv[yb, xa], lv[yb, xb]]
        out[sel] += wk[sel] * ((1 - a) * (1 - b) * q[0] + a * (1 - b) * q[1] + (1 - a) * b * q[2] + a * b * q[3])
        spread[sel] = np.maximum(spread[sel], (np.maximum.reduce(q) - np.minimum.reduce(q)) * max(lw, lh))
    return out, spread


def _dist_to_int(q):
    return np.abs(q - np.rint(q))


def _sector_mask(thickness, delta, view_dir, direction_sign, n, n_pole):
    """calc_sector_mask and update_sectors over arrays; returns (mask, width margin, start margin, pole): each margin is the distance
    in sectors to the nearest jump of the ceil or the truncation that decides the mask (+inf where none can flip); pole is set where
    a cosine near +-1 went through fast_acos's square root"""
    back = delta - view_dir * thickness
    cos = [np.sum(d / np.linalg.norm(d, axis=-1, keepdims=True) * view_dir, -1) for d in (delta, back)]
    pole = n_pole | (1.0 - np.abs(cos[0]) < POLE) | (1.0 - np.abs(cos[1]) < POLE)
    fb = [(direction_sign * -fast_acos(c) + n + HALF_PI) / math.pi for c in cos]
    lo_raw, hi_raw = (fb[1], fb[0]) if direction_sign >= 0 else (fb[0], fb[1])
    lo, hi = sat(lo_raw), sat(hi_raw)
    width = sat(hi - lo) * SECTORS
    angle = np.ceil(width).astype(np.int64)
    start = np.minimum((lo * SECTORS).astype(np.int64), SECTORS - 1)
    bits = np.where(angle > 0, (np.uint64(0xFFFFFFFF) >> (SECTORS - np.maximum(angle, 1)).astype(np.uint64)), np.uint64(0))
    mask = ((bits << start.astype(np.uint64)) & np.uint64(0xFFFFFFFF)).astype(np.uint64)
    # width: where both ends clamp to the same bound it is an exact 0 until the nearer end crosses that bound; a negative width
    # saturates to 0 until it crosses 0; otherwise ceil jumps at every integer
    both_below, both_above = (lo_raw < 0) & (hi_raw < 0), (lo_raw > 1) & (hi_raw > 1)
    w_raw = (hi - lo) * SECTORS
    w_margin = np.where(both_below, np.abs(np.maximum(lo_raw, hi_raw)) * SECTORS,
                        np.where(both_above, np.abs(np.minimum(lo_raw, hi_raw) - 1.0) * SECTORS,
                                 np.where(w_raw <= 0, -w_raw, _dist_to_int(w_raw))))
    # start: the truncation jumps at 1..31 (below 0 and at 32 the clamps keep it constant); it only matters for a non-empty mask
    s_raw = lo_raw * SECTORS
    s_live = (s_raw > 0.5) & (s_raw < SECTORS - 0.5) & (w_raw > 0)
    s_margin = np.where(s_live, _dist_to_int(s_raw), np.inf)
    return mask, w_margin, s_margin, pole


def _popcount(x):
    x = x.astype(np.uint64)
    c = np.zeros(x.shape, np.int64)
    for i in range(SECTORS):
        c += ((x >> np.uint64(i)) & np.uint64(1)).astype(np.int64)
    return c


def _main_rows(camera, settings, levels, normals, y0, y1, nudge=0.99999):
    proj = np.asarray(camera["projection"], f32).astype(f64)
    view = np.asarray(camera["view"], f32).astype(f64).reshape(4, 4).T
    far = f64(f32(camera["far_clip"]))
    lin = levels[0]
    h, w = lin.shape
    ys, xs = np.meshgrid(np.arange(y0, y1), np.arange(w), indexing="ij")
    ys, xs = ys.reshape(-1), xs.reshape(-1)
    res = np.array([w, h], f64)
    uv = np.stack([(xs + 0.5) / w, (ys + 0.5) / h], -1)
    depth_center = lin[ys, xs]
    sky_limit = far * 0.999
    sky = depth_center >= sky_limit
    ambiguous = np.abs(depth_center - sky_limit) <= FAR_MARGIN * far
    margin = np.full(xs.shape, np.inf)

    thickness = f64(f32(settings.thickness))
    slice_count = int(settings.slice_count)
    samples = int(settings.samples_per_slice_side)
    effect_radius = f64(f32(settings.effect_radius)) * 1.457
    falloff_range = 0.615 * effect_radius
    falloff_from = effect_radius * (1.0 - 0.615)
    falloff_mul = -1.0 / falloff_range
    falloff_add = falloff_from / falloff_range + 1.0
    mip_sampling_offset = 3.30

    def view_position(p, d):
        ndc = p * 2.0 - 1.0
        return np.stack([ndc[:, 0] / proj[0], ndc[:, 1] / proj[5], -np.ones(len(d))], -1) * d[:, None]

    ld = depth_center * nudge
    origin = view_position(uv, ld)
    view_dir = -origin / np.linalg.norm(origin, axis=-1, keepdims=True)
    wn = oct_to_vec3(normals[ys, xs, 2:4].astype(np.float16))  # the R16G16B16A16Sfloat normal attachment
    vn = wn @ view[:3, :3].T
    normal = vn / np.linalg.norm(vn, axis=-1, keepdims=True)
    nx, ny = r2_noise(xs, ys, settings.noise_index)
    screen_radius_uv = 0.5 * effect_radius * np.stack([np.full_like(ld, abs(proj[0])), np.full_like(ld, abs(proj[5]))], -1) / ld[:, None]
    screen_radius_pixels = screen_radius_uv[:, 0] * w
    min_s = 1.3 / np.maximum(screen_radius_pixels, 1.3)

    visibility = np.zeros(len(xs))
    slack = np.zeros(len(xs))
    for slice_t in range(slice_count):
        phi = (slice_t + nx.astype(f64)) / slice_count * math.pi
        omega = np.stack([np.cos(phi), np.sin(phi)], -1)
        direction = np.concatenate([omega, np.zeros((len(xs), 1))], -1)
        ortho = direction - np.sum(direction * view_dir, -1, keepdims=True) * view_dir
        ortho /= np.linalg.norm(ortho, axis=-1, keepdims=True)
        axis = np.cross(direction, view_dir)
        axis /= np.linalg.norm(axis, axis=-1, keepdims=True)
        projected = normal - axis * np.sum(normal * axis, -1, keepdims=True)
        plen_raw = np.linalg.norm(projected, axis=-1)
        ambiguous |= plen_raw < EPS
        plen = np.fmax(plen_raw, 1e-6)
        sign_norm = sign(np.sum(ortho * projected, -1))
        cos_norm = sat(np.sum(projected * view_dir, -1) / plen)
        n = sign_norm * fast_acos(cos_norm)
        n_pole = 1.0 - cos_norm < POLE
        sample_mul = np.stack([omega[:, 0], -omega[:, 1]], -1) * screen_radius_uv

        bitmask = np.zeros(len(xs), np.uint64)
        occlusion = np.zeros(len(xs))
        for sample_t in range(samples):
            k = f32(slice_t + sample_t * samples)
            sample_noise = frac32(ny + k * f32(0.6180339887498948482)).astype(f64)
            s = (sample_t + sample_noise) / samples
            s = s * s + min_s
            offset = s[:, None] * sample_mul
            lam = np.clip(np.log2(np.linalg.norm(offset * res, axis=-1)) - mip_sampling_offset, 0.0, LEVELS - 1.0)
            for sgn in (1.0, -1.0):
                p = uv + sgn * offset
                d, spread = sample_level(levels, p[:, 0], p[:, 1], lam)
                delta = view_position(p, d) - origin
                mask, mw, ms, pole = _sector_mask(thickness, delta, view_dir, sgn, n, n_pole)
                err = DELTA + POLE_ERR * pole + TAP_ERR * spread / np.linalg.norm(delta, axis=-1)
                margin = np.minimum(margin, np.minimum(mw, ms) / err)
                # a flipped ceil toggles one end bit of the arc, a flipped truncation both: each toggled bit moves this slice's
                # occlusion by at most 1 / 32 (it is counted at some sample's falloff in [0, 1] or not at all)
                slack += ((mw < err) * 1.0 + (ms < err) * 2.0) / (SECTORS * slice_count)
                falloff = sat(np.linalg.norm(delta, axis=-1) * falloff_mul + falloff_add)
                occlusion += falloff * _popcount(mask & ~bitmask) / SECTORS
                bitmask |= mask
        visibility += sat(1.0 - occlusion)
    ao = sat(visibility / slice_count)
    ao = np.where(sky, 1.0, ao)
    # a sky test or a projected normal that rounding can flip bounds nothing; otherwise the flips' slack does
    slack = np.where(ambiguous, np.inf, np.where(sky, 0.0, slack))
    margin = np.where(sky, np.inf, margin)
    return ao.reshape(y1 - y0, w), slack.reshape(y1 - y0, w), margin.reshape(y1 - y0, w)


def edges_from(lin):
    """calculate_edges over level 0: packUnorm4x8(left, right, top, bottom) per pixel"""
    h, w = lin.shape
    pad = np.pad(lin, 1, mode="edge")
    c = lin
    e = [pad[1:-1, :-2] - c, pad[1:-1, 2:] - c, pad[:-2, 1:-1] - c, pad[2:, 1:-1] - c]
    slope_lr, slope_tb = (e[1] - e[0]) * 0.5, (e[3] - e[2]) * 0.5
    adj = [e[0] + slope_lr, e[1] - slope_lr, e[2] + slope_tb, e[3] - slope_tb]
    scale = c * 0.011
    packed = np.zeros((h, w), np.uint32)
    for i in range(4):
        v = np.clip(1.25 - np.minimum(np.abs(e[i]), np.abs(adj[i])) / scale, 0.0, 1.0).astype(f32)
        packed |= np.rint(v * f32(255.0)).astype(np.uint32) << np.uint32(8 * i)
    return packed


def _unorm(p, i):
    return ((p >> np.uint32(8 * i)) & np.uint32(0xFF)).astype(f64) / 255.0


def denoise(noisy, edges, final_power):
    """vbgtao_denoise.slang over the whole plane (noisy as float64 values of the binary16 texels)"""
    pn, pe = np.pad(noisy, 1, mode="edge"), np.pad(edges, 1, mode="edge")
    h, w = noisy.shape

    def at(a, dx, dy):
        return a[1 + dy:1 + dy + h, 1 + dx:1 + dx + w]

    ec, el, er, et, eb = at(pe, 0, 0), at(pe, -1, 0), at(pe, 1, 0), at(pe, 0, -1), at(pe, 0, 1)
    lw, rw = _unorm(ec, 0) * _unorm(el, 1), _unorm(ec, 1) * _unorm(er, 0)
    tw, bw = _unorm(ec, 2) * _unorm(et, 3), _unorm(ec, 3) * _unorm(eb, 2)
    tl = 0.425 * (tw * _unorm(et, 0) + lw * _unorm(el, 2))
    tr = 0.425 * (tw * _unorm(et, 1) + rw * _unorm(er, 2))
    bl = 0.425 * (bw * _unorm(eb, 0) + lw * _unorm(el, 3))
    br = 0.425 * (bw * _unorm(eb, 1) + rw * _unorm(er, 3))
    taps = [((0, 0), 1.2), ((-1, 0), lw), ((1, 0), rw), ((0, -1), tw), ((0, 1), bw), ((-1, -1), tl), ((1, -1), tr), ((-1, 1), bl),
            ((1, 1), br)]
    s = sum(at(pn, dx, dy) * wt for (dx, dy), wt in taps)
    sw = sum(wt for _, wt in taps)
    return np.power(np.fmax(s / sw, 0.0), f64(f32(final_power)))


def max3(a):
    """the largest value of each pixel's 3 x 3 neighbourhood (clamped at the borders, as the denoise reads it)"""
    p = np.pad(a, 1, mode="edge")
    h, w = a.shape
    out = np.full(a.shape, -np.inf)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            out = np.maximum(out, p[1 + dy:1 + dy + h, 1 + dx:1 + dx + w])
    return out


def restate(camera, settings, depth, normals, rows=64, nudge=0.99999):
    """the three passes in binary64 over depth [H, W] (D32F) and normals [H, W, 4]; camera is a dict(projection=, view=, far_clip=).
    Returns dict(levels= float64 per level, edges= uint32, noisy= float64 (binary16 values), slack= how far rounding flips can move
    each noisy value (0: none can, inf: unbounded), margin= the nearest flip in sectors, ao=, ao_slack= the largest slack of each 3 x 3
    neighbourhood)"""
    depth = np.asarray(depth, f32)
    normals = np.asarray(normals, f32)
    h, w = depth.shape
    levels = depth_pyramid(camera["projection"], depth)
    edges = edges_from(levels[0])
    noisy, slack, margin = np.zeros((h, w)), np.zeros((h, w)), np.zeros((h, w))
    for y0 in range(0, h, rows):
        y1 = min(h, y0 + rows)
        v, s, m = _main_rows(camera, settings, levels, normals, y0, y1, nudge)
        noisy[y0:y1], slack[y0:y1], margin[y0:y1] = v.astype(np.float16).astype(f64), s, m
    ao = denoise(noisy, edges, settings.final_power)
    return dict(levels=levels, edges=edges, noisy=noisy, slack=slack, margin=margin, ao=ao, ao_slack=max3(slack))


def camera_dict(proj, view, far_clip=1000.0):
    return dict(projection=np.asarray(proj, f32).reshape(16), view=np.asarray(view, f32).reshape(16), far_clip=f32(far_clip))


# -- comparison ----------------------------------------------------------------------------------------------------------------------

def compare(got, want, settings, depth, label="", ambiguous_bound=AMBIGUOUS_BOUND):
    """asserts the rules of the module docstring for the planes `got` holds (mips, edges, noisy, ao: the oracle's or the device's
    layout); returns the measured statistics"""
    stats = {}
    held = np.isfinite(depth) & (want["levels"][0] < f64(1000.0) * 0.999)
    if "mips" in got:
        ref = pack_mips(want["levels"])
        ulps = np.abs(got["mips"].astype(f64) - ref) / np.spacing(np.abs(ref).astype(f32)).astype(f64)
        stats["mips_ulps"] = float(ulps.max())
        assert ulps.max() <= MIP_ULPS, f"{label} mips: {ulps.max():.1f} ulps at {int(np.argmax(ulps))}"
    if "edges" in got:
        db = max(int(np.abs(((got["edges"] >> np.uint32(8 * i)) & 0xFF).astype(np.int64)
                            - ((want["edges"] >> np.uint32(8 * i)) & 0xFF).astype(np.int64)).max()) for i in range(4))
        stats["edges_bytes"] = db
        assert db <= 1, f"{label} edges: a byte differs by {db}"
    slack = want["slack"]
    amb = slack > 0
    stats["ambiguous"] = float(amb[held].mean()) if held.any() else 0.0
    stats["unbounded"] = float(np.isinf(slack)[held].mean()) if held.any() else 0.0
    assert stats["ambiguous"] <= ambiguous_bound, f"{label}: {stats['ambiguous']:.4f} of the pixels are ambiguous"
    assert stats["unbounded"] <= UNBOUNDED_BOUND, f"{label}: {stats['unbounded']:.4f} of the pixels are unbounded"
    if "noisy" in got:
        o = got["noisy"].view(np.float16).astype(f64)
        r = want["noisy"]
        diff = np.abs(o - r)
        tol = np.spacing(np.minimum(o, r).astype(np.float16)).astype(f64) + 1e-6
        bad = np.argwhere(diff > tol + slack)
        stats["noisy_max"] = float(diff[~amb].max()) if (~amb).any() else 0.0
        stats["noisy_max_ambiguous"] = float(diff[amb & np.isfinite(slack)].max()) if (amb & np.isfinite(slack)).any() else 0.0
        stats["flipped"] = float(((diff > tol) & held).sum() / max(held.sum(), 1))
        assert bad.size == 0, f"{label} noisy: {len(bad)} pixels differ, first at {bad[:3].tolist()}: {o[tuple(bad[0])]} vs {r[tuple(bad[0])]}"
        assert stats["flipped"] <= FLIPPED_BOUND, f"{label} noisy: {stats['flipped']:.4f} of the pixels differ by a flipped decision"
    a, r = got["ao"].astype(f64), want["ao"]
    diff = np.abs(a - r)
    p = float(f32(settings.final_power))
    ao_slack = max3(slack)
    tight = ao_slack == 0
    moved = ao_slack + 2.0 ** -10  # the flips' slack and one binary16 ulp of every neighbour
    bound = np.where(tight, AO_TIGHT * max(1.0, p), p * moved if p >= 1.0 else moved ** p)
    bad = np.argwhere(diff > bound)
    stats["ao_max"] = float(diff[tight].max()) if tight.any() else 0.0
    stats["ao_max_all"] = float(diff.max())
    stats["ao_mean"] = float(diff[held].mean()) if held.any() else 0.0
    assert bad.size == 0, f"{label} ao: {len(bad)} pixels differ, first at {bad[:3].tolist()}: {a[tuple(bad[0])]} vs {r[tuple(bad[0])]}"
    assert stats["ao_mean"] <= AO_MEAN, f"{label} ao: mean |difference| {stats['ao_mean']:.2e}"
    return stats


# -- scenes: ray-cast in binary64 ----------------------------------------------------------------------------------------------------

def look(yaw_deg=0.0, pitch_deg=0.0, eye=(0.0, 0.0, 0.0)):
    yaw, pitch = math.radians(yaw_deg), math.radians(pitch_deg)
    fwd = np.array([-math.sin(yaw) * math.cos(pitch), math.sin(pitch), -math.cos(yaw) * math.cos(pitch)])
    return synth.look_at(eye, np.asarray(eye) + fwd, (0.0, 1.0, 0.0))


def _rays(w, h, proj, view):
    """world-space origin and per-pixel direction whose parameter t is the linear depth (view-space z of the direction is -1)"""
    p = np.asarray(proj, f32).astype(f64)
    v = np.asarray(view, f32).astype(f64).reshape(4, 4).T
    inv = np.linalg.inv(v)
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    ndc_x, ndc_y = (xs + 0.5) / w * 2 - 1, (ys + 0.5) / h * 2 - 1
    d_view = np.stack([ndc_x / p[0], ndc_y / p[5], -np.ones_like(ndc_x)], -1)
    return inv[:3, 3], d_view @ inv[:3, :3].T


def plane(point, normal, bounds=None):
    point, normal = np.asarray(point, f64), np.asarray(normal, f64)

    def hit(o, d):
        den = d @ normal
        with np.errstate(divide="ignore", invalid="ignore"):
            t = ((point - o) @ normal) / den
        ok = (den < 0) & (t > 0)
        if bounds is not None:
            q = o + d * np.where(ok, t, 0.0)[..., None]
            for axis, (lo, hi) in bounds.items():
                ok &= (q[..., axis] >= lo) & (q[..., axis] <= hi)
        return np.where(ok, t, np.inf), np.broadcast_to(normal, d.shape)
    return hit


def sphere(center, radius):
    c = np.asarray(center, f64)

    def hit(o, d):
        oc = o - c
        a = np.sum(d * d, -1)
        b = np.sum(d * oc, -1)
        disc = b * b - a * (oc @ oc - radius * radius)
        t = (-b - np.sqrt(np.maximum(disc, 0.0))) / a
        t = np.where((disc > 0) & (t > 0), t, np.inf)
        n = o + d * np.where(np.isfinite(t), t, 0.0)[..., None] - c
        return t, n / np.linalg.norm(n, axis=-1, keepdims=True)
    return hit


def box(lo, hi):
    lo, hi = np.asarray(lo, f64), np.asarray(hi, f64)

    def hit(o, d):
        with np.errstate(divide="ignore", invalid="ignore"):
            t0, t1 = (lo - o) / d, (hi - o) / d
        tn, tf = np.minimum(t0, t1), np.maximum(t0, t1)
        t_near, t_far = tn.max(-1), tf.min(-1)
        ok = (t_near <= t_far) & (t_near > 0)
        face = np.argmax(tn, -1)
        n = np.zeros(d.shape)
        np.put_along_axis(n, face[..., None], -np.sign(np.take_along_axis(d, face[..., None], -1)), -1)
        return np.where(ok, t_near, np.inf), n
    return hit


def raycast(w, h, proj, view, prims):
    """depth (D32F, reversed z, 0 where nothing is hit) and normals (oct(world normal) in .zw) of the nearest primitive per pixel"""
    o, d = _rays(w, h, proj, view)
    t = np.full((h, w), np.inf)
    n = np.zeros((h, w, 3))
    n[..., 2] = 1.0
    for prim in prims:
        tp, npr = prim(o, d)
        closer = tp < t
        t = np.where(closer, tp, t)
        n = np.where(closer[..., None], npr, n)
    p = np.asarray(proj, f32).astype(f64)
    depth = np.where(np.isfinite(t), p[14] / t - p[10], 0.0).astype(f32)
    normals = np.zeros((h, w, 4), f32)
    normals[..., 2:] = oct_encode(n)
    return depth, normals


FLOOR = plane((0.0, -1.0, 0.0), (0.0, 1.0, 0.0))


def scene(name, w, h):
    """(camera dict, depth, normals) of the named analytic scene; every one keeps a region of sky"""
    proj, _ = synth.camera_matrices(w, h)
    view = np.eye(4, dtype=f32).reshape(16)
    if name == "crease":  # test_gpu_gtao.crease_frame's floor y = -1 and wall z = -10, the wall ending at y = 3
        prims = [FLOOR, plane((0.0, 0.0, -10.0), (0.0, 0.0, 1.0), {1: (-1.0, 3.0)})]
    elif name == "box":  # a box standing on the floor in front of a wall: concave and convex edges, depth steps
        prims = [FLOOR, box((-1.0, -1.0, -7.0), (1.2, 0.6, -5.0)), plane((0.0, 0.0, -14.0), (0.0, 0.0, 1.0), {1: (-1.0, 2.5)})]
    elif name == "spheres":
        prims = [FLOOR, sphere((-1.5, -0.2, -6.0), 0.8), sphere((0.9, -0.55, -4.0), 0.45), sphere((0.4, 0.5, -9.0), 1.2)]
    elif name == "corridor":  # a narrow corridor with a pit in its floor, open to the sky
        prims = [plane((0.0, -1.0, 0.0), (0.0, 1.0, 0.0), {2: (-1e9, -6.0)}), plane((0.0, -1.0, 0.0), (0.0, 1.0, 0.0), {2: (-4.0, 1e9)}),
                 plane((0.0, -1.6, 0.0), (0.0, 1.0, 0.0)), plane((0.0, 0.0, -6.0), (0.0, 0.0, 1.0), {1: (-1.6, -1.0)}),
                 plane((0.0, 0.0, -4.0), (0.0, 0.0, -1.0), {1: (-1.6, -1.0)}),
                 plane((-0.7, 0.0, 0.0), (1.0, 0.0, 0.0), {1: (-1.6, 1.5)}), plane((0.7, 0.0, 0.0), (-1.0, 0.0, 0.0), {1: (-1.6, 1.5)})]
    elif name == "turned":  # the box scene under a camera with yaw and pitch, so the normals go through the view matrix
        view = look(23.0, -14.0, (0.6, 0.8, 1.5))
        prims = [FLOOR, box((-1.0, -1.0, -7.0), (1.2, 0.6, -5.0)), sphere((-2.0, -0.3, -5.0), 0.7)]
    elif name == "ramp":  # a slanted plane and a tilted floor under a turned camera: no normal is binary16-exact
        view = look(-17.0, -9.0, (0.3, 0.4, 0.0))
        prims = [plane((0.0, -1.3, 0.0), (0.08, 1.0, 0.05) / np.linalg.norm((0.08, 1.0, 0.05))),
                 plane((0.0, 0.0, -9.0), (0.35, 0.2, 1.0) / np.linalg.norm((0.35, 0.2, 1.0)), {1: (-2.0, 2.0)}),
                 sphere((1.2, -0.4, -5.5), 0.6)]
    elif name == "wavy":  # a floor whose shading normals tilt by up to 0.2 rad, as a normal map bends them, with no depth change
        prims = [FLOOR, box((-0.8, -1.0, -8.0), (0.6, 0.2, -6.5))]
    else:
        raise ValueError(name)
    depth, normals = raycast(w, h, proj, view, prims)
    if name == "wavy":
        ys, xs = np.meshgrid(np.arange(h) / h, np.arange(w) / w, indexing="ij")
        a, b = 0.2 * np.sin(37.0 * xs + 5.0 * ys), 0.2 * np.cos(23.0 * ys - 11.0 * xs)
        n = oct_to_vec3(normals[..., 2:4])
        n = n + a[..., None] * np.array([1.0, 0.0, 0.0]) + b[..., None] * np.array([0.0, 0.0, 1.0])
        normals[..., 2:] = oct_encode(n / np.linalg.norm(n, axis=-1, keepdims=True))
    return camera_dict(proj, view), depth, normals


def gtao_camera(cam):
    return abi.gtao_camera(cam["projection"], cam["view"], cam["far_clip"])


@pytest.fixture(scope="module")
def go():
    import os
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    import pyoracle_gtao

    pyoracle_gtao.build()
    return pyoracle_gtao


def _oracle(go, cam, settings, depth, normals):
    return go.generate_ambient_occlusion(gtao_camera(cam), settings, depth, normals)


SCENES = ("crease", "box", "spheres", "corridor", "turned", "ramp", "wavy")


@pytest.mark.parametrize("preset", range(4))
@pytest.mark.parametrize("name", SCENES)
def test_analytic_scene(go, name, preset):
    """every plane of the oracle agrees with the restatement on the ray-cast scenes at 211 x 97, and at 17 x 9 where the border clamp
    and the virtual pyramid reach every pixel"""
    for w, h in ((211, 97), (17, 9)):
        cam, depth, normals = scene(name, w, h)
        settings = abi.gtao_settings(preset)
        want = restate(cam, settings, depth, normals)
        compare(_oracle(go, cam, settings, depth, normals), want, settings, depth, f"{name} {w}x{h} preset {preset}",
                AMBIGUOUS_BOUND if w > 100 else AMBIGUOUS_BOUND_CROP)
        if w > 100:
            held = depth != 0
            assert 0.05 < (~held).mean() < 0.9 and (want["ao"][held] < 0.9).sum() > 50  # sky and occlusion in every scene


@pytest.mark.parametrize("seed", range(6))
def test_random_settings(go, seed):
    """random thickness, radius, slice and sample counts up to 16 / 8, noise_index and power, on the analytic scenes and on
    test_gpu_gtao's non-hostile random frame (normals that do not match the depth)"""
    rng = np.random.default_rng(700 + seed)
    w, h = ((211, 97), (160, 90), (17, 9))[seed % 3]
    settings = random_settings(rng)
    if seed < len(SCENES):
        cam, depth, normals = scene(SCENES[seed], w, h)
    else:
        proj, view = synth.camera_matrices(w, h, 31.0)
        cam = camera_dict(proj, view)
        depth, normals = random_frame(rng, w, h, proj, hostile=False)
    compare(_oracle(go, cam, settings, depth, normals), restate(cam, settings, depth, normals), settings, depth, f"seed {seed}",
            AMBIGUOUS_BOUND_RANDOM if w > 100 else AMBIGUOUS_BOUND_CROP)


@pytest.mark.parametrize("preset", range(4))
def test_random_frame(go, preset):
    rng = np.random.default_rng(90 + preset)
    w, h = 160, 90
    proj, view = synth.camera_matrices(w, h, 12.0 * preset)
    cam = camera_dict(proj, view)
    depth, normals = random_frame(rng, w, h, proj, hostile=False)
    settings = abi.gtao_settings(preset, noise_index=preset * 5)
    compare(_oracle(go, cam, settings, depth, normals), restate(cam, settings, depth, normals), settings, depth, f"preset {preset}",
            AMBIGUOUS_BOUND_RANDOM)


def facing_plane(w, h, distance):
    proj, _ = synth.camera_matrices(w, h)
    cam = camera_dict(proj, np.eye(4, dtype=f32).reshape(16))
    depth, normals = raycast(w, h, proj, cam["view"], [plane((0.0, 0.0, -distance), (0.0, 0.0, 1.0))])
    return cam, depth, normals


@pytest.mark.parametrize("preset", range(4))
def test_facing_plane_gains_at_most_a_sector_per_side(go, preset):
    """a plane facing the camera is not unoccluded: fast_acos(x) = (pi / 2 - 0.156583 |x|) sqrt(1 - |x|) has slope -0.942 at 0
    instead of -1, so a tap in the tangent plane whose horizon lies beyond pi / 2 maps to a small positive arc at the bottom of the
    slice (or just under its top for the other side) and ceil turns it into a whole sector.  The arc cannot reach a second one:
    fast_acos is within 0.011 rad of acos and the projected normal's angle n within 0.005, together far below a sector's pi / 32, and
    the arc starts at the clamped end, sector 0 (or ends at 31).  So each slice side gains at most one sector at falloff <= 1 and
    every noisy texel lies in [30 / 32, 1]; the oracle and the restatement both show it at 2 m and 10 m, with texels below 1"""
    w, h = 320, 180
    for distance in (2.0, 10.0):
        cam, depth, normals = facing_plane(w, h, distance)
        settings = abi.gtao_settings(preset)
        want = restate(cam, settings, depth, normals)
        got = _oracle(go, cam, settings, depth, normals)
        compare(got, want, settings, depth, f"plane at {distance} m")
        for noisy in (want["noisy"], got["noisy"].view(np.float16).astype(f64)):
            assert noisy.min() >= 30 / 32 and noisy.max() <= 1.0
            assert (noisy < 1.0).mean() > 0.5, (noisy < 1.0).mean()
        # without fast_acos's error the same plane is exactly unoccluded: the restatement with acos in its place
        exact = restate_with(cam, settings, depth, normals, fast_acos=np.arccos)
        assert (exact["noisy"] == 1.0).all()


def restate_with(cam, settings, depth, normals, **swap):
    """restate with some of this module's functions replaced"""
    g = globals()
    saved = {k: g[k] for k in swap}
    g.update(swap)
    try:
        return restate(cam, settings, depth, normals)
    finally:
        g.update(saved)


def test_distant_plane_is_exactly_unoccluded(go):
    """once the effect radius projects to under PIXEL_TOO_CLOSE_THRESHOLD (1.3 px), min_s = 1 puts every tap at least the world
    radius R = 1.457 * effect_radius from the nudged origin, where the falloff saturate((R - |delta|) / (0.615 R)) is 0: for 320 px
    and the default radius that is beyond 0.5 * R * projection[0][0] * 320 / 1.3 = 87.4 m.  At 100 m and 300 m both the oracle and
    the restatement give exactly 1 in the noisy and the final plane, at every preset"""
    w, h = 320, 180
    for distance in (100.0, 300.0):
        cam, depth, normals = facing_plane(w, h, distance)
        for preset in range(4):
            settings = abi.gtao_settings(preset)
            want = restate(cam, settings, depth, normals)
            got = _oracle(go, cam, settings, depth, normals)
            assert (want["noisy"] == 1.0).all() and (want["ao"] == 1.0).all()
            assert (got["noisy"] == 0x3C00).all() and (got["ao"] == 1.0).all()
