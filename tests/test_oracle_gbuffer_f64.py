"""The G-buffer decode oracle (oracle/oxc_oracle_gbuffer.c with orc_decode_visbuffer of oracle/oxc_oracle.c) against an independent
binary64 restatement of passes/visbuffer_decode.slang, Material::sample_* and TransformWorld of scene.slang, common/encoding.slang's
vec3_to_oct and SampleGrad as the Vulkan specification defines it, over scenes whose instances are non-uniformly scaled, sheared,
mirrored and tilted up to grazing angles under the perspective camera, with known answers on single planes.

The restatement is written from the shader text, vectorised over pixels, and reads only the scene arrays, the camera, the meshlet
instances, the vis buffer (which triangle owns a pixel), the material table, the samplers and the texel bytes.  It evaluates every
step in binary64:
- the vertex fetch (scene.slang:480-489: half positions and uvs, 10:10:10 normals read as a signed word, c / 511 - 1);
- to_world_positions and normal_matrix / to_world_normals (scene.slang:285-323): the matrix of the three cross products of
  transpose(mat3(world))'s rows, which is the cofactor matrix det(M) M^-T.  On a mirrored instance (det < 0) it reverses the
  normal; the restatement follows the text and does not "fix" that;
- compute_partial_derivatives and gradient_of (visbuffer_decode.slang:27-86) at the pixel-centre tex_coord of fullscreen.slang
  ((x + 0.5) / width, NDC = tex_coord * 2 - 1), with ddy scaled by -2 / resolution.y (:76);
- the uv transform uv * uv_size + uv_offset, ddx, ddy * uv_size (:117-122);
- the world normal, the tangent frame and the normal map (:128-167), vec3_to_oct (common/encoding.slang:17-21);
- Material::sample_* (scene.slang:110-159): albedo * rgba, the normal image's .rgb, emissive * .rgb, (metallic, roughness) * .bg,
  occlusion .r;
- SampleGrad: rho_x, rho_y = the lengths of ddx and ddy scaled to level-0 texels, lambda = log2(max(rho_x, rho_y)); lambda <= 0
  takes the mag filter, else the min filter; d' = clamp(lambda, 0, level_count - 1); mipmap nearest d = 0 for d' <= 0.5, else
  ceil(d' + 0.5) - 1; mipmap linear blends floor(d') and min(floor(d') + 1, q) by frac(d'); linear filtering at x = u * w - 0.5
  with the plain fractional weights (no 8-bit weight quantisation: DESIGN's deviation), nearest at floor(u * w); repeat,
  mirrored repeat ((n - 1) - mirror((i mod 2n) - n)) and clamp to edge; each texel converted before filtering (sRGB EOTF in
  binary64 on RGBA8_SRGB's rgb; R8 and RG8 fill (0, 0, 1) and (0, 1) as the component mapping does).
The shader text leaves NaN open; the restatement follows the GPU's arithmetic as the oracle's specification does: sign(NaN) = 0,
saturate(NaN) = 0, a NaN lambda takes the mag filter at level 0, and a mesh without normals has a NaN world normal.

Comparison rules (oracle against restatement).  The unit of every tolerance is a pixel's relative binary32 error of the geometry,
eps32 * cond, where cond = |inv_det| * max |ndc_i| * (longest NDC edge) * (|inv_w0| + |dv.x * ddx_sum| + |dv.y * ddy_sum|) /
|interp_inv_w|: the cancellation of the NDC determinant and of the interpolated 1/w (grazing planes).  Each constant is given with
the worst case measured over the scenes below and those of tests/test_gpu_gbuffer_f64.py (3 seeds of tilted planes and of deformed
instances at 320 x 192, the two crops, 2 seeds of deformed instances at 640 x 360, the 1920 x 1080 frame):
- COND_LIMIT = 1e4: pixels above it are excluded, under EXCLUDED_BOUND = 0.5 % of the decoded pixels (measured at most 0.055 %, all
  on sub-pixel triangles of the deformed instances).
- lambda, ddx, ddy, uv and uv gradients: within GEOM_REL = 2048 units times the quantity's scale: 1 for lambda, max |tc| for uv,
  max(|ddx_i|, |lambda_i|) for ddx (:82-83 subtract lambda from the neighbour's barycentrics) and that times max |tc| for the uv
  gradients.  Measured at most 522 (lambda at 640 x 360): margin 3.9.
- World normal and mapped normal: compared as unit vectors decoded from the oct codes, by angle, since the code flips sign at the oct
  seam.  The world normal within WORLD_ANGLE_REL = 64 units of 2^-23 + eps32 * cond (measured at most 20.5).  The mapped normal
  within MAPPED_ANGLE_REL = 1024 units of 2^-23 + eps32 * cond * (tcond + 1 + texels), where tcond = max(|pos_ddx| / |pos_ddx_s|,
  |pos_ddy| / |pos_ddy_s|) is the loss when the position derivatives are projected on a plane seen at a grazing angle and texels is
  the triangle's uv extent in texels of the finer level the sample reads (measured at most 348, on the 1920 x 1080 frame).  The
  mean angle over the decided pixels stays under MEAN_ANGLE = 1e-4 rad (measured at most 3.0e-5).  Which pixels are non-finite
  must agree exactly.
- Discrete decisions.  A pixel is ambiguous when, for any of its samples, lambda lies within DELTA_LAMBDA = 1e-3 of 0 (mag != min),
  the clamped lambda within DELTA_LAMBDA of k + 1/2 (mipmap nearest), u * w or v * h of a nearest-filtered level within
  DELTA_TEXEL = 1e-3 texels of an integer, or, under a normal map, the Jacobian determinant behind jacobian_sign or the triple
  product behind w's sign within DELTA_SIGN = 1e-4 (relative) of 0.  Ambiguous pixels stay under AMBIGUOUS_BOUND = 15 % of the
  decoded pixels (measured at most 8.7 %, a magnified near plane under a nearest filter).
- Every other pixel agrees on every channel of albedo, emissive and metallic / roughness / occlusion, relative to max(1, |value|),
  within CHANNEL_REL = 512 units of 2^-23 + eps32 * cond * (1 + texels): a texel coordinate carries the uv error times the texels
  the triangle spans at the level read, the level blend one lambda error (measured at most 123, on the 1920 x 1080 frame).
  These bounds are tight where the geometry is: on the tilted planes the allowed relative error is 1e-3 at the median and 2 % at
  the 99th percentile.  On the deformed instances' sub-pixel triangles the binary32 geometry itself is off by up to 1e-3 relative
  (cond up to COND_LIMIT), and the oracle's channels really differ by up to 0.26 there (a texel coordinate moved across a
  texel); the per-pixel bound follows that, and the mean guard below holds those scenes to systematic errors.
- Mean |difference| over all decided pixels stays under MEAN_TOL = 4e-5 per channel (measured at most 9.5e-6): a systematic
  misreading (a mirrored axis, a lost uv offset, a wrong level, a swapped channel) moves whole surfaces by 1e-2 and more.

Known answers that need no restatement: the cofactor world normal of a sheared, non-uniformly scaled and mirrored plane; the mip
level an oblique plane reads against log2 of its analytic footprint along the major axis; a normal map's tilt on an oblique,
uv-rotated and uv-mirrored plane against the analytic tangent frame.
"""
import math

import numpy as np
import pytest

from oxylus_b200 import abi, synth

f32 = np.float32
f64 = np.float64
EPS32 = 2.0 ** -24

COND_LIMIT = 1e4
EXCLUDED_BOUND = 0.005
GEOM_REL = 2048.0
ANGLE_FLOOR = 2.0 ** -23
WORLD_ANGLE_REL = 64.0
MAPPED_ANGLE_REL = 1024.0
DELTA_LAMBDA = 1e-3
DELTA_TEXEL = 1e-3
DELTA_SIGN = 1e-4
AMBIGUOUS_BOUND = 0.15
CHANNEL_FLOOR = 2.0 ** -23
CHANNEL_REL = 512.0
MEAN_TOL = 4e-5
MEAN_ANGLE = 1e-4


# -- scene.slang: the vertex fetch -------------------------------------------------------------------------------------------------

def _read(blob, dtype, byte_offset):
    """elements of `dtype` at byte offsets (every offset a multiple of the element size)"""
    return blob.view(dtype)[np.asarray(byte_offset, np.int64) // np.dtype(dtype).itemsize]


def fetch(sc, mi, total, vis32):
    """the triangle of every pixel (visbuffer_decode.slang:90-113): dict of per-pixel arrays over the decoded pixels (status 1) and the
    status plane (0 discarded, 1 decoded, 2 a vertex index >= vertex_count)"""
    blob = np.ascontiguousarray(sc.blob)
    h, w = vis32.shape
    v = vis32.reshape(-1).astype(np.int64)
    mii = (v >> abi.VIS_PRIMITIVE_BITS) & 0xFFFFFF
    tri = v & ((1 << abi.VIS_PRIMITIVE_BITS) - 1)
    status = np.zeros(h * w, np.int64)
    live = (v != 0xFFFFFFFF) & (mii != 0xFFFFFE) & (mii < total)
    pix = np.nonzero(live)[0]
    mi = mi[mii[pix]]
    inst = sc.mesh_instances[mi["mesh_instance_index"]]
    mesh = sc.meshes[inst["mesh_index"]]
    lod = mesh["lods"].astype(np.int64) + inst["lod_index"].astype(np.int64) * abi.MESH_LOD_DT.itemsize
    meshlets = _read(blob, np.uint64, lod + 8).astype(np.int64)
    local = _read(blob, np.uint64, lod + 24).astype(np.int64)
    indirect = _read(blob, np.uint64, lod + 32).astype(np.int64)
    meshlet = meshlets + mi["meshlet_index"].astype(np.int64) * abi.MESHLET_DT.itemsize
    ivo = _read(blob, np.uint32, meshlet).astype(np.int64)
    lto = _read(blob, np.uint32, meshlet + 4).astype(np.int64)
    micro = np.stack([blob[local + lto + tri[pix] * 3 + c] for c in range(3)], 1).astype(np.int64)  # scene.slang:336-342
    idx = _read(blob, np.uint32, indirect[:, None] + 4 * (ivo[:, None] + micro)).astype(np.int64)
    last = (mesh["vertex_count"].astype(np.int64) - 1) & 0xFFFFFFFF
    ok = (idx <= last[:, None]).all(1)  # :108-110
    status[pix] = np.where(ok, 1, 2)
    pix, inst, mesh, idx = pix[ok], inst[ok], mesh[ok], idx[ok]
    pos = _read(blob, np.uint16, mesh["vertex_positions"].astype(np.int64)[:, None, None] + 8 * idx[:, :, None] + 2 * np.arange(3))
    pos = pos.view(np.float16).astype(f64)
    has_n = mesh["vertex_normals"] != 0
    nrm = np.zeros((len(pix), 3, 3))
    packed = _read(blob, np.uint32, mesh["vertex_normals"].astype(np.int64)[has_n, None] + 4 * idx[has_n]).view(np.int32)
    nrm[has_n] = ((packed[:, :, None] >> np.array([20, 10, 0])) & 1023) / 511.0 - 1.0  # scene.slang:486-489
    has_t = mesh["texture_coords"] != 0
    tc = np.zeros((len(pix), 3, 2))  # scene.slang:390-399: no coordinates, all zero
    t = _read(blob, np.uint16, mesh["texture_coords"].astype(np.int64)[has_t, None, None] + 4 * idx[has_t][:, :, None] + 2 * np.arange(2))
    tc[has_t] = t.view(np.float16).astype(f64)
    world = sc.transforms["world"][inst["transform_index"]].astype(f64).reshape(-1, 4, 4).transpose(0, 2, 1)  # [col][row] -> M[r][c]
    return dict(pix=pix, status=status.reshape(h, w), pos=pos, normals=nrm, has_normals=has_n, tc=tc, world=world,
                material=inst["material_index"].astype(np.int64))


# -- scene.slang: TransformWorld ----------------------------------------------------------------------------------------------------

def to_world_positions(world, pos):
    """mul(world, f32x4(p, 1)) (:315-321)"""
    return np.einsum("nij,ncj->nci", world[:, :3, :3], pos) + world[:, None, :3, 3]


def normal_matrix(world):
    """:292-299: basis = transpose(mat3(world)), so basis[k] is column k of M; the result is transpose(mat3(rows)), whose columns are
    cross(b1, b2), cross(b2, b0), cross(b0, b1)"""
    b = [world[:, :3, k] for k in range(3)]
    return np.stack([np.cross(b[1], b[2]), np.cross(b[2], b[0]), np.cross(b[0], b[1])], axis=2)


# -- visbuffer_decode.slang ----------------------------------------------------------------------------------------------------------

def partial_derivatives(wp, pv, ndc, resolution):
    """compute_partial_derivatives (:42-86) in binary64; returns lambda, ddx, ddy ([n, 3] each) and the triangle's conditioning"""
    clip = np.einsum("ij,ncj->nci", pv[:, :3], wp) + pv[None, None, :, 3]
    inv_w = 1.0 / clip[:, :, 3]
    n = clip[:, :, :2] * inv_w[:, :, None]
    a, b = n[:, 2] - n[:, 1], n[:, 0] - n[:, 1]
    det = a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]  # determinant(f32x2x2(ndc_2 - ndc_1, ndc_0 - ndc_1)), rows
    with np.errstate(divide="ignore", invalid="ignore"):
        inv_det = 1.0 / det
        ddx = np.stack([n[:, 1, 1] - n[:, 2, 1], n[:, 2, 1] - n[:, 0, 1], n[:, 0, 1] - n[:, 1, 1]], 1) * inv_det[:, None] * inv_w
        ddy = np.stack([n[:, 2, 0] - n[:, 1, 0], n[:, 0, 0] - n[:, 2, 0], n[:, 1, 0] - n[:, 0, 0]], 1) * inv_det[:, None] * inv_w
        ddx_sum, ddy_sum = ddx.sum(1), ddy.sum(1)
        dv = ndc - n[:, 0]
        interp_inv_w = inv_w[:, 0] + dv[:, 0] * ddx_sum + dv[:, 1] * ddy_sum
        interp_w = 1.0 / interp_inv_w
        lam = interp_w[:, None] * (dv[:, 0, None] * ddx + dv[:, 1, None] * ddy)
        lam[:, 0] += interp_w * inv_w[:, 0]
        sx, sy = 2.0 / resolution[0], -2.0 / resolution[1]  # :74-78
        ddx, ddy, ddx_sum, ddy_sum = ddx * sx, ddy * sy, ddx_sum * sx, ddy_sum * sy
        ddx = (1.0 / (interp_inv_w + ddx_sum))[:, None] * (lam * interp_inv_w[:, None] + ddx) - lam  # :80-83
        ddy = (1.0 / (interp_inv_w + ddy_sum))[:, None] * (lam * interp_inv_w[:, None] + ddy) - lam
        edge = np.sqrt(np.maximum((a * a).sum(1), (b * b).sum(1)))
        terms = np.abs(inv_w[:, 0]) + np.abs(dv[:, 0] * ddx_sum) + np.abs(dv[:, 1] * ddy_sum)
        cond = np.abs(inv_det) * np.abs(n).max(axis=(1, 2)) * edge * terms / np.abs(interp_inv_w)
    return lam, ddx, ddy, np.where(np.isfinite(cond), cond, np.inf)


def sign(x):
    """HLSL sign with the GPU's NaN -> 0"""
    return np.where(x > 0, 1.0, np.where(x < 0, -1.0, 0.0))


def normalize(v):
    with np.errstate(divide="ignore", invalid="ignore"):
        return v / np.sqrt((v * v).sum(-1, keepdims=True))


def vec3_to_oct(v):
    """common/encoding.slang:17-21"""
    with np.errstate(divide="ignore", invalid="ignore"):
        p = v[:, :2] * (1.0 / np.abs(v).sum(1))[:, None]
    s = np.where(p >= 0, 1.0, -1.0)
    return np.where((v[:, 2] <= 0)[:, None], (1.0 - np.abs(p[:, ::-1])) * s, p)


def oct_to_vec3(e):
    """common/encoding.slang:7-15, to compare codes as unit vectors"""
    e = np.asarray(e, f64)
    v = np.concatenate([e, (1.0 - np.abs(e[:, :1]) - np.abs(e[:, 1:]))], 1)
    s = np.where(v[:, :2] >= 0, 1.0, -1.0)
    v[:, :2] = np.where((v[:, 2] < 0)[:, None], (1.0 - np.abs(v[:, 1::-1])) * s, v[:, :2])
    return normalize(v)


def angle(a, b):
    """angle between unit vectors, stable near 0"""
    return 2.0 * np.arcsin(np.minimum(np.linalg.norm(a - b, axis=-1) / 2.0, 1.0))


# -- SampleGrad (Vulkan specification, Texel Filtering / LOD / Addressing) --------------------------------------------------------

def srgb_eotf(c):
    c = np.asarray(c, f64)
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


def texels_rgba(level, fmt):
    """one level's texels as RGBA binary64, converted before filtering"""
    t = np.asarray(level, f64) / 255.0
    hgt, wid = t.shape[:2]
    out = np.zeros((hgt, wid, 4))
    out[..., 3] = 1.0
    if fmt == abi.IMAGE_R8_UNORM:
        out[..., 0] = t
    elif fmt == abi.IMAGE_RG8_UNORM:
        out[..., :2] = t
    else:
        out[:] = t
        if fmt == abi.IMAGE_RGBA8_SRGB:
            out[..., :3] = srgb_eotf(t[..., :3])
    return out


def wrap(i, n, mode):
    if mode == abi.ADDRESS_CLAMP_TO_EDGE:
        return np.clip(i, 0, n - 1)
    if mode == abi.ADDRESS_MIRRORED_REPEAT:
        t = np.mod(i, 2 * n) - n
        return (n - 1) - np.where(t >= 0, t, -(1 + t))
    return np.mod(i, n)


def _int(x):
    return np.where(np.isfinite(x), x, 0.0).astype(np.int64)


def sample_level(tex, u, v, filt, au, av):
    """tex: RGBA [h, w, 4]; u, v: [n]"""
    hgt, wid = tex.shape[:2]
    if filt == abi.FILTER_NEAREST:
        i, j = _int(np.floor(u * wid)), _int(np.floor(v * hgt))
        return tex[wrap(j, hgt, av), wrap(i, wid, au)]
    x, y = u * wid - 0.5, v * hgt - 0.5
    x0, y0 = np.floor(x), np.floor(y)
    a, b = (x - x0)[:, None], (y - y0)[:, None]
    i0, j0 = _int(x0), _int(y0)
    ia, ib, ja, jb = wrap(i0, wid, au), wrap(i0 + 1, wid, au), wrap(j0, hgt, av), wrap(j0 + 1, hgt, av)
    return ((1 - a) * (1 - b) * tex[ja, ia] + a * (1 - b) * tex[ja, ib] + (1 - a) * b * tex[jb, ia] + a * b * tex[jb, ib])


class Image:
    def __init__(self, levels, fmt):
        levels = levels if isinstance(levels, (list, tuple)) else [levels]
        self.tex = [texels_rgba(lv, fmt) for lv in levels]
        self.h0, self.w0 = self.tex[0].shape[:2]
        self.q = len(levels) - 1


def lod(img, dx, dy):
    """lambda = log2(max(rho_x, rho_y)), the gradients scaled to level-0 texels"""
    rx = np.hypot(dx[:, 0] * img.w0, dx[:, 1] * img.h0)
    ry = np.hypot(dy[:, 0] * img.w0, dy[:, 1] * img.h0)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.log2(np.maximum(rx, ry))


def sample_grad(img, smp, u, v, dx, dy):
    """returns (RGBA [n, 4], ambiguous [n])"""
    mag, mn, mip, au, av = (int(smp[k]) for k in ("mag_filter", "min_filter", "mipmap_mode", "address_u", "address_v"))
    lam = lod(img, dx, dy)
    d1 = np.where(lam > 0, np.minimum(lam, img.q), 0.0)  # NaN -> level 0, mag
    minify = lam > 0
    amb = np.zeros(len(u), bool)
    if mag != mn:
        amb |= np.abs(lam) < DELTA_LAMBDA
    if mip == abi.MIPMAP_NEAREST:
        lo = np.where(d1 <= 0.5, 0, np.ceil(d1 + 0.5) - 1).astype(np.int64)
        hi, frac = lo, np.zeros(len(u))
        amb |= (np.abs(d1 - np.round(d1 - 0.5) - 0.5) < DELTA_LAMBDA) & (d1 > 0) & (d1 < img.q)
    else:
        lo = np.floor(d1).astype(np.int64)
        hi, frac = np.minimum(lo + 1, img.q), d1 - lo
    filt_of = np.where(minify, mn, mag)
    parts = [(lo, np.ones(len(u)))] if mip == abi.MIPMAP_NEAREST else [(lo, 1.0 - frac), (hi, frac)]
    out = np.zeros((len(u), 4))
    for lv, weight in parts:
        for level in np.unique(lv):
            tex = img.tex[level]
            hgt, wid = tex.shape[:2]
            for filt in {mn, mag}:
                m = np.nonzero((lv == level) & (filt_of == filt) & (weight > 0))[0]
                if not len(m):
                    continue
                out[m] += weight[m, None] * sample_level(tex, u[m], v[m], filt, au, av)
                if filt == abi.FILTER_NEAREST:
                    fu, fv = u[m] * wid, v[m] * hgt
                    amb[m] |= (np.abs(fu - np.round(fu)) < DELTA_TEXEL) | (np.abs(fv - np.round(fv)) < DELTA_TEXEL)
    return out, amb


def half(x):
    return np.asarray(x, np.uint16).view(np.float16).astype(f64)


# -- the whole decode -------------------------------------------------------------------------------------------------------------

def restate(sc, mi, total, cam, vis32, materials, images, samplers):
    """the four planes (oct codes for normal.xy / .zw), the geometry planes and the per-pixel ambiguity / conditioning, over the
    decoded pixels of `vis32`.  images: list of (levels, format) as the material table holds them; samplers: SAMPLER_DT or None."""
    h, w = vis32.shape
    f = fetch(sc, mi, total, vis32)
    pix, n_px = f["pix"], len(f["pix"])
    pv = cam["projection_view"][0].astype(f64).reshape(4, 4).T
    res = cam["resolution"][0].astype(f64)
    cam_pos = cam["position"][0].astype(f64)
    ndc = np.stack([((pix % w) + 0.5) / w, ((pix // w) + 0.5) / h], 1) * 2.0 - 1.0
    wp = to_world_positions(f["world"], f["pos"])
    lam, ddx, ddy, cond = partial_derivatives(wp, pv, ndc, res)
    tc = f["tc"]
    uv, uv_dx, uv_dy = (np.einsum("nc,ncj->nj", d, tc) for d in (lam, ddx, ddy))  # gradient_of (:32-39)
    nm = normal_matrix(f["world"])
    wn = np.einsum("nij,ncj->nci", nm, f["normals"])
    world_normal = normalize(np.einsum("nc,nci->ni", lam, wn))  # :136-137; no normals: 0 / 0 = NaN
    rel = wp - cam_pos  # :128-134
    pdx, pdy = np.einsum("nc,nci->ni", ddx, rel), np.einsum("nc,nci->ni", ddy, rel)

    out = {k: np.zeros((n_px, 4)) for k in abi.GBUFFER_PLANES}
    amb = np.zeros(n_px, bool)
    bad = np.zeros(n_px, bool)
    tcond = np.ones(n_px)
    texels = np.zeros(n_px)  # the triangle's uv extent in texels of the finer level each sample reads, the largest over its samples
    imgs = [Image(t, fmt) for t, fmt in images]
    default = np.array([abi.sampler()], dtype=abi.SAMPLER_DT)[0]
    for m in np.unique(f["material"]):
        sel = np.nonzero(f["material"] == m)[0]
        if m >= len(materials):
            bad[sel] = True
            continue
        mat = materials[m]
        smp = samplers[mat["sampler_index"]] if samplers is not None and mat["sampler_index"] < len(samplers) else default
        size, offset = half(mat["uv_size"]), half(mat["uv_offset"])
        extent = np.abs(size) * (tc[sel].max(1) - tc[sel].min(1))
        u = uv[sel] * size + offset  # :119-122
        dx, dy = uv_dx[sel] * size, uv_dy[sel] * size
        flags = int(mat["flags"])

        def sample(slot):
            img = imgs[int(mat[slot])]
            lam = lod(img, dx, dy)
            finest = np.exp2(-np.floor(np.where(lam > 0, np.minimum(lam, img.q), 0.0)))  # the finer level it reads
            texels[sel] = np.maximum(texels[sel], np.maximum(extent[:, 0] * img.w0, extent[:, 1] * img.h0) * finest)
            s, a = sample_grad(img, smp, u[:, 0], u[:, 1], dx, dy)
            amb[sel] |= a
            return s

        albedo = np.broadcast_to(half(mat["albedo_color"]), (len(sel), 4)).copy()  # scene.slang:110-119
        if flags & abi.MATERIAL_HAS_ALBEDO_IMAGE:
            albedo *= sample("albedo_image_index")
        emissive = np.broadcast_to(half(mat["emissive_color"]), (len(sel), 3)).copy()  # :130-139
        if flags & abi.MATERIAL_HAS_EMISSIVE_IMAGE:
            emissive *= sample("emissive_image_index")[:, :3]
        mr = np.broadcast_to(np.array([half(mat["metallic_factor"]), half(mat["roughness_factor"])]), (len(sel), 2)).copy()  # :141-150
        if flags & abi.MATERIAL_HAS_METALLIC_ROUGHNESS_IMAGE:
            mr *= sample("metallic_roughness_image_index")[:, [2, 1]]  # .bg
        occ = np.ones(len(sel))  # :152-158
        if flags & abi.MATERIAL_HAS_OCCLUSION_IMAGE:
            occ = sample("occlusion_image_index")[:, 0]

        # :139-167 the tangent frame and the normal map
        n = world_normal[sel]
        px_s = pdx[sel] - (pdx[sel] * n).sum(1, keepdims=True) * n
        py_s = pdy[sel] - (pdy[sel] * n).sum(1, keepdims=True) * n
        jac = dx[:, 0] * dy[:, 1] - dx[:, 1] * dy[:, 0]
        js = sign(jac)[:, None]
        tangent = js * (dy[:, 1, None] * px_s - dx[:, 1, None] * py_s)
        tangent = np.where(js != 0, normalize(tangent), tangent)
        with np.errstate(divide="ignore", invalid="ignore"):
            tcond[sel] = np.maximum(np.linalg.norm(pdx[sel], axis=1) / np.linalg.norm(px_s, axis=1),
                                    np.linalg.norm(pdy[sel], axis=1) / np.linalg.norm(py_s, axis=1))
        triple = (pdy[sel] * np.cross(n, pdx[sel])).sum(1)
        wsign = js * sign(triple)[:, None]
        bitangent = -wsign * np.cross(n, tangent)
        normal = n
        if flags & abi.MATERIAL_HAS_NORMAL_IMAGE:
            e = sample("normal_image_index")[:, :3] * 2.0 - 1.0
            if flags & abi.MATERIAL_NORMAL_FLIP_Y:
                e[:, 1] = -e[:, 1]
            if flags & abi.MATERIAL_NORMAL_TWO_COMPONENT:
                e[:, 2] = np.sqrt(np.clip(1.0 - (e[:, :2] ** 2).sum(1), 0.0, 1.0))
            normal = normalize(e[:, :1] * tangent + e[:, 1:2] * bitangent + e[:, 2:] * n)
            scale = lambda a, b: np.abs(a) <= DELTA_SIGN * b  # noqa: E731
            amb[sel] |= scale(jac, np.abs(dx[:, 0] * dy[:, 1]) + np.abs(dx[:, 1] * dy[:, 0])) & (jac != 0)
            mag = np.linalg.norm(n, axis=1) * np.linalg.norm(pdx[sel], axis=1) * np.linalg.norm(pdy[sel], axis=1)
            amb[sel] |= scale(triple, mag) & (triple != 0) & (js[:, 0] != 0)
        out["albedo"][sel] = albedo
        out["normal"][sel, :2] = vec3_to_oct(normal)
        out["normal"][sel, 2:] = vec3_to_oct(n)
        out["emissive"][sel, :3] = emissive
        out["metallic_roughness_occlusion"][sel, :2] = mr
        out["metallic_roughness_occlusion"][sel, 2] = occ
    for k in out:
        out[k][bad] = 0.0
    geom = dict(lambda_=lam, ddx=ddx, ddy=ddy, uv=uv, uv_ddx=uv_dx, uv_ddy=uv_dy, tc=tc)
    return dict(pix=pix, status=f["status"], planes=out, geom=geom, cond=cond, tcond=tcond, ambiguous=amb, bad=bad,
                world_normal=world_normal, det=np.linalg.det(f["world"][:, :3, :3]), has_uv=f["tc"].any(axis=(1, 2)),
                texels=texels)


# -- scenes -------------------------------------------------------------------------------------------------------------------------

def rotation(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def linear_part(rng, i):
    """rotation x shear x non-uniform scale (axis ratios up to 8), mirrored in one axis on every third"""
    s = 2.0 ** rng.uniform(-1.5, 1.5, 3)
    shear = np.eye(3)
    if i % 2:
        shear[np.triu_indices(3, 1)] = rng.uniform(-0.8, 0.8, 3)
    if i % 3 == 2:
        s[rng.integers(0, 3)] *= -1.0
    return rotation(rng) @ shear @ np.diag(s)


def set_world(sc, k, m3, t):
    world = np.eye(4, dtype=f32)  # [col][row]
    world[:3, :3] = np.asarray(m3, f32).T
    world[3, :3] = t
    sc.transforms["world"][k] = world.reshape(16)


def deformed_scene(seed, width, height, n_meshlets=20_000, n_materials=48, scale=6.0, bench=False):
    """synth.make_scene's instances with their rotation x uniform scale replaced by linear_part, scaled up so that triangles span
    from a pixel to tens of pixels; random materials.  bench=True starts from the scene bench.py measures (make_scene's default seed
    and mesh count) instead of a small seeded one."""
    if bench:
        sc = synth.make_scene(n_meshlets, config_index=2, width=width, height=height)
    else:
        sc = synth.make_scene(n_meshlets, config_index=2, width=width, height=height, n_unique_meshes=16, seed=1000 + seed)
    rng = np.random.default_rng(seed)
    for k in range(len(sc.transforms)):
        w = sc.transforms["world"][k].reshape(4, 4)
        s = np.linalg.norm(w[0, :3])
        set_world(sc, k, linear_part(rng, k) * s * scale, w[3, :3])
    sc.mesh_instances["material_index"] = rng.integers(0, n_materials, sc.mesh_instance_count)
    return sc


def tilt(theta, phi):
    """rotation by theta about the in-plane axis (cos phi, sin phi, 0)"""
    a = np.array([math.cos(phi), math.sin(phi), 0.0])
    k = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(theta) * k + (1 - math.cos(theta)) * k @ k


def planes_scene(seed, width, height, n=24, n_materials=48):
    """n quads (tests/helpers_scene.quad_scene's mesh: local [-0.5, 0.5]^2 at z = 0.5, normal +z, uv = xy + 0.5) under the perspective
    camera, each tilted 30-85 degrees to the view, non-uniformly scaled, sheared or mirrored, from 2 to 80 units away and from a few
    pixels to most of the screen across.  Instance 0 (mesh 1) has no normals and instances 1 and 2 (mesh 2) no texture coordinates;
    they sit 2 units away, in front of the others."""
    from tests.helpers_scene import quad_scene

    base, _ = quad_scene(width, height, attributes=True)
    rng = np.random.default_rng(seed)
    meshes = np.concatenate([base.meshes] * 3)
    meshes["vertex_normals"][1] = 0
    meshes["texture_coords"][2] = 0
    inst = np.zeros(n, dtype=abi.MESH_INSTANCE_DT)
    inst["mesh_index"][:3] = (1, 2, 2)
    inst["transform_index"] = np.arange(n)
    inst["meshlet_instance_visibility_offset"] = np.arange(n)
    inst["material_index"] = rng.integers(0, n_materials, n)
    sc = synth.Scene(meshes, inst, np.zeros(n, dtype=abi.TRANSFORM_DT), base.blob, n, width, height, seed)
    aspect = width / height
    for k in range(n):
        d = 2.0 if k < 3 else math.exp(rng.uniform(math.log(3.0), math.log(80.0)))
        size = d * (0.4 if k < 3 else rng.uniform(0.05, 1.2))
        s = np.array([size * 2.0 ** rng.uniform(-1.5, 1.5), size * 2.0 ** rng.uniform(-1.5, 1.5), size])
        shear = np.eye(3)
        if k % 2:
            shear[0, 1] = rng.uniform(-0.8, 0.8)
        if k % 3 == 2:
            s[k % 2] *= -1.0  # mirrored in x or y: det < 0
        m3 = tilt(math.radians(rng.uniform(30.0, 85.0)), rng.uniform(0, 2 * math.pi)) @ shear @ np.diag(s)
        if k % 3 != 2:
            m3 = np.diag([-1.0, 1.0, -1.0]) @ m3  # turned about y: the camera's y flip makes the unmirrored quad's +z side its back
        x = (-0.5, 0.5, 0.0)[k] if k < 3 else rng.uniform(-0.6, 0.6)
        t = np.array([x * d * 0.577 * aspect, rng.uniform(-0.6, 0.6) * d * 0.577, -d]) - m3 @ [0.0, 0.0, 0.5]
        set_world(sc, k, m3, t)
    return sc


def odd_images(rng):
    """tests.test_gpu_gbuffer.random_images plus a truncated non-square chain (the clamp at level_count - 1 above a 1 x 1 level) and an
    odd non-square chain; format = index % 4 as random_materials expects"""
    import pyoracle as orc
    from tests.test_gpu_gbuffer import random_images

    images = random_images(rng)
    l0 = rng.integers(0, 256, (16, 64, 4), dtype=np.uint8)
    images.append((orc.mip_chain(l0)[:3], abi.IMAGE_RGBA8_SRGB))
    images.append((orc.mip_chain(rng.integers(0, 256, (7, 13, 2), dtype=np.uint8)), abi.IMAGE_RG8_UNORM))
    return images


def material_table(seed, n_materials=48):
    import pyoracle as orc
    from tests.test_gpu_gbuffer import random_materials, random_samplers

    rng = np.random.default_rng(seed)
    images = odd_images(rng)
    samplers = random_samplers(rng)
    mats = random_materials(rng, n_materials, len(images), len(samplers))
    return dict(materials=mats, images=images, samplers=samplers, host=orc.MaterialTable(mats, images, samplers))


def cpu_vis(orc, sc, cam):
    """the oracle's two-pass frame: (host scene, meshlet instances, total, vis32)"""
    hs = orc.HostScene(sc)
    ref = orc.cpu_frame(hs, cam, sc.width, sc.height, np.zeros((sc.max_meshlet_instance_count + 31) // 32, np.uint32), None, 8)
    v32, _ = orc.resolve(ref["vis64"])
    return hs, ref["meshlet_instances"], int(ref["visibility"]["total"][0]), v32


# -- the comparison -----------------------------------------------------------------------------------------------------------------

CHANNELS = (("albedo", slice(0, 4)), ("emissive", slice(0, 3)), ("metallic_roughness_occlusion", slice(0, 3)))


def compare(r, planes, geom=None):
    """checks the planes ({plane: float32 [H, W, 4]}) and, when given, orc.decode_visbuffer's geometry planes of a decode against the
    restatement r under the module's rules; returns the measured worst cases (each as the ratio to its unit)"""
    pix = r["pix"]
    n = len(pix)
    assert n > 0
    flat = {k: p.reshape(-1, 4)[pix].astype(f64) for k, p in planes.items()}
    well = r["cond"] <= COND_LIMIT
    unit = np.where(well, r["cond"], 0.0) * EPS32  # the relative binary32 error of the geometry at each pixel
    out = dict(decoded=n, excluded=float(1.0 - well.mean()))
    assert out["excluded"] <= EXCLUDED_BOUND, out
    if geom is not None:
        assert (geom["lambda_"].reshape(-1, 4)[pix, 3] == 1.0).all()
        g = r["geom"]
        tcs = np.abs(g["tc"]).max(axis=(1, 2))
        got = dict(lambda_=geom["lambda_"].reshape(-1, 4)[pix, :3], ddx=geom["ddx"].reshape(-1, 4)[pix, :3],
                   ddy=geom["ddy"].reshape(-1, 4)[pix, :3], uv=geom["uv_normal"].reshape(-1, 4)[pix, :2],
                   uv_ddx=geom["uv_grad"].reshape(-1, 4)[pix, :2], uv_ddy=geom["uv_grad"].reshape(-1, 4)[pix, 2:])
        out["geom"] = 0.0
        for k, v in got.items():
            scale = {"lambda_": np.ones(n), "uv": tcs}.get(k)
            if scale is None:
                d = g["ddx" if k in ("ddx", "uv_ddx") else "ddy"]  # :82-83 subtract lambda: the difference of two O(lambda) terms
                scale = np.maximum(np.abs(d), np.abs(g["lambda_"])).max(1) * (tcs if k.startswith("uv") else 1.0)
            err = np.abs(v.astype(f64) - g[k]).max(1)[well] / (np.maximum(scale, 1e-30) * unit)[well]
            assert np.isfinite(err).all(), k
            out["geom"] = max(out["geom"], float(err.max()))
            assert err.max() <= GEOM_REL, (k, err.max())
    amb, bad = r["ambiguous"] | ~well, r["bad"]
    out["world_angle"] = out["mapped_angle"] = 0.0
    sampled = 1.0 + r["texels"]  # a texel coordinate carries the uv error times the texels it spans, the level blend one lambda error
    out["mean_angle"] = 0.0
    for lo, name, bound, cnd in ((2, "world", WORLD_ANGLE_REL, 1.0), (0, "mapped", MAPPED_ANGLE_REL, r["tcond"] + sampled)):
        want, got = r["planes"]["normal"][:, lo:lo + 2], flat["normal"][:, lo:lo + 2]
        fin = np.isfinite(want).all(1)
        np.testing.assert_array_equal(np.isfinite(got).all(1), fin, err_msg=f"{name} normal: the non-finite pixels differ")
        keep = fin & ~amb & ~bad
        a = angle(oct_to_vec3(got[keep]), oct_to_vec3(want[keep]))
        ratio = a / (ANGLE_FLOOR + (unit * cnd)[keep])
        out[name + "_angle"] = float(ratio.max(initial=0.0))
        assert out[name + "_angle"] <= bound, (name, out)
        out["mean_angle"] = max(out["mean_angle"], float(a.mean()) if len(a) else 0.0)
        assert out["mean_angle"] <= MEAN_ANGLE, (name, out)
    out["ambiguous"] = float(r["ambiguous"].mean())
    assert out["ambiguous"] <= AMBIGUOUS_BOUND, out
    decided = ~amb & ~bad
    out["channel"] = out["mean"] = 0.0
    for k, sl in CHANNELS:
        want, got = r["planes"][k][:, sl], flat[k][:, sl]
        np.testing.assert_array_equal(got[bad], 0.0)
        err = np.abs(got - want) / np.maximum(np.abs(want), 1.0)
        ratio = err[decided] / (CHANNEL_FLOOR + (unit * sampled)[decided, None])
        assert np.isfinite(ratio).all(), k
        out["channel"] = max(out["channel"], float(ratio.max(initial=0.0)))
        assert ratio.max(initial=0.0) <= CHANNEL_REL, (k, out)
        mean = np.abs(got - want)[decided].mean(0)
        out["mean"] = max(out["mean"], float(mean.max()))
        assert mean.max() <= MEAN_TOL, (k, mean)
    return out


def oracle_decode(orc, gb, hs, mi, total, cam, v32, table):
    want, bad = gb.decode_gbuffer(hs, mi, total, cam, v32, table["host"], init=np.float32(-7.25))
    return want, orc.decode_visbuffer(hs, mi, total, cam, v32)


def check_scene(orc, gb, sc, seed):
    """the oracle's decode of the oracle's frame of `sc` against the restatement; returns (measured worst cases, restatement)"""
    cam = synth.make_camera(sc.width, sc.height, sc.mesh_instance_count)
    hs, mi, total, v32 = cpu_vis(orc, sc, cam)
    table = material_table(seed)
    want, geom = oracle_decode(orc, gb, hs, mi, total, cam, v32, table)
    r = restate(sc, mi, total, cam, v32, table["materials"], table["images"], table["samplers"])
    np.testing.assert_array_equal(r["status"] == 0, want["albedo"][:, :, 0] == np.float32(-7.25))
    return compare(r, want, geom), r


@pytest.fixture(scope="module")
def gb():
    import pyoracle_gbuffer

    pyoracle_gbuffer.build()
    return pyoracle_gbuffer


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_tilted_planes_against_restatement(orc, gb, seed):
    """quads tilted 30-85 degrees, near and far, non-uniformly scaled, sheared and mirrored, some without normals or texture
    coordinates, from a few pixels to most of the 320 x 192 frame"""
    m, r = check_scene(orc, gb, planes_scene(seed, 320, 192), seed)
    assert m["decoded"] > 1500
    assert (r["det"] < 0).sum() > 100 and (r["det"] > 0).sum() > 100
    assert (~np.isfinite(r["world_normal"]).all(1)).sum() > 100 and (~r["has_uv"]).sum() > 100


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_deformed_instances_against_restatement(orc, gb, seed):
    """synth.make_scene's height-field meshlets with non-uniform, sheared and mirrored transforms at 320 x 192"""
    m, r = check_scene(orc, gb, deformed_scene(seed, 320, 192), seed)
    assert m["decoded"] > 10_000
    assert (r["det"] < 0).sum() > 2000


@pytest.mark.parametrize("kind", ["planes", "deformed"])
def test_border_crop_against_restatement(orc, gb, kind):
    """odd, small frames (53 x 37, 61 x 29) whose triangles run across every border"""
    sc = planes_scene(4, 53, 37) if kind == "planes" else deformed_scene(4, 61, 29)
    m, r = check_scene(orc, gb, sc, 4)
    assert m["decoded"] > 300


# -- known answers ------------------------------------------------------------------------------------------------------------------

def one_plane(m3, d, width=160, height=96):
    """planes_scene's quad alone, linear part m3, centred d units ahead of the camera"""
    full = planes_scene(0, width, height, n=3)
    sc = synth.Scene(full.meshes, full.mesh_instances[:1].copy(), full.transforms[:1].copy(), full.blob, 1, width, height, 0)
    sc.mesh_instances["mesh_index"] = sc.mesh_instances["material_index"] = 0
    set_world(sc, 0, m3, np.array([0.0, 0.0, -d]) - np.asarray(m3) @ [0.0, 0.0, 0.5])
    return sc


@pytest.mark.parametrize("mirrored", [False, True])
def test_world_normal_is_the_cofactor_normal(orc, gb, mirrored):
    """a plane tilted 55 degrees, sheared and scaled 1 : 3 : 7: the decoded world normal (normal.zw) is normalize(M^-T n) * sign(det M)
    on every pixel, to a few binary32 ulps in angle; mirrored in x, that is the reversed geometric normal, as the reference's cofactor
    matrix gives it"""
    shear = np.eye(3)
    shear[0, 1] = 0.6
    base = tilt(np.radians(55.0), 0.7) @ shear @ np.diag([1.0, 3.0, 7.0])
    m3 = base @ np.diag([-1.0, 1.0, 1.0]) if mirrored else np.diag([-1.0, 1.0, -1.0]) @ base  # planes_scene's orientations
    sc = one_plane(m3, 6.0)
    cam = synth.make_camera(sc.width, sc.height, 1)
    hs, mi, total, v32 = cpu_vis(orc, sc, cam)
    want, _ = oracle_decode(orc, gb, hs, mi, total, cam, v32, material_table(0))
    got = want["normal"][:, :, 2:][v32 != 0xFFFFFFFF]
    assert len(got) > 200
    m = np.asarray(sc.transforms["world"][0], f64).reshape(4, 4).T[:3, :3]
    geometric = np.linalg.inv(m).T @ [0.0, 0.0, 1.0]
    expect = geometric / np.linalg.norm(geometric) * np.sign(np.linalg.det(m))
    assert (np.linalg.det(m) < 0) == mirrored
    a = angle(oct_to_vec3(got), np.broadcast_to(expect, (len(got), 3)))
    assert a.max() < 8 * 2.0 ** -23, a.max()
    assert (np.dot(expect, geometric) < 0) == mirrored


def plane_uv(m3, t, cam, ndc):
    """analytic texture coordinate of planes_scene's quad (uv = local xy + 0.5) where the camera ray through `ndc` meets it"""
    inv_pv = np.linalg.inv(cam["projection_view"][0].astype(f64).reshape(4, 4).T)
    eye = cam["position"][0].astype(f64)
    far = np.concatenate([ndc, np.full((len(ndc), 1), 0.5), np.ones((len(ndc), 1))], 1) @ inv_pv.T
    ray = far[:, :3] / far[:, 3:] - eye
    inv = np.linalg.inv(m3)
    o, d = inv @ (eye - t), ray @ inv.T  # the ray in the quad's local frame
    s = (0.5 - o[2]) / d[:, 2]
    return o[:2] + s[:, None] * d[:, :2] + 0.5


def test_mip_level_follows_the_analytic_footprint(orc, gb):
    """a plane tilted 72 degrees about x, textured (uv_size 6) with a 64 x 64 chain whose level k is one flat colour, sampled nearest /
    nearest / mipmap nearest: every pixel reads the level that the Vulkan rule picks from lambda = log2 of the larger of the analytic
    footprints, |uv(x + 1) - uv(x)| and |uv(y - 1) - uv(y)| in texels (the decode's ddx and ddy are those forward differences, :66-83).
    The plane is foreshortened along y, so the x axis alone would pick another level on many pixels."""
    levels = [np.full((64 >> k, 64 >> k, 4), (40 * k + 10, 200 - 30 * k, 7 * k, 255), np.uint8) for k in range(7)]
    m = np.zeros(1, dtype=abi.MATERIAL_DT)
    m[0]["flags"] = abi.MATERIAL_HAS_ALBEDO_IMAGE
    m[0]["albedo_color"] = [int(np.float16(1.0).view(np.uint16))] * 4
    m[0]["uv_size"] = [int(np.float16(6.0).view(np.uint16))] * 2
    smp = np.array([(abi.FILTER_NEAREST, abi.FILTER_NEAREST, abi.MIPMAP_NEAREST, abi.ADDRESS_REPEAT, abi.ADDRESS_REPEAT)], dtype=abi.SAMPLER_DT)
    import pyoracle
    table = dict(host=pyoracle.MaterialTable(m, [(levels, abi.IMAGE_RGBA8_UNORM)], smp))
    m3 = np.diag([-1.0, 1.0, -1.0]) @ tilt(np.radians(72.0), 0.0) @ np.diag([6.0, 6.0, 1.0])
    sc = one_plane(m3, 4.0)
    t = sc.transforms["world"][0].reshape(4, 4)[3, :3].astype(f64)
    m3 = sc.transforms["world"][0].reshape(4, 4)[:3, :3].T.astype(f64)
    cam = synth.make_camera(sc.width, sc.height, 1)
    hs, mi, total, v32 = cpu_vis(orc, sc, cam)
    want, _ = oracle_decode(orc, gb, hs, mi, total, cam, v32, table)
    ys, xs = np.nonzero(v32 != 0xFFFFFFFF)
    ndc = np.stack([(xs + 0.5) / sc.width, (ys + 0.5) / sc.height], 1) * 2.0 - 1.0
    uv = plane_uv(m3, t, cam, ndc) * 6.0
    fx = np.linalg.norm(plane_uv(m3, t, cam, ndc + [2.0 / sc.width, 0.0]) * 6.0 - uv, axis=1) * 64
    fy = np.linalg.norm(plane_uv(m3, t, cam, ndc + [0.0, -2.0 / sc.height]) * 6.0 - uv, axis=1) * 64

    def level(rho):
        d = np.clip(np.log2(rho), 0.0, 6.0)
        return np.where(d <= 0.5, 0, np.ceil(d + 0.5) - 1).astype(int), d

    k, d = level(np.maximum(fx, fy))
    clear = np.abs(d - np.floor(d) - 0.5) > 1e-2  # away from a rounding edge
    colour = np.array([lv[0, 0, 0] for lv in levels], f64) / 255.0
    got = want["albedo"][ys, xs, 0]
    assert clear.sum() > 1000 and len(np.unique(k[clear])) >= 3
    np.testing.assert_array_equal(got[clear], colour[k[clear]].astype(f32))
    kx, _ = level(fx)
    assert (kx[clear] != k[clear]).mean() > 0.3


@pytest.mark.parametrize("uv_size", [(1.0, 1.0), (-1.0, 1.0)])
def test_normal_map_tilt_in_the_analytic_tangent_frame(orc, gb, uv_size):
    """a plane tilted 50 degrees, sheared and scaled 2 : 5, whose texture coordinates are the local xy rotated by atan(4 / 3) and
    scaled by 10 (integers at the corners, exact in binary16), optionally mirrored in u by uv_size; a 1 x 1 normal map holds the tilt
    e = (200, 90, 230) / 255 * 2 - 1.  The mapped normal is normalize(e.x T + e.y B + e.z n) in the analytic frame of the plane:
    n the geometric normal, T = normalize(dp/du), B = -w cross(n, T) with w = sign(n . (dp/du x dp/dv)) (:144-150 with the position
    and uv differences of one plane, whose ratios are the exact dp/du, dp/dv)."""
    import pyoracle

    rot = np.array([[0.6, -0.8], [0.8, 0.6]]) * 10.0
    shear = np.eye(3)
    shear[0, 1] = 0.5
    m3 = np.diag([-1.0, 1.0, -1.0]) @ tilt(np.radians(50.0), 2.0) @ shear @ np.diag([2.0, 5.0, 1.0])
    sc = one_plane(m3, 5.0)
    sc.blob = sc.blob.copy()
    corners = np.array([[-0.5, -0.5], [0.5, -0.5], [0.5, 0.5], [-0.5, 0.5]])  # tests/helpers_scene.quad_scene's vertices
    off = int(sc.meshes["texture_coords"][0])
    sc.blob[off:off + 16] = synth.quantize_half((corners @ rot.T).astype(f32)).view(np.uint8).reshape(-1)
    texel = np.array([200, 90, 230, 255], np.uint8).reshape(1, 1, 4)
    m = np.zeros(1, dtype=abi.MATERIAL_DT)
    m[0]["flags"] = abi.MATERIAL_HAS_NORMAL_IMAGE
    m[0]["uv_size"] = [int(np.float16(x).view(np.uint16)) for x in uv_size]
    smp = np.array([(abi.FILTER_NEAREST, abi.FILTER_NEAREST, abi.MIPMAP_NEAREST, abi.ADDRESS_REPEAT, abi.ADDRESS_REPEAT)], dtype=abi.SAMPLER_DT)
    table = dict(host=pyoracle.MaterialTable(m, [(texel, abi.IMAGE_RGBA8_UNORM)], smp))
    cam = synth.make_camera(sc.width, sc.height, 1)
    hs, mi, total, v32 = cpu_vis(orc, sc, cam)
    want, _ = oracle_decode(orc, gb, hs, mi, total, cam, v32, table)
    got = want["normal"][v32 != 0xFFFFFFFF]
    assert len(got) > 1000
    m3 = sc.transforms["world"][0].reshape(4, 4)[:3, :3].T.astype(f64)
    jac = np.diag(uv_size) @ rot  # local xy -> uv
    dp = m3[:, :2] @ np.linalg.inv(jac)  # columns dp/du, dp/dv
    n = np.linalg.inv(m3).T @ [0.0, 0.0, 1.0]
    n = n / np.linalg.norm(n) * np.sign(np.linalg.det(m3))
    t_ = dp[:, 0] / np.linalg.norm(dp[:, 0])
    w = np.sign(np.dot(n, np.cross(dp[:, 0], dp[:, 1])))
    b = -w * np.cross(n, t_)
    e = texel[0, 0, :3] / 255.0 * 2.0 - 1.0
    mapped = e[0] * t_ + e[1] * b + e[2] * n
    mapped /= np.linalg.norm(mapped)
    np.testing.assert_array_less(angle(oct_to_vec3(got[:, 2:]), np.broadcast_to(n, (len(got), 3))), 8 * 2.0 ** -23)
    a = angle(oct_to_vec3(got[:, :2]), np.broadcast_to(mapped, (len(got), 3)))
    assert a.max() < 3e-5, a.max()  # measured at most 6.5e-6: the forward differences of a plane seen at 50 degrees
    assert angle(mapped[None], n[None])[0] > 0.3  # the tilt moves the normal well away from n
