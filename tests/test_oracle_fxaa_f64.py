"""An independent binary64 restatement of FXAA, written from the shader text (passes/fxaa/fxaa.slang fs_main with LinearSamplerClamped
and the HLSL max / min NaN rules), against the binary32 oracle (oracle/oxc_oracle_fxaa.c).  Frames: lit frames of the PBR oracle over
the PBR tests' G-buffer planes (as tests/test_oracle_post_f64.py builds them), synthetic HDR frames, and edge, bar and noise frames.

The restatement is binary64 except for the sampler's coordinates, which it forms in binary32 as the shader does (the pixel centre,
the offset taps, the half-pixel shift, the walk's positions and the final uv), so that its bilinear weights are the oracle's; a
binary64 coordinate would put a pixel centre's weights at exactly 0, where binary32 blends in a neighbour by a rounding.  Its lumas
then differ from the oracle's by binary32 roundings, bounded by ROUNDING times the magnitude of the tapped texels and carried through
the square root.  So the discrete decisions can flip between the two: the sign of a luma's dot product where a texel has a negative
channel (sqrt of a negative sum is NaN), the early exit, is_horizontal, is1_steepest, each reached test, and correct_variation (the
sign of the chosen end's delta, and center < local_average).  A decision is within its margin when its operands differ by at most
SPREAD times the largest luma error of the pixel so far plus ROUNDING times their size; such a pixel is ambiguous, and ambiguous
pixels are counted and bounded, not compared: at most AMBIGUOUS_SHARE of a frame, and NOISE_AMBIGUOUS_SHARE of the noise frame.  An exact binary64 tie is ambiguous too: when the six absolute values
of edge_horizontal and edge_vertical open with the same signs, the two are often the same sum of lumas in a different order, which
binary32 rounds apart; on these frames such ties make up most of the ambiguous pixels (about 9 % of a lit or HDR frame, a third of
the noise frame, half of whose texels are black).  is_direction1 and the final max are not discrete: at a
tie of distance1 and distance2, pixel_offset is 0 on either side, and max is continuous.  Every other pixel agrees with the oracle
within TOL times the largest magnitude in its 5 x 5 neighbourhood."""
import numpy as np
import pytest

from tests.test_gpu_fxaa import bars_frame, diagonal_frame, noise_frame
from tests.test_oracle_post_f64 import hdr_frame, lit_frame

ROUNDING = 1e-6         # a few binary32 roundings, relative
SPREAD = 16.0           # the largest factor a decision's operands take from the lumas (edge_horizontal adds eight, two doubled)
TOL = 1e-4              # of the 5 x 5 neighbourhood's largest magnitude
AMBIGUOUS_SHARE = 0.12
NOISE_AMBIGUOUS_SHARE = 0.4
QUALITY = [1.0, 1.0, 1.0, 1.0, 1.0, 1.5, 2.0, 2.0, 2.0, 2.0, 4.0, 8.0]


f32 = np.float32


def vmax(a, b):  # HLSL max: a NaN operand yields the other one
    return a if (b != b or a > b) else b


def vmin(a, b):
    return a if (b != b or a < b) else b


@pytest.fixture(scope="module")
def so():
    import pyoracle_fxaa

    pyoracle_fxaa.build()
    return pyoracle_fxaa


class Restated:
    """fs_main in binary64 on one frame.  pixel() returns the colour; after it, `close` says whether a decision was within its margin
    and `path` holds ('exit',) or ('walk', steps taken, correct_variation)"""

    def __init__(self, frame):
        self.f = frame.astype(np.float64)
        self.h, self.w = frame.shape[:2]

    def decide(self, a, b):
        size = max(abs(a), abs(b)) if a == a and b == b else 0.0
        if abs(a - b) <= SPREAD * self.err + ROUNDING * size:
            self.close = True

    def sample(self, u, v, dx=0, dy=0):
        """Sample(uv, int2(dx, dy)) at binary32 u, v: x = (u * W + dx) - 0.5 in binary32, the blend in binary64"""
        with np.errstate(invalid="ignore", over="ignore"):
            x = f32(f32(f32(u) * f32(self.w)) + f32(dx)) - f32(0.5)
            y = f32(f32(f32(v) * f32(self.h)) + f32(dy)) - f32(0.5)
        x0, y0 = np.floor(np.float64(x)), np.floor(np.float64(y))
        wx, wy = np.float64(x) - x0, np.float64(y) - y0
        ix, iy = (0 if x0 != x0 else int(x0)), (0 if y0 != y0 else int(y0))  # a NaN coordinate: index 0, NaN weights
        cx = [min(max(ix + k, 0), self.w - 1) for k in (0, 1)]
        cy = [min(max(iy + k, 0), self.h - 1) for k in (0, 1)]
        t = [self.f[cy[j], cx[i]] for j in (0, 1) for i in (0, 1)]
        top = t[0] + wx * (t[1] - t[0])
        bot = t[2] + wx * (t[3] - t[2])
        rgb = np.array([q[:3] for q in t])
        finite = rgb[np.isfinite(rgb)]
        self.negative = bool((rgb < 0).any())
        a = [np.abs(q[:3]) for q in t]  # the blend of the magnitudes: the size of the terms binary32 rounds
        atop, abot = a[0] + wx * np.abs(a[1] - a[0]) + wx * a[0], a[2] + wx * np.abs(a[3] - a[2]) + wx * a[2]
        size = atop + wy * np.abs(abot - atop) + wy * atop
        return top + wy * (bot - top), ROUNDING * (float(np.nanmax(size)) if finite.size == rgb.size else 0.0)

    def luma(self, u, v, dx=0, dy=0):
        c, err = self.sample(u, v, dx, dy)
        s = c[0] * 0.299 + c[1] * 0.587 + c[2] * 0.114
        if self.negative and abs(s) <= err:  # its sign: sqrt of a negative sum is NaN
            self.close = True
        if s == s and err > 0:
            self.err = max(self.err, min(np.sqrt(err), err / (2 * np.sqrt(abs(s))) if s else np.inf))
        with np.errstate(invalid="ignore"):
            return np.sqrt(s)

    def pixel(self, px, py):
        self.close, self.err = False, 0.0
        w, h = self.w, self.h
        u, v = f32(f32(px + 0.5) / f32(w)), f32(f32(py + 0.5) / f32(h))
        iu, iv = f32(1.0) / f32(w), f32(1.0) / f32(h)
        L = lambda dx, dy: self.luma(u, v, dx, dy)  # Sample(uv, int2(dx, dy))
        center, _ = self.sample(u, v)
        lc = self.luma(u, v)
        ld, lu, ll, lr = L(0, -1), L(0, 1), L(-1, 0), L(1, 0)
        lmin = vmin(lc, vmin(vmin(ld, lu), vmin(ll, lr)))
        lmax = vmax(lc, vmax(vmax(ld, lu), vmax(ll, lr)))
        rng = lmax - lmin
        self.decide(rng, vmax(0.0312, lmax * 0.125))
        if rng < vmax(0.0312, lmax * 0.125):
            self.path = ("exit",)
            return center
        ldl, lur, lul, ldr = L(-1, -1), L(1, 1), L(-1, 1), L(1, -1)
        eh = abs(-2.0 * ll + (ldl + lul)) + abs(-2.0 * lc + (ld + lu)) * 2.0 + abs(-2.0 * lr + (ldr + lur))
        ev = abs(-2.0 * lu + (lur + lul)) + abs(-2.0 * lc + (ll + lr)) * 2.0 + abs(-2.0 * ld + (ldl + ldr))
        self.decide(eh, ev)
        horizontal = eh >= ev
        step = iv if horizontal else iu
        l1, l2 = (ld, lu) if horizontal else (ll, lr)
        g1, g2 = l1 - lc, l2 - lc
        self.decide(abs(g1), abs(g2))
        gs = 0.25 * vmax(abs(g1), abs(g2))
        if abs(g1) >= abs(g2):
            step, avg = -step, 0.5 * (l1 + lc)
        else:
            avg = 0.5 * (l2 + lc)
        # the coordinates in binary32
        cur = [u, v]
        cur[1 if horizontal else 0] += f32(step * f32(0.5))
        off = [iu, f32(0.0)] if horizontal else [f32(0.0), iv]
        uv1 = [cur[0] - off[0], cur[1] - off[1]]
        uv2 = [cur[0] + off[0], cur[1] + off[1]]

        def end(uv):
            lum = self.luma(uv[0], uv[1])
            e = lum - avg
            self.decide(abs(e), gs)
            return e

        e1, e2 = end(uv1), end(uv2)
        r1, r2 = abs(e1) >= gs, abs(e2) >= gs
        if not r1:
            uv1 = [uv1[0] - off[0] * f32(QUALITY[1]), uv1[1] - off[1] * f32(QUALITY[1])]
        if not r2:
            uv2 = [uv2[0] + off[0] * f32(QUALITY[1]), uv2[1] + off[1] * f32(QUALITY[1])]
        steps = 1
        if not (r1 and r2):
            for i in range(2, 12):
                steps = i
                if not r1:
                    e1 = end(uv1)
                if not r2:
                    e2 = end(uv2)
                r1, r2 = abs(e1) >= gs, abs(e2) >= gs
                if not r1:
                    uv1 = [uv1[0] - off[0] * f32(QUALITY[i]), uv1[1] - off[1] * f32(QUALITY[i])]
                if not r2:
                    uv2 = [uv2[0] + off[0] * f32(QUALITY[i]), uv2[1] + off[1] * f32(QUALITY[i])]
                if r1 and r2:
                    break
        d1 = float(u - uv1[0]) if horizontal else float(v - uv1[1])
        d2 = float(uv2[0] - u) if horizontal else float(uv2[1] - v)
        e = e1 if d1 < d2 else e2
        self.decide(lc, avg)
        self.decide(e, 0.0)
        correct = (e < 0.0) != (lc < avg)
        final = (-vmin(d1, d2) / (d1 + d2) + 0.5) if correct else 0.0
        lavg = (1.0 / 12.0) * (2.0 * ((ld + lu) + (ll + lr)) + (ldl + lul) + (ldr + lur))
        s1 = vmin(vmax(abs(lavg - lc) / rng, 0.0), 1.0)
        s2 = (-2.0 * s1 + 3.0) * s1 * s1
        final = vmax(final, s2 * s2 * 0.75)
        self.path = ("walk", steps, correct)
        fuv = [u, v]
        fuv[1 if horizontal else 0] += f32(f32(final) * step)
        return self.sample(fuv[0], fuv[1])[0]


FRAMES = [("lit-96x64", lambda: lit_frame(96, 64, 1)), ("lit-161x90", lambda: lit_frame(161, 90, 2)),
          ("hdr-128x72", lambda: hdr_frame(128, 72, 3)), ("hdr-67x33", lambda: hdr_frame(67, 33, 4)),
          ("diag-80x48", lambda: diagonal_frame(80, 48, 0.3)), ("bars-72x90", lambda: bars_frame(72, 90)),
          ("noise-48x32", lambda: noise_frame(np.random.default_rng(5), 48, 32))]


def compare(so, frame, label):
    """(ambiguous pixels, paths of the compared pixels); asserts every unambiguous pixel within TOL"""
    h, w = frame.shape[:2]
    got = so.fxaa(frame)
    r = Restated(frame)
    mag = np.abs(frame.astype(np.float64))
    mag[~np.isfinite(mag)] = 0.0
    scale = np.pad(mag.max(axis=2), 2, mode="edge")
    ambiguous, paths = 0, []
    for y in range(h):
        for x in range(w):
            want = r.pixel(x, y)
            if r.close:
                ambiguous += 1
                continue
            paths.append(r.path)
            tol = TOL * scale[y:y + 5, x:x + 5].max() + 1e-30
            err = np.abs(got[y, x].astype(np.float64) - want).max()
            assert err <= tol, f"{label} ({x}, {y}) {r.path}: {got[y, x]} != {want}"
    share = NOISE_AMBIGUOUS_SHARE if label.startswith("noise") else AMBIGUOUS_SHARE
    assert ambiguous <= share * w * h, f"{label}: {ambiguous} ambiguous pixels of {w * h}"
    return ambiguous, paths


@pytest.mark.parametrize("name", [n for n, _ in FRAMES])
def test_restatement_equals_the_oracle(so, name):
    _, paths = compare(so, dict(FRAMES)[name](), name)
    assert sum(p[0] == "walk" for p in paths) >= 100  # the walk is compared on every frame


def test_the_frames_reach_every_path(so):
    """the compared pixels of all frames together take the early exit, a false and a true correct_variation, and a walk that ends
    after every step 1..11 (11 also being the exhausted walk)"""
    seen = set()
    for name, make in FRAMES:
        _, paths = compare(so, make(), name)
        seen |= {p[:2] for p in paths} | {("cv", p[2]) for p in paths if p[0] == "walk"}
    assert ("exit",) in seen and ("cv", False) in seen and ("cv", True) in seen
    assert {("walk", i) for i in range(1, 12)} <= seen, sorted(s for s in seen if s[0] == "walk")
